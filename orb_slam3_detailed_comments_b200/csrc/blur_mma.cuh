// blur_mma.cuh -- K5 on the tensor cores: GaussianBlur 7x7 sigma=2 BORDER_REFLECT_101 in OpenCV's fixed-point form
// (ORBextractor.cc:1629-1637; the same arithmetic as k_blur in extractor_kernels.cuh), both passes as u8 x u8 -> s32 IMMA.
//
//   out[y][x] = ( sum_r sum_c  k[r] k[c] p[y+r-3][x+c-3]  + 32768 ) >> 16,   k = {18, 34, 48, 56, 48, 34, 18}
//
// is a banded integer matrix product, and mma.sync m16n8k32 .u8.u8.s32 computes integer products exactly in any order, so the result
// is bit-identical to k_blur by construction.  One warp owns a 16-column strip of a 128 x 96 tile and walks down it 16 output rows
// at a time:
//
//   pass H   T[x][r] = sum_c Kh[x][c] P[r][c]: A = the banded Kh (16 output columns x 32 window columns, window column c is image
//            column x0 - 4 + c so that the B fragment is 4-byte aligned), B = 8 staged rows, read as plain 32-bit shared-memory words
//            (lane (g, t) holds bytes 4t..4t+3 and 16+4t..19+4t of row g).  One IMMA = 16 columns x 8 rows of T (<= 65280).
//   pass V   out[y][x] = sum_y' Kv[y][y'] T[y'][x]: B comes straight from pass H's accumulators.  Lane (g, t) holds T[rows 2t, 2t+1]
//            of column g (c0, c1) and g + 8 (c2, c3) of every pass-H block; those of blocks 0 and 1 are exactly the bytes of a B
//            fragment b0 (rows 4t..4t+3) under the K permutation sigma(4t + i) = {2t, 2t+1, 8+2t, 9+2t}[i], blocks 2 and 3 give b1
//            (sigma(16 + k) = 16 + sigma(k)).  Permuting the columns of the constant Kv by sigma leaves the product unchanged, so no
//            shuffle and no shared-memory round trip sits between the two passes.  T does not fit a byte: T = 256 hi + lo, one IMMA
//            per plane, acc = 256 acc_hi + acc_lo (the rounding constant 32768 rides in acc_lo's C operand).
//
// 16 output rows need 22 window rows, so a step reads pass-H blocks 0..2 (block 3 is zero in Kv and stays zero in b1) and the last
// block of one step is the first of the next: 2 pass-H + 4 pass-V IMMA per 16 x 16 outputs.  The tile and a 3-pixel halo are
// staged into shared memory with BORDER_REFLECT_101 applied while staging, so the IMMA loop has no edge code; results go through
// shared memory and leave as 16-byte row segments.  Written only inside the level's blur_pitch rows, as k_blur does.
//
// The constant A fragments (Kh and the sigma-permuted Kv) of every lane come from bm_fragments(), which is plain host code: the
// handle uploads its table once, and tests/test_blur_mma_emul.py builds the same table on the host and replays the kernel's
// dataflow lane by lane against the oracle.
#pragma once
#include <stdint.h>

#include "devmath.cuh"

namespace orbdev {

// the Q0.8 taps of OpenCV's 7x7 sigma=2 kernel; zero outside 0..6
inline int bm_tap(int d) {
    static const int k[7] = {18, 34, 48, 56, 48, 34, 18};
    return d >= 0 && d < 7 ? k[d] : 0;
}
// window row that K index k of a pass-V fragment stands for (the accumulator layout of pass H, see above)
inline int bm_sigma(int k) {
    const int q = k & 15, t = q >> 2, i = q & 3;
    return (k & 16) + (i < 2 ? 2 * t + i : 8 + 2 * t + (i - 2));
}
// frag[r * 32 + lane]: r = 0..3 the A fragment of Kh (pass H), r = 4..7 that of the sigma-permuted Kv (pass V).
// m16n8k32 A layout: register r of lane (g = lane / 4, t = lane % 4) holds row g + 8 (r & 1), columns 16 (r >> 1) + 4t .. + 3.
inline void bm_fragments(uint32_t* frag) {
    for (int r = 0; r < 4; ++r)
        for (int lane = 0; lane < 32; ++lane) {
            const int m = (lane >> 2) + 8 * (r & 1);
            uint32_t h = 0, v = 0;
            for (int i = 0; i < 4; ++i) {
                const int k = 16 * (r >> 1) + 4 * (lane & 3) + i;
                h |= (uint32_t)bm_tap(k - m - 1) << (8 * i);         // Kh[x][c]: window column c = image column x0 - 4 + c
                v |= (uint32_t)bm_tap(bm_sigma(k) - m) << (8 * i);   // Kv[y][y']: window row y' = image row y0 - 3 + y'
            }
            frag[r * 32 + lane] = h;
            frag[(4 + r) * 32 + lane] = v;
        }
}

}  // namespace orbdev

#define BM_TW 128                      // columns per CTA: 8 warps x 16
#define BM_TH 96                       // output rows per CTA: 6 steps of 16
#define BM_SROW 144                    // bytes per staged row: image columns X0 - 8 .. X0 + 135 (36 words: conflict-free B loads)

#if defined(__CUDACC__)
namespace orb {

struct BlurMmaPlan {
    const uint32_t* frag;              // bm_fragments() table, 8 x 32 words
    int tileBase[ORB_MAX_LEVELS + 1];  // first tile of every level (BM_TW x BM_TH tiles)
    int tilesX[ORB_MAX_LEVELS];
};

// Launches k_blur_mma (csrc/blur_mma.cu) on `st`: grid (tiles, batch).  The kernel is built into its own library,
// liborbslam3_b200_blur.so, which liborbslam3_b200.so links: the launch error, if any, is returned here.
cudaError_t launch_blur_mma(const ExtractGeom& g, const BlurMmaPlan& p, int tiles, int batch, cudaStream_t st);

}  // namespace orb
#endif
