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

#if defined(__CUDACC__)   // BlurMmaPlan and k_blur_mma, compiled into extractor.cu (the host emulation builds only the part above)
namespace orb {

struct BlurMmaPlan {
    const uint32_t* frag;              // bm_fragments() table, 8 x 32 words
    int tileBase[ORB_MAX_LEVELS + 1];  // first tile of every level (BM_TW x BM_TH tiles)
    int tilesX[ORB_MAX_LEVELS];
};

__device__ __forceinline__ void bm_mma(int (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1, int c) {
    asm("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};"
        : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "r"(c));
}

// pass H of the 8 staged rows starting at `row` (already offset by this lane's g): the accumulators as (lo, lo, hi, hi) byte pairs
// of columns g (p0) and g + 8 (p1), rows 2t and 2t + 1
__device__ __forceinline__ void bm_pass_h(const uint32_t* row, const uint32_t (&ah)[4], uint32_t& p0, uint32_t& p1) {
    int d[4];
    bm_mma(d, ah, row[0], row[4], 0);
    p0 = __byte_perm(d[0], d[1], 0x5140);
    p1 = __byte_perm(d[2], d[3], 0x5140);
}

// pass V of 8 columns from the byte pairs of pass-H blocks a, b, c; stores output rows g and g + 8, columns 2t, 2t + 1
__device__ __forceinline__ void bm_pass_v(uint32_t a, uint32_t b, uint32_t c, const uint32_t (&av)[4], uint8_t* out) {
    int lo[4], hi[4];
    bm_mma(lo, av, __byte_perm(a, b, 0x5410), c & 0xffffu, 32768);
    bm_mma(hi, av, __byte_perm(a, b, 0x7632), c >> 16, 0);
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = (uint32_t)lo[i] + ((uint32_t)hi[i] << 8);   // < 2^24: byte 2 is the result
    *reinterpret_cast<uint16_t*>(out) = (uint16_t)__byte_perm(o[0], o[1], 0x0062);
    *reinterpret_cast<uint16_t*>(out + 8 * BM_SROW) = (uint16_t)__byte_perm(o[2], o[3], 0x0062);
}

__device__ __forceinline__ int bm_reflect(int i, int n) {   // BORDER_REFLECT_101 for an overshoot of a few pixels
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return i;
}

__global__ void __launch_bounds__(256) k_blur_mma(const __grid_constant__ ExtractGeom g, const __grid_constant__ BlurMmaPlan P) {
    __shared__ __align__(16) uint8_t s_in[(BM_TH + 8) * BM_SROW + 16];   // + 2 rows and 16 bytes read under zero weights only
    __shared__ __align__(16) uint8_t s_out[BM_TH * BM_SROW];
    const int tileId = blockIdx.x, img = blockIdx.y;
    int l = 0;
    while (l + 1 < g.nlevels && tileId >= P.tileBase[l + 1]) ++l;
    const LevelGeom& G = g.lv[l];
    const int local = tileId - P.tileBase[l];
    const int ty = local / P.tilesX[l], tx = local - ty * P.tilesX[l];
    const int X0 = tx * BM_TW, Y0 = ty * BM_TH;
    const int w = G.w, h = G.h;
    const uint8_t* __restrict__ src = G.base + (int64_t)img * G.img_stride;

    // stage rows Y0 - 3 .. Y0 + BM_TH + 2 (those up to h + 2), columns X0 - 8 .. X0 + 135: the 8-byte words that lie inside the
    // row (a caller-owned level 0 is only 8-byte aligned), then byte by byte the reflected columns -3 .. -1 and the columns from the
    // last whole word to w + 2.  No load waits for another: the words go by cp.async, the edge bytes are all loaded before the first
    // is stored.  (A byte path that packs its word inside the word loop waits out one memory round trip per word, and nearly every
    // warp of a tile at a left or right image edge holds such a word: 0.169 instead of 0.138 ms per 128-image batch on an H100, both
    // at six CTAs per SM.  Without a register cap the kernel takes 48 registers and runs five CTAs per SM: 0.130 ms; capped at six, 40
    // registers and a spill: 0.138 ms.)
    // What is not staged (columns -8 .. -4, past w + 2, rows past h + 2) feeds zero weights, pitch padding or rows that are not stored.
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gq = lane >> 2, tq = lane & 3;
    uint32_t ah[4], av[4];   // issued first: their latency hides behind the staging
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        ah[r] = __ldg(P.frag + r * 32 + lane);
        av[r] = __ldg(P.frag + (4 + r) * 32 + lane);
    }
    const int srows = min(BM_TH + 6, h - Y0 + 6);
    constexpr int kWords = (BM_TH + 6) * (BM_SROW / 8);
#pragma unroll
    for (int idx = threadIdx.x; idx < kWords; idx += 256) {   // cp.async: every word in flight at once, none through registers
        const int i = idx / (BM_SROW / 8), c = X0 - 8 + 8 * (idx - i * (BM_SROW / 8));
        if (i < srows && c >= 0 && c + 8 <= w)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(s_in + 8 * idx)),
                         "l"(src + (int64_t)bm_reflect(Y0 - 3 + i, h) * G.pitch + c)
                         : "memory");
    }
    const int nL = X0 == 0 ? 3 : 0;                                                       // columns -3 .. -1
    const int rBeg = max(w & ~7, X0 - 8), nR = max(min(w + 3, X0 + BM_SROW - 8) - rBeg, 0);   // columns rBeg .. w + 2
    const int per = nL + nR;                                                              // <= 3 + 10
    if (per > 0) {   // CTA-uniform
        constexpr int kEdge = ((BM_TH + 6) * 13 + 255) / 256;
        uint32_t eb[kEdge];   // shared-memory offset << 8 | byte; ~0 = nothing to stage
#pragma unroll
        for (int e = 0; e < kEdge; ++e) {
            const int idx = threadIdx.x + 256 * e, i = idx / per, j = idx - i * per;
            const int col = j < nL ? j - 3 : rBeg + (j - nL);
            eb[e] = i < srows ? ((uint32_t)(i * BM_SROW + col - (X0 - 8)) << 8) |
                                    __ldg(src + (int64_t)bm_reflect(Y0 - 3 + i, h) * G.pitch + bm_reflect(col, w))
                              : ~0u;
        }
#pragma unroll
        for (int e = 0; e < kEdge; ++e)
            if (eb[e] != ~0u) s_in[eb[e] >> 8] = (uint8_t)eb[e];
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
    __syncthreads();

    if (X0 + 16 * warp < w) {   // warp-uniform
        // window column 4t of this warp's strip: byte 16 warp + 4 + 4t of a staged row
        const uint32_t* in = reinterpret_cast<const uint32_t*>(s_in) + gq * (BM_SROW / 4) + 4 * warp + 1 + tq;
        uint8_t* out = s_out + gq * BM_SROW + 16 * warp + 2 * tq;
        const int steps = min(BM_TH, h - Y0 + 15) >> 4;
        uint32_t a0, a1;
        bm_pass_h(in, ah, a0, a1);
        for (int s = 0; s < steps; ++s) {
            uint32_t b0, b1, c0, c1;
            bm_pass_h(in + (16 * s + 8) * (BM_SROW / 4), ah, b0, b1);
            bm_pass_h(in + (16 * s + 16) * (BM_SROW / 4), ah, c0, c1);
            bm_pass_v(a0, b0, c0, av, out + 16 * s * BM_SROW);       // columns 0..7 of the strip
            bm_pass_v(a1, b1, c1, av, out + 16 * s * BM_SROW + 8);   // columns 8..15
            a0 = c0;
            a1 = c1;
        }
    }
    __syncthreads();

    uint8_t* __restrict__ dst = G.blur + (int64_t)img * G.blur_stride;
    const int rows = min(BM_TH, h - Y0);
    for (int idx = threadIdx.x; idx < rows * (BM_TW / 16); idx += 256) {
        const int r = idx / (BM_TW / 16), q = idx % (BM_TW / 16);
        if (X0 + 16 * q < w)   // pitch padding absorbs the tail: blur_pitch = round_up(w, 16)
            *reinterpret_cast<uint4*>(dst + (int64_t)(Y0 + r) * G.blur_pitch + X0 + 16 * q) =
                *reinterpret_cast<const uint4*>(s_out + r * BM_SROW + 16 * q);
    }
}

}  // namespace orb
#endif
