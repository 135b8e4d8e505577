// extractor_kernels.cuh -- sm_90a kernels of ORBextractor::operator()
// (/root/reference/src/ORBextractor.cc:1557-1682).  All kernels are batched: blockIdx.{y|z} or a
// division of blockIdx.x selects the image, so one launch covers a whole batch of frames.
#pragma once
#include "common.cuh"
#include "devmath.cuh"
#include "quadtree_core.cuh"
#include "resize_core.cuh"

namespace orb {
using namespace orbdev;

// umax of the radius-15 disc (ORBextractor.cc:542-570), verified against the constructor's
// arithmetic on the host at handle creation.
__device__ __constant__ int c_umax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};

// ---------------------------------------------------------------------------------------------
// K1  ComputePyramid (ORBextractor.cc:1687-1738): level l from level l-1, cv::resize INTER_LINEAR
// fixed-point model (SURVEY App. A.1).  One thread = 4 destination pixels = one 32-bit store.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_resize(const __grid_constant__ ExtractGeom g, int l, const int2* __restrict__ taps) {
    const LevelGeom& D = g.lv[l];
    const LevelGeom& S = g.lv[l - 1];
    const int dx4 = (blockIdx.x * 32 + threadIdx.x) * 4;
    const int dy = blockIdx.y * 8 + threadIdx.y;
    if (dx4 >= D.w || dy >= D.h) return;
    const uint8_t* src = S.base + (int64_t)blockIdx.z * S.img_stride;
    uint8_t* dst = D.base + (int64_t)blockIdx.z * D.img_stride;
    uint32_t packed = 0;
    if (D.area2x) {
        const uint8_t* a = src + (int64_t)(2 * dy) * S.pitch;
        const uint8_t* b = a + S.pitch;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int x = dx4 + i;
            if (x < D.w) {
                const int v = (a[2 * x] + a[2 * x + 1] + b[2 * x] + b[2 * x + 1] + 2) >> 2;
                packed |= (uint32_t)v << (8 * i);
            }
        }
    } else {
        const int2 ty = __ldg(&taps[D.tapOff + D.w + dy]);
        const int sy0 = ty.x, sy1 = min(sy0 + 1, S.h - 1);
        const int b0 = ty.y & 0xffff, b1 = (int)((uint32_t)ty.y >> 16);
        const uint8_t* a = src + (int64_t)sy0 * S.pitch;
        const uint8_t* b = src + (int64_t)sy1 * S.pitch;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int x = dx4 + i;
            if (x < D.w) {
                const int2 tx = __ldg(&taps[D.tapOff + x]);
                const int x0 = tx.x, x1 = min(x0 + 1, S.w - 1);
                const int c0 = tx.y & 0xffff, c1 = (int)((uint32_t)tx.y >> 16);
                const int r0 = (int)__ldg(a + x0) * c0 + (int)__ldg(a + x1) * c1;
                const int r1 = (int)__ldg(b + x0) * c0 + (int)__ldg(b + x1) * c1;
                const int v = (((b0 * (r0 >> 4)) >> 16) + ((b1 * (r1 >> 4)) >> 16) + 2) >> 2;
                packed |= (uint32_t)v << (8 * i);
            }
        }
    }
    *reinterpret_cast<uint32_t*>(dst + (int64_t)dy * D.pitch + dx4) = packed;
}

// k_resize_v2: one thread = 4 destination pixels x RS2_ROWS (4 or 8) destination rows.  The x taps are decoded once per thread, and the
// horizontal interpolation of a source row is computed once and shared by the two destination rows that read it (at scale 1.2 four
// out of five destination rows start on the source row the previous one ended on), so a destination pixel costs ~1.4 source-row
// interpolations instead of 2 and a quarter of the tap / address work.  Same arithmetic, same order: bit-exact with k_resize.
template <int RS2_ROWS>
__global__ void __launch_bounds__(256) k_resize_v2(const __grid_constant__ ExtractGeom g, int l, const int2* __restrict__ taps) {
    const LevelGeom& D = g.lv[l];
    const LevelGeom& S = g.lv[l - 1];
    const int dx4 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4;
    const int dy0 = (blockIdx.y * 8 + (threadIdx.x >> 5)) * RS2_ROWS;
    if (dx4 >= D.w || dy0 >= D.h) return;
    const uint8_t* __restrict__ src = S.base + (int64_t)blockIdx.z * S.img_stride;
    uint8_t* __restrict__ dst = D.base + (int64_t)blockIdx.z * D.img_stride + dx4;
    int xo0[4], xo1[4], c0[4], c1[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int2 tx = __ldg(&taps[D.tapOff + min(dx4 + i, D.w - 1)]);   // columns past the width feed the pitch padding only
        xo0[i] = tx.x; xo1[i] = min(tx.x + 1, S.w - 1);
        c0[i] = tx.y & 0xffff; c1[i] = (int)((uint32_t)tx.y >> 16);
    }
    int have = -1;     // source row whose horizontal interpolation sits in hc[]
    int hc[4] = {0, 0, 0, 0};
    const int nrow = min(RS2_ROWS, D.h - dy0);
    for (int k = 0; k < nrow; ++k) {   // warp-uniform: a warp is 32 threads of one destination row group
        const int2 ty = __ldg(&taps[D.tapOff + D.w + dy0 + k]);
        const int sy0 = ty.x, sy1 = min(sy0 + 1, S.h - 1);
        const int b0 = ty.y & 0xffff, b1 = (int)((uint32_t)ty.y >> 16);
        int h0[4], h1[4];
        if (sy0 == have) {
#pragma unroll
            for (int i = 0; i < 4; ++i) h0[i] = hc[i];
        } else {
            const uint8_t* a = src + (int64_t)sy0 * S.pitch;
#pragma unroll
            for (int i = 0; i < 4; ++i) h0[i] = ((int)__ldg(a + xo0[i]) * c0[i] + (int)__ldg(a + xo1[i]) * c1[i]) >> 4;
        }
        if (sy1 == sy0) {
#pragma unroll
            for (int i = 0; i < 4; ++i) h1[i] = h0[i];
        } else {
            const uint8_t* b = src + (int64_t)sy1 * S.pitch;
#pragma unroll
            for (int i = 0; i < 4; ++i) h1[i] = ((int)__ldg(b + xo0[i]) * c0[i] + (int)__ldg(b + xo1[i]) * c1[i]) >> 4;
        }
        uint32_t packed = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int v = (((b0 * h0[i]) >> 16) + ((b1 * h1[i]) >> 16) + 2) >> 2;
            packed |= (uint32_t)v << (8 * i);
            hc[i] = h1[i];
        }
        have = sy1;
        if (dx4 + 4 > D.w) packed &= 0xffffffffu >> (8 * (dx4 + 4 - D.w));   // as k_resize: zero past the width
        *reinterpret_cast<uint32_t*>(dst + (int64_t)(dy0 + k) * D.pitch) = packed;
    }
}

// k_resize_v3: k_resize_v2's work split, the source rows by aligned word loads + PRMT + IDP.2A (resize_core.cuh).
__global__ void __launch_bounds__(256) k_resize_v3(const __grid_constant__ ExtractGeom g, int l, const int2* __restrict__ taps, const uint8_t* src_end) {
    const LevelGeom& D = g.lv[l];
    const LevelGeom& S = g.lv[l - 1];
    const int dx4 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 4;
    const int dy0 = (blockIdx.y * 8 + (threadIdx.x >> 5)) * 4;
    if (dx4 >= D.w || dy0 >= D.h) return;
    const int* t2 = reinterpret_cast<const int*>(taps + D.tapOff);
    rs_thread<4>(S.base + (int64_t)blockIdx.z * S.img_stride, S.w, S.h, S.pitch, src_end, D.base + (int64_t)blockIdx.z * D.img_stride, D.w, D.h,
                 D.pitch, t2, t2 + 2 * D.w, dx4, dy0);
}

// ---------------------------------------------------------------------------------------------
// K2  per-cell FAST-9/16 + NMS + 20->7 fallback (ORBextractor.cc:1069-1166, SURVEY App. A.3).
// One CTA = one 35-px cell of one level of one image.  The cell window (+ alignment slack) is
// staged in shared memory as 32-bit words; each thread scores 4 adjacent pixels per task with the
// packed 16x2 DPX form (VIMNMX3.U16x2), NMS runs on the byte-packed score map, survivors are
// appended to the level's candidate list (order-free: the quadtree re-derives the reference order
// from the coordinates).
// ---------------------------------------------------------------------------------------------
#define FAST_ROWS 76   // upper bound on the staged rows of a cell (hCell + 6); the kernel sizes its arrays from ExtractGeom::fastRows
#define FAST_TW 22
#define FAST_THREADS 128

__device__ __forceinline__ uint32_t shift_word(uint32_t L, uint32_t C, uint32_t R, int dx) {
    switch (dx) {
        case 1: return __byte_perm(C, R, 0x4321);
        case 2: return __byte_perm(C, R, 0x5432);
        case 3: return __byte_perm(C, R, 0x6543);
        case -1: return __byte_perm(L, C, 0x6543);
        case -2: return __byte_perm(L, C, 0x5432);
        case -3: return __byte_perm(L, C, 0x4321);
        default: return C;
    }
}

#define FAST_PW 46   // 16x2-packed pixel pairs per staged row (tile width <= 88 px)

__global__ void __launch_bounds__(FAST_THREADS) k_fast_cells(const __grid_constant__ ExtractGeom g, uint32_t* __restrict__ cand,
                                                            int* __restrict__ candCnt, int* __restrict__ err) {
    // The window is staged twice as 16x2-packed pixel pairs: pe[r][i] = (px 2i, px 2i+1), po[r][i] = (px 2i+1, px 2i+2).
    // Every ring sample of a pixel pair is then ONE 32-bit shared-memory load already in the layout the packed DPX
    // min/max instructions want (no per-sample byte permutes).  Rows are sized for the tallest cell of this geometry.
    extern __shared__ __align__(16) uint32_t fast_smem[];
    const int R = g.fastRows;
    uint32_t (*pe)[FAST_PW] = reinterpret_cast<uint32_t (*)[FAST_PW]>(fast_smem);
    uint32_t (*po)[FAST_PW] = pe + R;
    uint32_t (*se)[FAST_PW] = po + R;   // scores >= T (else 0) of the even-aligned pairs, 16x2
    // NMS result, one byte per pixel; the list of pixel pairs that pass the high-speed test lives in the same bytes
    // (dead before the NMS writes)
    uint32_t (*tile)[FAST_TW] = reinterpret_cast<uint32_t (*)[FAST_TW]>(se + R);
    uint16_t* lst = reinterpret_cast<uint16_t*>(tile);
    __shared__ int s_warp[FAST_THREADS / 32 + 1];
    __shared__ int s_base;
    __shared__ int s_nlist;

    const int cell = blockIdx.x, img = blockIdx.y, tid = threadIdx.x;
    int l = 0;
    while (l + 1 < g.nlevels && cell >= g.lv[l + 1].cellBase) ++l;
    const LevelGeom& G = g.lv[l];
    const int local = cell - G.cellBase;
    const int ci = local / G.nCols, cj = local - ci * G.nCols;
    const int x0 = 16 + cj * G.wCell, y0 = 16 + ci * G.hCell;
    if (x0 >= G.maxBX - 6 || y0 >= G.maxBY - 3) return;  // ORBextractor.cc:1105,1120
    const int x1 = min(x0 + G.wCell + 6, G.maxBX), y1 = min(y0 + G.hCell + 6, G.maxBY);
    const int cw = x1 - x0, ch = y1 - y0;
    if (cw < 7 || ch < 7) return;  // cv::FAST tests nothing
    const int tx0 = x0 + 3, tx1 = x1 - 3, ty0 = y0 + 3, ty1 = y1 - 3;
    const int gx0 = (tx0 & ~3) - 4;
    const int ngrp = ((tx1 - 1) >> 2) - (tx0 >> 2) + 1;
    const int nW = ngrp + 2;   // <= 21 words per staged row
    // (t * magic) >> 20 == t / n exactly for t < 2048, n <= 32 (checked exhaustively); ntask <= 1330
    const uint32_t magicG = (1u << 20) / (uint32_t)ngrp + 1u;
    const uint8_t* src = G.base + (int64_t)img * G.img_stride + (int64_t)y0 * G.pitch + gx0;

    {   // staging: one thread per 32-bit word of the window (flat index => every thread has several independent
        // global loads in flight); the following word is re-read through L1 instead of a second shared-memory pass
        const uint32_t magicW = (1u << 20) / (uint32_t)nW + 1u;   // exact for i < 2048 (ch * nW <= 1596)
        for (int i = tid; i < ch * nW; i += FAST_THREADS) {
            const int r = (int)(((uint32_t)i * magicW) >> 20), c = i - r * nW;
            const uint32_t* rowp = reinterpret_cast<const uint32_t*>(src + (int64_t)r * G.pitch);
            const uint32_t w = __ldg(rowp + c);
            const uint32_t nx = (c + 1 < nW) ? __ldg(rowp + c + 1) : 0u;
            *reinterpret_cast<uint2*>(&pe[r][2 * c]) = make_uint2(__byte_perm(w, 0u, 0x4140), __byte_perm(w, 0u, 0x4342));
            *reinterpret_cast<uint2*>(&po[r][2 * c]) = make_uint2(__byte_perm(w, 0u, 0x4241), (w >> 24) | ((nx & 0xffu) << 16));
            *reinterpret_cast<uint2*>(&se[r][2 * c]) = make_uint2(0u, 0u);
        }
    }
    if (tid == 0) s_nlist = 0;
    __syncthreads();

    const int ntask = (ty1 - ty0) * ngrp;          // one task = 4 adjacent pixels = two 16x2 pairs
    const int ntaskW = (ntask + 31) & ~31;         // warp-uniform trip count (ballots inside)
    const int lane = tid & 31, wid = tid >> 5;
    const unsigned lt = (1u << lane) - 1u;
    int thr = g.iniTh;
    // Frame cells are searched at iniThFAST first and, only if that leaves the cell empty, again at minThFAST
    // (ORBextractor.cc:1135-1148).  A corner at threshold T has score >= T, and a score below T never suppresses one
    // at or above it, so each pass only needs the scores >= its own T.
    for (int pass = 0; pass < 2; ++pass) {
        thr = pass ? g.minTh : g.iniTh;
        const uint32_t T2p1 = (uint32_t)(thr + 1) * 0x00010001u;
        // A: high-speed test of every pixel pair; the survivors are compacted into lst[]
        for (int t = tid; t < ntaskW; t += FAST_THREADS) {
            uint32_t pa = 0u, pb = 0u;
            int code = 0;
            if (t < ntask) {
                const int row = (int)(((uint32_t)t * magicG) >> 20), grp = t - row * ngrp;
                const int r = row + 3, pA = 2 * (grp + 1);
                code = r * 64 + pA;
                // antipodal ring pairs (0,8) (2,10) (4,12) (6,14): (dx,dy) = (0,-3)/(0,3) (2,-2)/(-2,2) (3,0)/(-3,0) (2,2)/(-2,-2)
                const uint32_t *q0 = &pe[r - 3][pA], *q8 = &pe[r + 3][pA], *q2 = &pe[r - 2][pA + 1], *q10 = &pe[r + 2][pA - 1];
                const uint32_t *q4 = &po[r][pA + 1], *q12 = &po[r][pA - 2], *q6 = &pe[r + 2][pA + 1], *q14 = &pe[r - 2][pA - 1];
                const uint2 c = *reinterpret_cast<const uint2*>(&pe[r][pA]);   // pA is even: 8-byte aligned
                const uint32_t hiA = min_u16x2(min3_u16x2(max_u16x2(q0[0], q8[0]), max_u16x2(q2[0], q10[0]), max_u16x2(q4[0], q12[0])),
                                               max_u16x2(q6[0], q14[0]));
                const uint32_t loA = max_u16x2(max3_u16x2(min_u16x2(q0[0], q8[0]), min_u16x2(q2[0], q10[0]), min_u16x2(q4[0], q12[0])),
                                               min_u16x2(q6[0], q14[0]));
                const uint32_t hiB = min_u16x2(min3_u16x2(max_u16x2(q0[1], q8[1]), max_u16x2(q2[1], q10[1]), max_u16x2(q4[1], q12[1])),
                                               max_u16x2(q6[1], q14[1]));
                const uint32_t loB = max_u16x2(max3_u16x2(min_u16x2(q0[1], q8[1]), min_u16x2(q2[1], q10[1]), min_u16x2(q4[1], q12[1])),
                                               min_u16x2(q6[1], q14[1]));
                pa = fast_pretest_x2(c.x, hiA, loA, T2p1);
                pb = fast_pretest_x2(c.y, hiB, loB, T2p1);
            }
            const unsigned ma = __ballot_sync(0xffffffffu, pa != 0u), mb = __ballot_sync(0xffffffffu, pb != 0u);
            const int na = __popc(ma), n = na + __popc(mb);
            if (n) {   // warp-uniform
                int base = 0;
                if (lane == 0) base = atomicAdd(&s_nlist, n);
                base = __shfl_sync(0xffffffffu, base, 0);
                if (pa) lst[base + __popc(ma & lt)] = (uint16_t)code;
                if (pb) lst[base + na + __popc(mb & lt)] = (uint16_t)(code + 1);
            }
        }
        __syncthreads();
        // B: full score of the listed pairs only
        const int nl = s_nlist;
        for (int i = tid; i < nl; i += FAST_THREADS) {
            const int code = lst[i], r = code >> 6, p = code & 63;
            uint32_t ring[16];
            // ring offsets (dx,dy) clockwise from the top: even dx -> pe at p + dx/2, odd dx -> po at p + (dx-1)/2
#define RING_E(k, dy, h) ring[k] = pe[r + (dy)][p + (h)];
#define RING_O(k, dy, h) ring[k] = po[r + (dy)][p + (h)];
            RING_E(0, -3, 0)  RING_O(1, -3, 0)  RING_E(2, -2, 1)  RING_O(3, -1, 1)
            RING_O(4, 0, 1)   RING_O(5, 1, 1)   RING_E(6, 2, 1)   RING_O(7, 3, 0)
            RING_E(8, 3, 0)   RING_O(9, 3, -1)  RING_E(10, 2, -1) RING_O(11, 1, -2)
            RING_O(12, 0, -2) RING_O(13, -1, -2) RING_E(14, -2, -1) RING_O(15, -3, -1)
#undef RING_E
#undef RING_O
            const uint32_t s01 = fast_score_x2(pe[r][p], ring);
            const int xb = gx0 + 2 * p;
            const int s0 = (int)(s01 & 0xffffu) - 256, s1 = (int)(s01 >> 16) - 256;
            const uint32_t k0 = (s0 >= thr && xb >= tx0 && xb < tx1) ? (uint32_t)s0 : 0u;
            const uint32_t k1 = (s1 >= thr && xb + 1 >= tx0 && xb + 1 < tx1) ? (uint32_t)s1 : 0u;
            se[r][p] = k0 | (k1 << 16);
        }
        __syncthreads();

        // NMS on the 16x2 score map with packed 3-input max; the result is byte-packed per 4 pixels into tile[][]
        int has = 0;
        for (int t = tid; t < ntask; t += FAST_THREADS) {
            const int row = (int)(((uint32_t)t * magicG) >> 20), grp = t - row * ngrp;
            const int r = row + 3, wd = grp + 1, pA = 2 * wd;
            const uint32_t cA = se[r][pA], cB = se[r][pA + 1];
            uint32_t res = 0u;
            if ((cA | cB) != 0u) {
                const uint32_t* u = &se[r - 1][pA - 1];
                const uint32_t* m = &se[r][pA - 1];
                const uint32_t* d = &se[r + 1][pA - 1];
                const uint32_t u0 = u[0], u1 = u[1], u2 = u[2], u3 = u[3], m0 = m[0], m3 = m[3], d0 = d[0], d1 = d[1], d2 = d[2], d3 = d[3];
                // odd-aligned pairs (px 2i-1, 2i) / (px 2i+1, 2i+2) from two even pairs
                const uint32_t uA = max3_u16x2(__byte_perm(u0, u1, 0x5432), u1, __byte_perm(u1, u2, 0x5432));
                const uint32_t dA = max3_u16x2(__byte_perm(d0, d1, 0x5432), d1, __byte_perm(d1, d2, 0x5432));
                const uint32_t mA = max_u16x2(__byte_perm(m0, cA, 0x5432), __byte_perm(cA, cB, 0x5432));
                const uint32_t uB = max3_u16x2(__byte_perm(u1, u2, 0x5432), u2, __byte_perm(u2, u3, 0x5432));
                const uint32_t dB = max3_u16x2(__byte_perm(d1, d2, 0x5432), d2, __byte_perm(d2, d3, 0x5432));
                const uint32_t mB = max_u16x2(__byte_perm(cA, cB, 0x5432), __byte_perm(cB, m3, 0x5432));
                const uint32_t mxA = max3_u16x2(uA, dA, mA), mxB = max3_u16x2(uB, dB, mB);
                // strictly greater than all 8 neighbours: c >= mx + 1  <=>  max(c, mx + 1) == c   (scores <= 254)
                const uint32_t gA = max_u16x2(cA, mxA + 0x00010001u) ^ cA, gB = max_u16x2(cB, mxB + 0x00010001u) ^ cB;
                const uint32_t r0 = (gA & 0xffffu) ? 0u : (cA & 0xffffu), r1 = (gA >> 16) ? 0u : (cA >> 16);
                const uint32_t r2 = (gB & 0xffffu) ? 0u : (cB & 0xffffu), r3 = (gB >> 16) ? 0u : (cB >> 16);
                res = r0 | (r1 << 8) | (r2 << 16) | (r3 << 24);
                has |= (res != 0u);
            }
            tile[r][wd] = res;
        }
        if (__syncthreads_or(has) || pass == 1) break;  // also orders the tile[] writes
        // empty at iniThFAST: clear the score map and run the cell again at minThFAST
        for (int i = tid; i < ch * nW; i += FAST_THREADS) {
            const int r = (int)(((uint32_t)i * ((1u << 20) / (uint32_t)nW + 1u)) >> 20), c = i - r * nW;
            *reinterpret_cast<uint2*>(&se[r][2 * c]) = make_uint2(0u, 0u);
        }
        if (tid == 0) s_nlist = 0;
        __syncthreads();
    }
    const uint32_t thr4 = (uint32_t)thr * 0x01010101u;

    int cnt = 0;
    for (int t = tid; t < ntask; t += FAST_THREADS) {
        const int row = (int)(((uint32_t)t * magicG) >> 20), grp = t - row * ngrp;
        const uint32_t v = tile[row + 3][grp + 1];
        if (v) cnt += __popc(__vcmpgeu4(v, thr4) & 0x01010101u);
    }
    // CTA exclusive scan of cnt
    int inc = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int w = 0; w < FAST_THREADS / 32; ++w) {
            const int v = s_warp[w];
            s_warp[w] = run;
            run += v;
        }
        s_base = run ? atomicAdd(&candCnt[img * g.nlevels + l], run) : 0;
        s_warp[FAST_THREADS / 32] = run;
    }
    __syncthreads();
    const int total = s_warp[FAST_THREADS / 32];
    if (total == 0) return;
    int off = s_base + s_warp[wid] + inc - cnt;
    if (s_base + total > G.candCap) {
        if (tid == 0) atomicExch(&err[0], 1);
        return;
    }
    uint32_t* out = cand + (int64_t)img * g.candTotal + G.candOff;
    for (int t = tid; t < ntask; t += FAST_THREADS) {
        const int row = (int)(((uint32_t)t * magicG) >> 20), grp = t - row * ngrp;
        const uint32_t v = tile[row + 3][grp + 1];
        if (!v) continue;
        const int xb = gx0 + 4 * (grp + 1) - 16, yb = ty0 + row - 16;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t s = (v >> (8 * k)) & 0xffu;
            if (s >= (uint32_t)thr) out[off++] = qt_pack_cand(xb + k, yb, (int)s);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// K3  DistributeOctTree, one CTA per (level, image); see quadtree_core.cuh.
// ---------------------------------------------------------------------------------------------
#define QT_THREADS 256

// arr / ws are passed from branch-specific call sites so that the shared-memory instance is compiled
// with LDS/STS instead of generic loads.
__device__ __forceinline__ int qt_run(uint32_t* arr, void* ws, int cap, int n, int npow, const uint32_t* __restrict__ src,
                                      const QtGeom& q, uint32_t* out) {
    for (int i = threadIdx.x; i < npow; i += QT_THREADS) arr[i] = (i < n) ? qt_element(src[i], q) : 0xffffffffu;
    __syncthreads();
    qt_bitonic_sort(arr, npow);
    QtWork w;
    qt_work_carve(w, ws, cap);
    return qt_distribute(arr, n, q, w, out);
}

// levels [levelBegin, levelEnd) of every image; blockIdx.x = (level - levelBegin) * batch + image
__global__ void __launch_bounds__(QT_THREADS) k_quadtree(const __grid_constant__ ExtractGeom g, int batch, int levelBegin,
                                                        const uint32_t* __restrict__ cand, const int* __restrict__ candCnt,
                                                        uint32_t* __restrict__ sortScratch, char* __restrict__ nodeScratch,
                                                        int64_t nodeScratchStride, int sortCapSmem, int nodesInSmem,
                                                        int nodeCapMax, uint32_t* __restrict__ lvlKp, int* __restrict__ lvlCnt,
                                                        int* __restrict__ err) {
    extern __shared__ __align__(16) unsigned char qt_smem[];
    const int l = levelBegin + blockIdx.x / batch, img = blockIdx.x % batch;
    const LevelGeom& G = g.lv[l];
    int n = candCnt[img * g.nlevels + l];
    if (n > G.candCap) n = G.candCap;
    QtGeom q;
    q.regionW = G.maxBX - 16; q.regionH = G.maxBY - 16;
    q.nIni = G.nIni; q.hX = G.hX; q.N = G.quota;
    q.wCell = G.wCell; q.hCell = G.hCell; q.nCols = G.nCols;
#if defined(QT_PROFILE)
    q.prof_base = l == 0 ? 0 : 16;
#endif
    int npow = 2;
    while (npow < n) npow <<= 1;
    const uint32_t* src = cand + (int64_t)img * g.candTotal + G.candOff;
    uint32_t* out = lvlKp + (int64_t)img * g.kpTotal + G.kpOff;
    int cap = qt_node_cap(G.quota);
    if (cap > nodeCapMax) cap = nodeCapMax;
    uint32_t* garr = sortScratch + (int64_t)img * g.sortTotal + G.sortOff;
    void* gws = nodeScratch + ((int64_t)l * batch + img) * nodeScratchStride;
    int S;
    if (npow <= sortCapSmem) {
        uint32_t* sarr = reinterpret_cast<uint32_t*>(qt_smem);
        if (nodesInSmem) S = qt_run(sarr, qt_smem + (size_t)sortCapSmem * 4, cap, n, npow, src, q, out);
        else S = qt_run(sarr, gws, cap, n, npow, src, q, out);
    } else {
        if (nodesInSmem) S = qt_run(garr, qt_smem + (size_t)sortCapSmem * 4, cap, n, npow, src, q, out);
        else S = qt_run(garr, gws, cap, n, npow, src, q, out);
    }
    if (threadIdx.x == 0) {
        if (S < 0 || S > G.kpCap) {
            atomicExch(&err[1], 1);
            S = 0;
        }
        lvlCnt[img * g.nlevels + l] = S;
    }
}

// K3 variant 1: the candidate sort takes up to three butterfly stages per pass, and the ordered phase's std::sort is spread over the CTA
// instead of run by thread 0 (both in quadtree_sort_par.cuh).  A separate
// kernel so that k_quadtree -- green on the GPU tier -- keeps its machine code bit for bit (scripts/sass_fingerprint.py);
// selected with ORB_QT_VARIANT=1 at orbx_create until it has had its own device run.
__device__ __forceinline__ int qt_run_v1(uint32_t* arr, void* ws, int cap, int n, int npow, const uint32_t* __restrict__ src,
                                         const QtGeom& q, uint32_t* out) {
    QT_PROF_BEGIN();
    if (npow < 256) npow = 256;     // qt_bitonic_sort_w sorts whole 256-element warp blocks (every sort buffer holds >= 2048 elements)
    for (int i = threadIdx.x; i < npow; i += blockDim.x) arr[i] = (i < n) ? qt_element(src[i], q) : 0xffffffffu;
    __syncthreads();
    QT_TICK(q, 0)
    qt_bitonic_sort_w(arr, npow);
    QT_TICK(q, 1)
    QtWork w;
    qt_work_carve(w, ws, cap);
    return qt_distribute_v<1>(arr, n, q, w, out);
}

// MAXT = 256 (four CTAs per SM) for the small levels; MAXT = 1024 for the group that holds level 0, whose 128-per-batch CTAs each sort
// 4-8 k candidates: one CTA per SM either way, so four times the threads shorten the longest kernel of the stage.  The body only uses
// blockDim.x (QT_PAR_FOR, qt_exscan), never QT_THREADS.
template <int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) k_quadtree_v1(const __grid_constant__ ExtractGeom g, int batch, int levelBegin,
                                                           const uint32_t* __restrict__ cand, const int* __restrict__ candCnt,
                                                           uint32_t* __restrict__ sortScratch, char* __restrict__ nodeScratch,
                                                           int64_t nodeScratchStride, int sortCapSmem, int nodesInSmem,
                                                           int nodeCapMax, uint32_t* __restrict__ lvlKp, int* __restrict__ lvlCnt,
                                                           int* __restrict__ err) {
    extern __shared__ __align__(16) unsigned char qt_smem[];
    const int l = levelBegin + blockIdx.x / batch, img = blockIdx.x % batch;
    const LevelGeom& G = g.lv[l];
    int n = candCnt[img * g.nlevels + l];
    if (n > G.candCap) n = G.candCap;
    QtGeom q;
    q.regionW = G.maxBX - 16; q.regionH = G.maxBY - 16;
    q.nIni = G.nIni; q.hX = G.hX; q.N = G.quota;
    q.wCell = G.wCell; q.hCell = G.hCell; q.nCols = G.nCols;
#if defined(QT_PROFILE)
    q.prof_base = l == 0 ? 0 : 16;
#endif
    int npow = 2;
    while (npow < n) npow <<= 1;
    const uint32_t* src = cand + (int64_t)img * g.candTotal + G.candOff;
    uint32_t* out = lvlKp + (int64_t)img * g.kpTotal + G.kpOff;
    int cap = qt_node_cap(G.quota);
    if (cap > nodeCapMax) cap = nodeCapMax;
    uint32_t* garr = sortScratch + (int64_t)img * g.sortTotal + G.sortOff;
    void* gws = nodeScratch + ((int64_t)l * batch + img) * nodeScratchStride;
    int S;
    if (npow <= sortCapSmem) {
        uint32_t* sarr = reinterpret_cast<uint32_t*>(qt_smem);
        if (nodesInSmem) S = qt_run_v1(sarr, qt_smem + (size_t)sortCapSmem * 4, cap, n, npow, src, q, out);
        else S = qt_run_v1(sarr, gws, cap, n, npow, src, q, out);
    } else {
        if (nodesInSmem) S = qt_run_v1(garr, qt_smem + (size_t)sortCapSmem * 4, cap, n, npow, src, q, out);
        else S = qt_run_v1(garr, gws, cap, n, npow, src, q, out);
    }
    if (threadIdx.x == 0) {
        if (S < 0 || S > G.kpCap) {
            atomicExch(&err[1], 1);
            S = 0;
        }
        lvlCnt[img * g.nlevels + l] = S;
    }
}

// ---------------------------------------------------------------------------------------------
// K3b  output slot of every keypoint (ORBextractor.cc:1656-1678): emission order is level-major;
// keypoints whose scaled x lies in [lap0, lap1] fill the output from the back, the others from the
// front.  One CTA per image.  Also per-image totals.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_order(const __grid_constant__ ExtractGeom g, const uint32_t* __restrict__ lvlKp,
                                              const int* __restrict__ lvlCnt, int lap0, int lap1,
                                              int* __restrict__ slot, int* __restrict__ nkp, int* __restrict__ mono) {
    extern __shared__ int ord_flags[];  // kpTotal ints + 40
    __shared__ int s_off[ORB_MAX_LEVELS + 1];
    const int img = blockIdx.x;
    if (threadIdx.x == 0) {
        int run = 0;
        for (int l = 0; l < g.nlevels; ++l) {
            s_off[l] = run;
            run += lvlCnt[img * g.nlevels + l];
        }
        s_off[g.nlevels] = run;
    }
    __syncthreads();
    const int total = s_off[g.nlevels];
    const uint32_t* kp = lvlKp + (int64_t)img * g.kpTotal;
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
        int l = 0;
        while (e >= s_off[l + 1]) ++l;
        const uint32_t c = kp[g.lv[l].kpOff + (e - s_off[l])];
        float x = (float)((int)(c & 0xfffu) + 16);
        if (l != 0) x = fmul(x, g.lv[l].scale);
        const bool lapping = (x >= (float)lap0) && (x <= (float)lap1);
        ord_flags[e] = lapping ? 0 : 1;
    }
    __syncthreads();
    int* tmp = ord_flags + g.kpTotal;
    // keep the raw flag: after the scan flag[e] = (scan[e+1] - scan[e])
    const int nmono = qt_exscan(ord_flags, total, tmp);
    for (int e = threadIdx.x; e < total; e += blockDim.x) {
        const int before = ord_flags[e];
        const int nxt = (e + 1 < total) ? ord_flags[e + 1] : nmono;
        const bool is_mono = nxt != before;
        slot[(int64_t)img * g.kpTotal + e] = is_mono ? before : (total - 1 - (e - before));
    }
    if (threadIdx.x == 0) {
        nkp[img] = total;
        mono[img] = nmono;
    }
}

// exclusive scan of the per-image keypoint counts -> first compact output row of every image
__global__ void k_offsets(const int* __restrict__ nkp, int batch, int* __restrict__ offsets) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        int run = 0;
        for (int b = 0; b < batch; ++b) {
            offsets[b] = run;
            run += nkp[b];
        }
        offsets[batch] = run;
    }
}

// ---------------------------------------------------------------------------------------------
// K5  GaussianBlur 7x7 sigma=2 BORDER_REFLECT_101, OpenCV's fixed-point path (SURVEY App. A.2;
// ORBextractor.cc:1629-1637): Q0.8 kernel {18,34,48,56,48,34,18}, horizontal pass Q8.8 (u16), vertical pass
// Q16.16, (acc + 32768) >> 16.
// No shared memory: a thread owns 4 adjacent columns and marches down BLUR_ROWS rows with the last 7 horizontal
// results in registers.  The horizontal pass runs on packed u16x2 lanes: with pixel sums <= 510 and an
// accumulator <= 65280 a plain 32-bit IMAD multiplies both lanes at once without a carry between them.
// ---------------------------------------------------------------------------------------------
#define BLUR_TW 128     // columns per CTA (32 threads x 4 px)
#define BLUR_TH 256     // rows per CTA (8 thread rows x BLUR_ROWS); idle thread rows exit at once
#define BLUR_ROWS 32

__device__ __forceinline__ int reflect101(int i, int n) {
    if (i < 0) i = -i;
    if (i >= n) i = 2 * n - 2 - i;
    return i;  // valid for n >= 4 and |overshoot| <= 3 (every pyramid level is far larger)
}

// horizontal 7-tap of 4 adjacent pixels at columns x0..x0+3 of row `p`; returns packed Q8.8 results:
// lo = (px0 | px2 << 16), hi = (px1 | px3 << 16)
// mode 0: interior (three aligned word loads); mode 1: left edge, x0 == 0 (columns -3 .. -1 reflect to 3 .. 1: one PRMT of the first
// word); mode 2: right edge: ten byte loads, window column x0 - 3 + k read at itself while k < kr and at its mirror image
// 2w - 2 - column from there on (BORDER_REFLECT_101; columns past w + 2 only feed the pitch padding).  With the reflect
// arithmetic inside the row loop the edge path was a large share of k_blur's instructions -- a warp that holds one edge lane runs it for
// every row.
template <bool DP4A>
__device__ __forceinline__ void blur_h4(const uint8_t* __restrict__ p, int x0, int mode, int kr, int colA, int colB, uint32_t* __restrict__ h) {
    uint32_t w0, w1, w2;   // bytes x0-4 .. x0+7
    if (mode == 0) {
        const uint32_t* q = reinterpret_cast<const uint32_t*>(p + x0 - 4);
        w0 = __ldg(q); w1 = __ldg(q + 1); w2 = __ldg(q + 2);
    } else if (mode == 1) {
        const uint32_t* q = reinterpret_cast<const uint32_t*>(p);
        w1 = __ldg(q); w2 = __ldg(q + 1);
        w0 = __byte_perm(w1, 0u, 0x1230);
    } else {
        uint32_t b[10];
#pragma unroll
        for (int k = 0; k < 10; ++k) b[k] = (uint32_t)__ldg(p + (k < kr ? colA + k : colB - k));
        w0 = (b[0] << 8) | (b[1] << 16) | (b[2] << 24);
        w1 = b[3] | (b[4] << 8) | (b[5] << 16) | (b[6] << 24);
        w2 = b[7] | (b[8] << 8) | (b[9] << 16);
    }
    if constexpr (DP4A) {   // pixel i = bytes 1+i .. 7+i of the window: two 4-byte dot products with the Q8 kernel (IDP.4A.U8.U8)
        const uint32_t cA = 18u | (34u << 8) | (48u << 16) | (56u << 24), cB = 48u | (34u << 8) | (18u << 16);
        h[0] = __dp4a(__byte_perm(w0, w1, 0x4321), cA, __dp4a(__byte_perm(w1, w2, 0x4321), cB, 0u));
        h[1] = __dp4a(__byte_perm(w0, w1, 0x5432), cA, __dp4a(__byte_perm(w1, w2, 0x5432), cB, 0u));
        h[2] = __dp4a(__byte_perm(w0, w1, 0x6543), cA, __dp4a(__byte_perm(w1, w2, 0x6543), cB, 0u));
        h[3] = __dp4a(w1, cA, __dp4a(w2, cB, 0u));
    } else {
    // S_k = the 4 pixels shifted by k-3 (bytes 1+k .. 4+k of the 12-byte window), split into even / odd lanes
    uint32_t e[7], o[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
        const int off = 1 + k;   // first byte of S_k inside (w0,w1,w2)
        uint32_t sk;
        if (off < 4) sk = __byte_perm(w0, w1, 0x3210 + 0x1111 * off);
        else if (off == 4) sk = w1;
        else sk = __byte_perm(w1, w2, 0x3210 + 0x1111 * (off - 4));
        e[k] = __byte_perm(sk, 0u, 0x4240);
        o[k] = __byte_perm(sk, 0u, 0x4341);
    }
    const uint32_t lo = 18u * (e[0] + e[6]) + 34u * (e[1] + e[5]) + 48u * (e[2] + e[4]) + 56u * e[3];   // px 0 | px 2 << 16, each <= 65280
    const uint32_t hi = 18u * (o[0] + o[6]) + 34u * (o[1] + o[5]) + 48u * (o[2] + o[4]) + 56u * o[3];   // px 1 | px 3 << 16
    h[0] = lo & 0xffffu; h[2] = lo >> 16; h[1] = hi & 0xffffu; h[3] = hi >> 16;
    }
}

template <bool DP4A>
__global__ void __launch_bounds__(256, 4) k_blur(const __grid_constant__ ExtractGeom g) {
    const int tileId = blockIdx.x, img = blockIdx.y;
    int l = 0;
    while (l + 1 < g.nlevels && tileId >= g.lv[l + 1].tileBase) ++l;
    const LevelGeom& G = g.lv[l];
    const int local = tileId - G.tileBase;
    const int ty = local / G.tilesX, tx = local - ty * G.tilesX;
    const int x0 = tx * BLUR_TW + 4 * (threadIdx.x & 31);
    const int y0 = ty * BLUR_TH + BLUR_ROWS * (threadIdx.x >> 5);
    if (x0 >= G.w || y0 >= G.h) return;
    const uint8_t* __restrict__ src = G.base + (int64_t)img * G.img_stride;
    uint8_t* __restrict__ dst = G.blur + (int64_t)img * G.blur_stride;
    const int mode = (x0 + 8 <= G.w) ? (x0 >= 4 ? 0 : 1) : 2;
    const int colA = x0 - 3, kr = G.w - colA, colB = 2 * G.w - 2 - colA;   // mode 2: window column colA + k, mirrored from k == kr on
    // horizontal results of the last 7 rows, unpacked to one 32-bit value per pixel (Q8.8 <= 65280).  (Measured and dropped: the vertical
    // pass by IDP.2A on (h[r-1] | h[r] << 16) pairs -- 5 instead of 10 instructions per pixel by count, 0.295 instead of 0.264 ms.)
    uint32_t hwin[7][4];
    const int rows = min(BLUR_ROWS, G.h - y0);
    // 7 rows per trip: the window slot r % 7 == j is then a compile-time register index, and the body (1/5 of the fully
    // unrolled form) stays resident in the instruction cache -- the 38-row unroll was 124 KB of code and stalled on fetch
    for (int rb = 0; rb < BLUR_ROWS + 6; rb += 7) {
#pragma unroll
        for (int j = 0; j < 7; ++j) {
            const int r = rb + j;
            if (r < rows + 6) {
                const int y = reflect101(y0 + r - 3, G.h);
                blur_h4<DP4A>(src + (int64_t)y * G.pitch, x0, mode, kr, colA, colB, hwin[j]);
                if (r >= 6) {
                    // rows r-6 .. r are in the window; output row y0 + r - 6
                    uint32_t packed = 0u;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const uint32_t acc = 18u * (hwin[(j + 1) % 7][k] + hwin[j][k]) + 34u * (hwin[(j + 2) % 7][k] + hwin[(j + 6) % 7][k]) +
                                             48u * (hwin[(j + 3) % 7][k] + hwin[(j + 5) % 7][k]) + 56u * hwin[(j + 4) % 7][k];
                        packed |= ((acc + 32768u) >> 16) << (8 * k);
                    }
                    *reinterpret_cast<uint32_t*>(dst + (int64_t)(y0 + r - 6) * G.blur_pitch + x0) = packed;   // pitch padding absorbs the tail
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// K4+K6  IC_Angle (ORBextractor.cc:91-138) + computeOrbDescriptor (:150-203), one warp per keypoint.
// Writes the final cv::KeyPoint record and the 32 descriptor bytes at the compact output row.
// ---------------------------------------------------------------------------------------------
#define OD_WARPS 8

__global__ void __launch_bounds__(OD_WARPS * 32) k_orient_describe(const __grid_constant__ ExtractGeom g, const uint32_t* __restrict__ lvlKp,
                                                                  const int* __restrict__ lvlCnt, const int* __restrict__ slot,
                                                                  const int* __restrict__ offsets, const uint32_t* __restrict__ patT,
                                                                  orbx_keypoint* __restrict__ kps, uint8_t* __restrict__ desc) {
    // patT: the 256 point pairs as one 32-bit word each (xa, ya, xb, yb as int8), transposed so that lane's k-th pair sits at
    // [k][lane] -- built once per handle in global memory.  (Round 1 staged it per CTA from __constant__ memory: 32 different constant
    // addresses per load serialise, and the staging + barrier were a large share of the kernel's stall samples.)
    const int img = blockIdx.y;
    const int lane = threadIdx.x & 31;
    const int e = blockIdx.x * OD_WARPS + (threadIdx.x >> 5);
    int l = 0, first = 0;
    {   // level of emission index e: lanes 0 .. nlevels-1 hold the level counts, a shuffle scan gives the running totals
        const int c = lane < g.nlevels ? lvlCnt[img * g.nlevels + lane] : 0;
        int incl = c;
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) {
            const int v = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += v;
        }
        const unsigned m = __ballot_sync(0xffffffffu, lane < g.nlevels && e < incl);
        if (m == 0u) return;  // warp-uniform
        l = __ffs(m) - 1;
        first = __shfl_sync(0xffffffffu, incl - c, l);
    }
    const LevelGeom& G = g.lv[l];
    const uint32_t c = lvlKp[(int64_t)img * g.kpTotal + G.kpOff + (e - first)];
    const int x = (int)(c & 0xfffu) + 16, y = (int)((c >> 12) & 0xfffu) + 16, score = (int)(c >> 24);

    // intensity centroid over the radius-15 disc: lane u+15 owns COLUMN u and walks the 31 rows, so every load
    // instruction of the warp touches one 31-byte segment (one cache line) and the 31 loads are independent.
    // (Measured and dropped: lane = row with nine word loads and IDP.4A against weight tables -- 30 % fewer instructions for the
    // kernel, but every load instruction then touches 31 cache lines: 0.225 instead of 0.184 ms.)
    int m10 = 0, m01 = 0;
    if (lane < 31) {
        constexpr int um[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};   // == c_umax, as immediates
        const int u = lane - 15, au = u < 0 ? -u : u;
        const uint8_t* q = G.base + (int64_t)img * G.img_stride + (int64_t)(y - 15) * G.pitch + x + u;
        const int64_t pitch = G.pitch;
        int cs = 0;
#pragma unroll
        for (int v = -15; v <= 15; ++v) {
            const int val = (au <= um[v < 0 ? -v : v]) ? (int)__ldg(q) : 0;
            q += pitch;
            cs += val;
            m01 += v * val;
        }
        m10 = u * cs;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        m10 += __shfl_xor_sync(0xffffffffu, m10, o);
        m01 += __shfl_xor_sync(0xffffffffu, m01, o);
    }
    const float angle = fast_atan2_deg((float)m01, (float)m10);

    // steered BRIEF: lane = descriptor byte
    const float factorPI = (float)(3.14159265358979323846 / 180.f);
    float sa, ca;
    glibc_sincosf(fmul(angle, factorPI), &sa, &ca);
    const uint8_t* cb = G.blur + (int64_t)img * G.blur_stride + (int64_t)y * G.blur_pitch + x;
    uint32_t val = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const uint32_t pw = __ldg(patT + 32 * k + lane);
        const float xa = (float)(int8_t)(pw & 0xffu), ya = (float)(int8_t)((pw >> 8) & 0xffu), xb = (float)(int8_t)((pw >> 16) & 0xffu),
                    yb = (float)(int8_t)(pw >> 24);
        const int ra = round_half_even(fadd(fmul(xa, sa), fmul(ya, ca))), ca_ = round_half_even(fsub(fmul(xa, ca), fmul(ya, sa)));
        const int rb = round_half_even(fadd(fmul(xb, sa), fmul(yb, ca))), cb_ = round_half_even(fsub(fmul(xb, ca), fmul(yb, sa)));
        const int t0 = __ldg(cb + (int64_t)ra * G.blur_pitch + ca_);
        const int t1 = __ldg(cb + (int64_t)rb * G.blur_pitch + cb_);
        val |= (uint32_t)(t0 < t1) << k;
    }
    const int row = offsets[img] + slot[(int64_t)img * g.kpTotal + e];
    // gather 4 descriptor bytes per word; lanes 0..7 store
    uint32_t w = val & 0xffu;
    w |= (__shfl_down_sync(0xffffffffu, val, 1) & 0xffu) << 8;
    w |= (__shfl_down_sync(0xffffffffu, val, 2) & 0xffu) << 16;
    w |= (__shfl_down_sync(0xffffffffu, val, 3) & 0xffu) << 24;
    const uint32_t w4 = __shfl_sync(0xffffffffu, w, (lane & 7) * 4);
    if (lane < 8) reinterpret_cast<uint32_t*>(desc + (int64_t)row * 32)[lane] = w4;
    if (lane == 8) {
        orbx_keypoint kp;
        float fx = (float)x, fy = (float)y;
        if (l != 0) {
            fx = fmul(fx, G.scale);
            fy = fmul(fy, G.scale);
        }
        kp.x = fx; kp.y = fy; kp.size = G.patch; kp.angle = angle; kp.response = (float)score;
        kp.octave = l; kp.class_id = -1;
        kps[row] = kp;
    }
}

}  // namespace orb

#include "fast_cells_v2.cuh"
