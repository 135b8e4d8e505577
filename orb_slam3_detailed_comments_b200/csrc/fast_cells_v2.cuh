// fast_cells_v2.cuh -- K2, second formulation of the per-cell FAST-9/16 + NMS + 20->7 fallback
// (ORBextractor.cc:1069-1166; cv::FAST(cell, thr, nms = true) per 35-px cell, SURVEY App. A.3).
//
// Same result as k_fast_cells (the candidate list of a level is order-free: the quadtree re-derives the reference order from the
// coordinates), about half the instructions.  What changed, each from an ncu source page of k_fast_cells:
//   * the cell geometry comes from a host-built table (one 8-byte record per NON-EMPTY cell) instead of a per-CTA level search,
//     two integer divisions and the bounds logic;
//   * the window is staged 8 pixels per step (one 64-bit load, two 128-bit shared stores) into rows sized from the geometry
//     (28 pixel pairs at 640x480 instead of a fixed 46), so a CTA needs ~14 KB instead of ~30 KB of shared memory;
//   * the pixel pairs that pass the high-speed test are compacted into a list (ballot + popc into one segment per warp: no
//     atomics), the scored pairs with a non-zero score into a second one, and the non-maximum suppression visits only those
//     (a byte score map; the round-1 kernel ran the NMS over every pixel); the score itself works on the raw ring values
//     (max over the arcs of the arc minimum, centre subtracted once: 16 fewer instructions per pair);
//   * the row stride of the staging arrays is a template parameter for the usual geometry (35-37 px cells: 28 pairs), so every
//     ring offset is an immediate of its shared-memory load;
//   * survivors are appended straight to the level's candidate list with one warp-aggregated global atomic per 32 list entries:
//     the round-1 count pass, CTA scan and second pass over the tile are gone, and so are two of the six CTA barriers.
// A cell empty at iniThFAST is run again at minThFAST; the score map needs no clearing in between (a pixel's score does not
// depend on the threshold; every score >= iniThFAST is written again with the same value).
#pragma once

namespace orb {

struct FastPlan {
    const uint2* cells;   // x: x0 | y0 << 12 | level << 24 (window origin, level coordinates); y: cw | ch << 8 (window size)
    int nCells;
    int R;                // staged rows   (max window height)
    int PW;               // row stride of the staging arrays in 16x2 pixel pairs: ODD (lanes of a warp work on consecutive ROWS)
    int LW;               // entries per pair list
};

#define FAST2_THREADS 128

// TMA (1-D bulk copy) staging of the window: ORB_FAST_TMA=1.  A window row is one 64-byte, 16-byte aligned span of the level image
// (the staged columns start at gx0 & ~15 and end before gx0 + 64 for 35-37 px cells), so thread r arms nothing and issues ONE
// cp.async.bulk for row r; thread 0 arms the mbarrier with the byte count of the whole window.  The raw bytes land in shared
// memory and are expanded to the 16x2 pairs from there.  SASS: UBLKCP.S.G, SYNCS.ARRIVE.TRANS64, SYNCS.PHASECHK.TRANS64.TRYWAIT.
__device__ __forceinline__ uint32_t fast_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fast_mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(fast_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fast_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(fast_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void fast_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(fast_smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(fast_smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void fast_mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "FAST_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra FAST_DONE;\n"
        "bra FAST_WAIT;\n"
        "FAST_DONE:\n"
        "}\n" ::"r"(fast_smem_u32(bar)),
        "r"(parity)
        : "memory");
}

// PWC > 0: the row stride is a compile-time constant (every ring offset becomes an immediate of the shared-memory load);
// PWC == 0: taken from the plan at run time (any geometry).
template <int PWC, bool TMA = false>
__global__ void __launch_bounds__(FAST2_THREADS, 8)
k_fast_cells_v2(const __grid_constant__ ExtractGeom g, const __grid_constant__ FastPlan fp, uint32_t* __restrict__ cand,
                int* __restrict__ candCnt, int* __restrict__ err) {
    extern __shared__ __align__(16) uint32_t fast2_smem[];
    // Bank layout: a warp's 32 lanes work on 32 consecutive ROWS of one column of 4-pixel groups, and every row stride (PW words
    // for pe / po, WS words for the score map) is odd, so each shared-memory load of the high-speed test touches 32 different banks
    // (the round-2 first cut, lanes along a row with an even stride, spent half of its shared-memory wavefronts on bank conflicts).
    const int R = fp.R, PW = PWC > 0 ? PWC : fp.PW, WS = ((PW - 1) >> 1) | 1, SBW = 4 * WS, RP = (R * PW + 3) & ~3;
    uint32_t* pe = fast2_smem;                       // pe[r][i] = (px 2i, px 2i+1) as 16x2
    uint32_t* po = pe + RP;                          // po[r][i] = (px 2i+1, px 2i+2)
    uint8_t* sb = reinterpret_cast<uint8_t*>(po + RP);       // score (>= T, else 0) per staged pixel, one byte each
    const int sbBytes = (R * SBW + 15) & ~15;
    // pair lists (r * 64 + pair index), one segment of LW entries per warp so that appending needs no atomics (ptxas wraps every
    // one-lane shared-memory atomic into a ~15-instruction warp-aggregation sequence of its own); readers walk the four segments
    // back to back.  lst1: pairs that pass the high-speed test; lst2: pairs whose score reaches the threshold.
    uint16_t* lst1 = reinterpret_cast<uint16_t*>(sb + sbBytes);
    uint16_t* lst2 = lst1 + 4 * fp.LW;
    uint16_t* const my1 = lst1 + (threadIdx.x >> 5) * fp.LW;   // this warp's segments
    uint16_t* const my2 = lst2 + (threadIdx.x >> 5) * fp.LW;
    __shared__ __align__(16) int s_c1[4], s_c2[4];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, img = blockIdx.y;
    const int LW = fp.LW;

    const uint2 cr = fp.cells[blockIdx.x];
    const int x0 = cr.x & 0xfff, y0 = (cr.x >> 12) & 0xfff, l = cr.x >> 24, cw = cr.y & 0xff, ch = (cr.y >> 8) & 0xff;
    const LevelGeom& G = g.lv[l];
    const int tx0 = x0 + 3, tx1 = x0 + cw - 3, ty0 = y0 + 3, ty1 = y0 + ch - 3;
    const int gx0 = (((tx0 & ~3) - 4) & ~7);                 // staged column 0 (8-byte aligned in the level image)
    const int wd0 = ((tx0 & ~3) - gx0) >> 2;                 // 4-pixel word of the first tested group: 1 or 2
    const int ngrp = ((tx1 - 1) >> 2) - (tx0 >> 2) + 1;
    const int nC8 = (wd0 + ngrp + 2) >> 1;                   // 8-byte chunks per staged row (one margin word on the right)
    const uint8_t* src = G.base + (int64_t)img * G.img_stride + (int64_t)y0 * G.pitch + gx0;

    if (TMA) {   // the window's rows by bulk copies into a raw byte tile, then expanded from shared memory
        __shared__ __align__(8) uint64_t s_bar;
        uint8_t* raw = reinterpret_cast<uint8_t*>(lst2 + 4 * fp.LW);      // R rows of 64 bytes, 16-byte aligned
        const int gx16 = gx0 & ~15, shift = gx0 - gx16;                   // gx0 is 8-byte aligned: shift is 0 or 8
        const uint32_t rowBytes = (uint32_t)min(64, G.pitch - gx16);      // a multiple of 16; the last cells of a row stop at the pitch
        if (tid == 0) {
            fast_mbar_init(&s_bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();
        if (tid == 0) fast_mbar_expect_tx(&s_bar, (uint32_t)ch * rowBytes);
        if (tid < ch) fast_bulk_g2s(raw + 64 * tid, src - shift + (int64_t)tid * G.pitch, rowBytes, &s_bar);
        for (int i = tid; i < (sbBytes >> 4); i += FAST2_THREADS) reinterpret_cast<uint4*>(sb)[i] = make_uint4(0u, 0u, 0u, 0u);
        fast_mbar_wait(&s_bar, 0u);
        const uint32_t magicC = (1u << 20) / (uint32_t)nC8 + 1u;
        const int total = ch * nC8;
        for (int i = tid; i < total; i += FAST2_THREADS) {
            const int r = (int)(((uint32_t)i * magicC) >> 20), c = i - r * nC8;
            const uint8_t* rp = raw + 64 * r + shift + 8 * c;
            const uint2 w = *reinterpret_cast<const uint2*>(rp);
            const uint32_t nx = (c + 1 < nC8) ? *reinterpret_cast<const uint32_t*>(rp + 8) : 0u;
            uint32_t* de = pe + r * PW + 4 * c;
            uint32_t* dp = de + RP;
            de[0] = __byte_perm(w.x, 0u, 0x4140); de[1] = __byte_perm(w.x, 0u, 0x4342);
            de[2] = __byte_perm(w.y, 0u, 0x4140); de[3] = __byte_perm(w.y, 0u, 0x4342);
            dp[0] = __byte_perm(w.x, 0u, 0x4241); dp[1] = __byte_perm(w.x, w.y, 0x4433) & 0x00ff00ffu;
            dp[2] = __byte_perm(w.y, 0u, 0x4241); dp[3] = __byte_perm(w.y, nx, 0x4433) & 0x00ff00ffu;
        }
    } else
    {   // staging, three rows of loads in flight per thread (a cell is 2.4 rounds of 128 eight-pixel chunks at 640x480)
        const uint32_t magicC = (1u << 20) / (uint32_t)nC8 + 1u;   // (i * magic) >> 20 == i / n exactly for i < 2048, n <= 32
        const int total = ch * nC8;
        for (int base = tid; base < total; base += 3 * FAST2_THREADS) {
            uint2 w[3];
            uint32_t nx[3];
            int off[3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int i = base + k * FAST2_THREADS;
                off[k] = -1;
                if (i < total) {
                    const int r = (int)(((uint32_t)i * magicC) >> 20), c = i - r * nC8;
                    const uint2* rowp = reinterpret_cast<const uint2*>(src + (int64_t)r * G.pitch);
                    w[k] = __ldg(rowp + c);
                    nx[k] = (c + 1 < nC8) ? __ldg(reinterpret_cast<const uint32_t*>(rowp + c + 1)) : 0u;
                    off[k] = r * PW + 4 * c;
                }
            }
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (off[k] >= 0) {
                    uint32_t* de = pe + off[k];
                    uint32_t* dp = de + RP;
                    de[0] = __byte_perm(w[k].x, 0u, 0x4140); de[1] = __byte_perm(w[k].x, 0u, 0x4342);
                    de[2] = __byte_perm(w[k].y, 0u, 0x4140); de[3] = __byte_perm(w[k].y, 0u, 0x4342);
                    dp[0] = __byte_perm(w[k].x, 0u, 0x4241); dp[1] = __byte_perm(w[k].x, w[k].y, 0x4433) & 0x00ff00ffu;
                    dp[2] = __byte_perm(w[k].y, 0u, 0x4241); dp[3] = __byte_perm(w[k].y, nx[k], 0x4433) & 0x00ff00ffu;
                }
            }
        }
        for (int i = tid; i < (sbBytes >> 4); i += FAST2_THREADS) reinterpret_cast<uint4*>(sb)[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    __syncthreads();

    const int ntask = (ty1 - ty0) * ngrp;          // one task = 4 adjacent pixels = two 16x2 pairs
    const int ntaskW = (ntask + 31) & ~31;         // warp-uniform trip count (ballots inside)
    const int nrow = ty1 - ty0;
    const uint32_t magicR = (1u << 20) / (uint32_t)nrow + 1u;   // (t * magic) >> 20 == t / nrow exactly while t * nrow < 2^20
    const unsigned lt = (1u << lane) - 1u;
    uint32_t* out = cand + (int64_t)img * g.candTotal + G.candOff;
    int* cnt = candCnt + img * g.nlevels + l;

    for (int pass = 0; pass < 2; ++pass) {
        const int thr = pass ? g.minTh : g.iniTh;
        const uint32_t T2p1 = (uint32_t)(thr + 1) * 0x00010001u;
        // A: cv::FAST's high-speed test on every pixel pair (a 9-arc holds one pixel of each antipodal ring pair); survivors -> lst1
        int wn = 0;   // entries of this warp's segment (warp-uniform)
        for (int t = tid; t < ntaskW; t += FAST2_THREADS) {
            uint32_t pa = 0u, pb = 0u;
            int code = 0;
            if (t < ntask) {
                const int grp = (int)(((uint32_t)t * magicR) >> 20), row = t - grp * nrow;   // column-major: lane -> row
                const int r = row + 3, pA = 2 * (wd0 + grp);
                code = r * 64 + pA;
                const uint32_t* e = pe + r * PW + pA;
                const uint32_t* o = e + RP;
                // antipodal ring pairs (0,8) (2,10) (4,12) (6,14): (dx,dy) = (0,-3)/(0,3) (2,-2)/(-2,2) (3,0)/(-3,0) (2,2)/(-2,-2)
                const uint2 c = make_uint2(e[0], e[1]);
                const uint2 q0 = make_uint2(e[-3 * PW], e[-3 * PW + 1]), q8 = make_uint2(e[3 * PW], e[3 * PW + 1]);
                const uint2 q12 = make_uint2(o[-2], o[-1]);
                const uint32_t *q2 = e - 2 * PW + 1, *q10 = e + 2 * PW - 1, *q4 = o + 1, *q6 = e + 2 * PW + 1, *q14 = e - 2 * PW - 1;
                const uint32_t hiA = min_u16x2(min3_u16x2(max_u16x2(q0.x, q8.x), max_u16x2(q2[0], q10[0]), max_u16x2(q4[0], q12.x)),
                                               max_u16x2(q6[0], q14[0]));
                const uint32_t loA = max_u16x2(max3_u16x2(min_u16x2(q0.x, q8.x), min_u16x2(q2[0], q10[0]), min_u16x2(q4[0], q12.x)),
                                               min_u16x2(q6[0], q14[0]));
                const uint32_t hiB = min_u16x2(min3_u16x2(max_u16x2(q0.y, q8.y), max_u16x2(q2[1], q10[1]), max_u16x2(q4[1], q12.y)),
                                               max_u16x2(q6[1], q14[1]));
                const uint32_t loB = max_u16x2(max3_u16x2(min_u16x2(q0.y, q8.y), min_u16x2(q2[1], q10[1]), min_u16x2(q4[1], q12.y)),
                                               min_u16x2(q6[1], q14[1]));
                pa = fast_pretest_x2(c.x, hiA, loA, T2p1);
                pb = fast_pretest_x2(c.y, hiB, loB, T2p1);
            }
            const unsigned ma = __ballot_sync(0xffffffffu, pa != 0u), mb = __ballot_sync(0xffffffffu, pb != 0u);
            const int na = __popc(ma);
            if (pa) my1[wn + __popc(ma & lt)] = (uint16_t)code;
            if (pb) my1[wn + na + __popc(mb & lt)] = (uint16_t)(code + 1);
            wn += na + __popc(mb);
        }
        if (lane == 0) s_c1[wid] = wn;
        __syncthreads();
        // B: full score of the listed pairs; pairs with a non-zero score go on to lst2
        const int4 c1 = *reinterpret_cast<const int4*>(s_c1);
        const int n1 = c1.x + c1.y + c1.z + c1.w;
        wn = 0;
        for (int i = tid; i < ((n1 + 31) & ~31); i += FAST2_THREADS) {
            uint32_t kk = 0u;
            int code = 0;
            if (i < n1) {
                int j = i, sg = 0;
                if (j >= c1.x) { j -= c1.x; sg = LW; if (j >= c1.y) { j -= c1.y; sg = 2 * LW; if (j >= c1.z) { j -= c1.z; sg = 3 * LW; } } }
                code = lst1[sg + j];
                const int r = code >> 6, p = code & 63;
                const uint32_t* e = pe + r * PW + p;
                const uint32_t* o = e + RP;
                uint32_t ring[16];
                // ring offsets (dx,dy) clockwise from the top: even dx -> pe at p + dx/2, odd dx -> po at p + (dx-1)/2
                ring[0] = e[-3 * PW];      ring[1] = o[-3 * PW];      ring[2] = e[-2 * PW + 1];  ring[3] = o[-PW + 1];
                ring[4] = o[1];            ring[5] = o[PW + 1];       ring[6] = e[2 * PW + 1];   ring[7] = o[3 * PW];
                ring[8] = e[3 * PW];       ring[9] = o[3 * PW - 1];   ring[10] = e[2 * PW - 1];  ring[11] = o[PW - 2];
                ring[12] = o[-2];          ring[13] = o[-PW - 2];     ring[14] = e[-2 * PW - 1]; ring[15] = o[-3 * PW - 1];
                const uint32_t s01 = fast_score_raw_x2(e[0], ring);
                const int xb = gx0 + 2 * p;
                const int s0 = (int)(s01 & 0xffffu) - 256, s1 = (int)(s01 >> 16) - 256;
                const uint32_t k0 = (s0 >= thr && xb >= tx0 && xb < tx1) ? (uint32_t)s0 : 0u;
                const uint32_t k1 = (s1 >= thr && xb + 1 >= tx0 && xb + 1 < tx1) ? (uint32_t)s1 : 0u;
                kk = k0 | (k1 << 8);
                if (kk) *reinterpret_cast<uint16_t*>(sb + r * SBW + 2 * p) = (uint16_t)kk;
            }
            const unsigned m = __ballot_sync(0xffffffffu, kk != 0u);
            if (kk) my2[wn + __popc(m & lt)] = (uint16_t)code;
            wn += __popc(m);
        }
        if (lane == 0) s_c2[wid] = wn;
        __syncthreads();   // every score is in the map
        const int4 c2 = *reinterpret_cast<const int4*>(s_c2);
        const int n2 = c2.x + c2.y + c2.z + c2.w;
        // C: 3x3 non-maximum suppression of the listed pairs (strictly greater than all 8 neighbours, cv::FAST), survivors appended
        int has = 0;
        for (int i = tid; i < ((n2 + 31) & ~31); i += FAST2_THREADS) {
            uint32_t s0 = 0u, s1 = 0u;
            int xo = 0, yo = 0;
            if (i < n2) {
                int j = i, sg = 0;
                if (j >= c2.x) { j -= c2.x; sg = LW; if (j >= c2.y) { j -= c2.y; sg = 2 * LW; if (j >= c2.z) { j -= c2.z; sg = 3 * LW; } } }
                const int code = lst2[sg + j], r = code >> 6, p = code & 63;
                const int bm1 = 2 * p - 1;                            // first of the four bytes px 2p-1 .. 2p+2
                const uint32_t sel = 0x3210u + 0x1111u * (uint32_t)(bm1 & 3);
                const uint32_t* wrow = reinterpret_cast<const uint32_t*>(sb + r * SBW) + (bm1 >> 2);
                const uint32_t u = __byte_perm(wrow[-WS], wrow[-WS + 1], sel), m = __byte_perm(wrow[0], wrow[1], sel),
                               d = __byte_perm(wrow[WS], wrow[WS + 1], sel);
                const uint32_t up = max3_u16x2(__byte_perm(u, 0u, 0x4140), __byte_perm(u, 0u, 0x4241), __byte_perm(u, 0u, 0x4342));
                const uint32_t dn = max3_u16x2(__byte_perm(d, 0u, 0x4140), __byte_perm(d, 0u, 0x4241), __byte_perm(d, 0u, 0x4342));
                const uint32_t md = max_u16x2(__byte_perm(m, 0u, 0x4140), __byte_perm(m, 0u, 0x4342));
                const uint32_t c = __byte_perm(m, 0u, 0x4241);
                const uint32_t mx = max3_u16x2(up, dn, md);
                // strictly greater than all 8 neighbours: c >= mx + 1  <=>  max(c, mx + 1) == c   (scores <= 254)
                const uint32_t gt = max_u16x2(c, mx + 0x00010001u) ^ c;
                s0 = (gt & 0xffffu) ? 0u : (c & 0xffffu);
                s1 = (gt >> 16) ? 0u : (c >> 16);
                xo = gx0 + 2 * p - 16;
                yo = y0 + r - 16;
            }
            const unsigned m0 = __ballot_sync(0xffffffffu, s0 != 0u), m1 = __ballot_sync(0xffffffffu, s1 != 0u);
            const int n0 = __popc(m0), n = n0 + __popc(m1);
            if (n) {   // warp-uniform
                has = 1;
                int gb = 0;
                if (lane == 0) gb = atomicAdd(cnt, n);
                gb = __shfl_sync(0xffffffffu, gb, 0);
                if (gb + n > G.candCap) {
                    if (lane == 0) atomicExch(&err[0], 1);
                } else {
                    if (s0) out[gb + __popc(m0 & lt)] = qt_pack_cand(xo, yo, (int)s0);
                    if (s1) out[gb + n0 + __popc(m1 & lt)] = qt_pack_cand(xo + 1, yo, (int)s1);
                }
            }
        }
        // empty at iniThFAST: once more at minThFAST (ORBextractor.cc:1143-1148).  The barrier also orders this pass's reads of the
        // lists and counters before the next pass's writes.
        if (__syncthreads_or(has) || pass == 1) break;
    }
}

}  // namespace orb
