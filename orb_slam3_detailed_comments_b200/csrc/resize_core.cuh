// resize_core.cuh -- one thread of k_resize_v3: 4 destination pixels x ROWS destination rows of the chained cv::resize(INTER_LINEAR)
// fixed-point model (ORBextractor.cc:1687-1738, SURVEY App. A.1), written so that the identical source runs as a device function and
// on the host (tests/host_emul, against the oracle's resize).
//
// k_resize_v2 spends a large share of its instructions and most of its stall samples on the eight byte loads of a source row
// (ncu source page).  Here a source row's bytes x0 .. x0 + 7 (x0 = the first tap of the thread's first pixel) are
// three aligned word loads and two funnel shifts; pixel i's tap pair (p[x0_i], p[x0_i + 1]) is one PRMT with a per-thread selector,
// and c0 * p0 + c1 * p1 is ONE IDP.2A: the 11-bit coefficients are the two 16-bit operands, the pixels the two byte operands.
// The clamped tap x1 = min(x0 + 1, w - 1) differs from x0 + 1 only where the table has c1 = 0, so the product is the same.
// A thread whose three words would end past the source buffer (the last bytes of a caller-owned level 0) takes the byte loads.
#pragma once
#include <cmath>
#include "devmath.cuh"

namespace orbdev {

ORB_HD uint32_t rs_funnel(uint32_t lo, uint32_t hi, uint32_t sh) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
}
ORB_HD uint32_t rs_perm(uint32_t a, uint32_t b, uint32_t sel) {   // result byte k = byte (sel >> 4k) & 7 of the pair (a = bytes 0-3, b = 4-7)
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, sel);
#else
    const uint64_t v = (uint64_t)a | ((uint64_t)b << 32);
    uint32_t r = 0;
    for (int k = 0; k < 4; ++k) r |= (uint32_t)((v >> (8 * ((sel >> (4 * k)) & 7u))) & 0xffu) << (8 * k);
    return r;
#endif
}
ORB_HD uint32_t rs_dp2a_lo(uint32_t a, uint32_t b, uint32_t c) {  // c + a.lo16 * b.byte0 + a.hi16 * b.byte1
#if defined(__CUDA_ARCH__)
    return __dp2a_lo(a, b, c);
#else
    return c + (a & 0xffffu) * (b & 0xffu) + (a >> 16) * ((b >> 8) & 0xffu);
#endif
}

// cv::resize INTER_LINEAR tap table (SURVEY App. A.1): {source index, c0 | c1 << 16} per destination coordinate (host)
inline void rs_linear_taps(int ssize, int dsize, int* out2) {
    const double scale = (double)ssize / dsize;
    for (int d = 0; d < dsize; ++d) {
        float f = (float)((d + 0.5) * scale - 0.5);
        int s = (int)floorf(f);
        f -= (float)s;
        if (s < 0) { s = 0; f = 0.f; }
        if (s >= ssize - 1) { s = ssize - 1; f = 0.f; }
        const int c0 = (int)lrintf((1.f - f) * 2048.f), c1 = (int)lrintf(f * 2048.f);
        out2[2 * d] = s;
        out2[2 * d + 1] = (c0 & 0xffff) | (c1 << 16);
    }
}

struct RsTaps {          // the x taps of the thread's 4 destination pixels
    int x00;             // first source column of pixel 0
    uint32_t sel[4];     // PRMT selector of pixel i's byte pair inside the 8 bytes from x00
    uint32_t cc[4];      // c0 | c1 << 16
    int xo0[4], xo1[4];  // byte-load path: source columns (x1 clamped)
    bool wide;           // the four pairs fit in the 8 bytes from x00
};

// taps: {source index, c0 | c1 << 16} per destination column (host-built, extractor.cu linear_taps)
ORB_HD void rs_load_taps(const int* taps2 /* int2 as pairs */, int dx4, int dw, int sw, RsTaps& T) {
    T.wide = true;
    for (int i = 0; i < 4; ++i) {
        const int d = dx4 + i < dw ? dx4 + i : dw - 1;   // columns past the width feed the pitch padding only
        const int x0 = taps2[2 * d];
        const uint32_t c = (uint32_t)taps2[2 * d + 1];
        if (i == 0) T.x00 = x0;
        const int off = x0 - T.x00;
        T.xo0[i] = x0; T.xo1[i] = x0 + 1 < sw ? x0 + 1 : sw - 1;
        T.cc[i] = c;
        if (off < 0 || off > 6) { T.wide = false; T.sel[i] = 0; }
        else T.sel[i] = (uint32_t)off | ((uint32_t)(off + 1) << 4);
    }
}

// horizontal interpolation of the 4 pixels on one source row, >> 4
ORB_HD void rs_hrow4(const uint8_t* row, const uint8_t* src_end, const RsTaps& T, int h[4]) {
    const uint8_t* p = row + T.x00;
    const uint32_t al = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(p - al);
    if (T.wide && reinterpret_cast<const uint8_t*>(w + 3) <= src_end) {
        const uint32_t w0 = w[0], w1 = w[1], w2 = w[2];
        const uint32_t lo = rs_funnel(w0, w1, 8u * al), hi = rs_funnel(w1, w2, 8u * al);
        for (int i = 0; i < 4; ++i) h[i] = (int)(rs_dp2a_lo(T.cc[i], rs_perm(lo, hi, T.sel[i]), 0u) >> 4);
    } else {
        for (int i = 0; i < 4; ++i)
            h[i] = ((int)row[T.xo0[i]] * (int)(T.cc[i] & 0xffffu) + (int)row[T.xo1[i]] * (int)(T.cc[i] >> 16)) >> 4;
    }
}

// the whole thread: destination pixels dx4 .. dx4 + 3 of rows dy0 .. dy0 + ROWS - 1.  src / dst: the level images of this batch
// item; src_end: one past the last readable byte of the source BUFFER.  Rows share source-row interpolations as in k_resize_v2.
template <int ROWS>
ORB_HD void rs_thread(const uint8_t* src, int sw, int sh, int spitch, const uint8_t* src_end, uint8_t* dst, int dw, int dh, int dpitch,
                      const int* taps2x, const int* taps2y, int dx4, int dy0) {
    RsTaps T;
    rs_load_taps(taps2x, dx4, dw, sw, T);
    int have = -1;
    int hc[4] = {0, 0, 0, 0};
    const int nrow = ROWS < dh - dy0 ? ROWS : dh - dy0;
    for (int k = 0; k < nrow; ++k) {
        const int sy0 = taps2y[2 * (dy0 + k)];
        const uint32_t by = (uint32_t)taps2y[2 * (dy0 + k) + 1];
        const int sy1 = sy0 + 1 < sh ? sy0 + 1 : sh - 1;
        const int b0 = (int)(by & 0xffffu), b1 = (int)(by >> 16);
        int h0[4], h1[4];
        if (sy0 == have) {
            for (int i = 0; i < 4; ++i) h0[i] = hc[i];
        } else {
            rs_hrow4(src + (int64_t)sy0 * spitch, src_end, T, h0);
        }
        if (sy1 == sy0) {
            for (int i = 0; i < 4; ++i) h1[i] = h0[i];
        } else {
            rs_hrow4(src + (int64_t)sy1 * spitch, src_end, T, h1);
        }
        uint32_t packed = 0;
        for (int i = 0; i < 4; ++i) {
            const int v = (((b0 * h0[i]) >> 16) + ((b1 * h1[i]) >> 16) + 2) >> 2;
            packed |= (uint32_t)v << (8 * i);
            hc[i] = h1[i];
        }
        have = sy1;
        if (dx4 + 4 > dw) packed &= 0xffffffffu >> (8 * (dx4 + 4 - dw));   // as k_resize: zero past the width
        *reinterpret_cast<uint32_t*>(dst + (int64_t)(dy0 + k) * dpitch + dx4) = packed;
    }
}

}  // namespace orbdev
