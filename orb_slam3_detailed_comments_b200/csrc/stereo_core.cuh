// stereo_core.cuh -- Frame::ComputeStereoMatches (/root/reference/src/Frame.cc:1102-1358) for ONE left keypoint, written so that the
// identical source runs as a device function (one thread per left keypoint in k_stereo_match_v1) and on the host
// (tests/host_emul, against the oracle).  Differences from k_stereo_match (round 1, one warp per left keypoint scanning ALL
// right keypoints): the right keypoints are bucketed by image row once per CTA (the reference's vRowIndices, Frame.cc:1134-1156,
// reduced to one bucket per keypoint plus a +-window scan), so a left keypoint looks at ~4 % of them; the 11 x 11 SAD over 11
// shifts is done by the same thread.  Arithmetic, gates and tie rule are k_stereo_match's: the best candidate is the minimum of
// (distance << 16 | right index), i.e. "first strictly smaller" in ascending right index whatever the scan order.
#pragma once
#include "devmath.cuh"

namespace orbdev {

struct StLevel {            // raw (unblurred) pyramid level of this stereo pair
    const uint8_t* L;
    const uint8_t* R;
    int pitchL, pitchR, wR;
    float scale, inv_scale;
};

struct StRight {            // right keypoints of this pair, staged (Frame.cc:1134-1156)
    const float* x;         // kpR.pt.x
    const int* band;        // minr (low 16, signed) | maxr << 16
    const signed char* oct;
    const int* row_off;     // [H + 1] bucket b = floor(kpR.pt.y) clamped to [0, H)
    const int* row_ent;     // right indices by bucket (any order inside a bucket)
    int H, W;               // rows, scan half-window: every candidate of row v lies in buckets [v - W, v + W]
};

ORB_HD int st_popc(uint32_t v) {
#if defined(__CUDA_ARCH__)
    return __popc(v);
#else
    return __builtin_popcount(v);
#endif
}

// bytes [sh/8 .. sh/8 + 3] of the 8-byte little-endian pair (lo, hi); sh = 0, 8, 16, 24
ORB_HD uint32_t st_funnel(uint32_t lo, uint32_t hi, uint32_t sh) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_r(lo, hi, sh);
#else
    return sh ? (lo >> sh) | (hi << (32u - sh)) : lo;
#endif
}
// acc + sum of |a_i - b_i| over the four bytes (VABSDIFF4.U8 with accumulate: one instruction on sm_90a)
ORB_HD uint32_t st_sad4(uint32_t a, uint32_t b, uint32_t acc) {
#if defined(__CUDA_ARCH__)
    uint32_t d;
    asm("vabsdiff4.u32.u32.u32.add %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(acc));
    return d;
#else
    for (int i = 0; i < 4; ++i) {
        const int x = (int)((a >> (8 * i)) & 0xffu) - (int)((b >> (8 * i)) & 0xffu);
        acc += (uint32_t)(x < 0 ? -x : x);
    }
    return acc;
#endif
}

ORB_HD int st_row_bucket(float y, int H) {
    int b = (int)floorf(y);
    return b < 0 ? 0 : (b >= H ? H - 1 : b);
}

// half-window in rows that covers minr..maxr of every right keypoint: r = 2 * scale[nlevels - 1], maxr = ceil(y + r), minr = floor(y - r)
ORB_HD int st_scan_window(float maxScale) { return (int)ceilf(fmul(2.0f, maxScale)) + 1; }

ORB_HD void stereo_match_one(float uL, float vL, int octL, const uint32_t* dl /* 8 words */, const StRight& R, const uint8_t* rdesc,
                             const StLevel* lv, float bf, float b, float* out_u, float* out_d, int* out_sad) {
    *out_u = -1.0f; *out_d = -1.0f; *out_sad = -1;
    const float minZ = b, maxD = fdiv(bf, minZ);
    const int vLi = (int)vL;
    const float minU = fsub(uL, maxD), maxU = uL;
    if (maxU < 0) return;
    uint32_t a[8];
    for (int k = 0; k < 8; ++k) a[k] = dl[k];
    uint32_t best = (100u << 16) | 0xffffu;   // TH_HIGH, ORBmatcher.cc:36
    int r0 = vLi - R.W, r1 = vLi + R.W;
    if (r0 < 0) r0 = 0;
    if (r1 > R.H - 1) r1 = R.H - 1;
    for (int n = (r0 <= r1 ? R.row_off[r0] : 0), ne = (r0 <= r1 ? R.row_off[r1 + 1] : 0); n < ne; ++n) {
        const int j = R.row_ent[n];
        const int band = R.band[j];
        const int minr = (int)(short)(band & 0xffff), maxr = band >> 16;
        if (vLi < minr || vLi > maxr) continue;
        const int oc = R.oct[j];
        if (oc < octL - 1 || oc > octL + 1) continue;
        const float uR = R.x[j];
        if (!(uR >= minU && uR <= maxU)) continue;
        const uint32_t* dr = reinterpret_cast<const uint32_t*>(rdesc + (size_t)j * 32);
        uint32_t d = 0;
        for (int k = 0; k < 8; ++k) d += (uint32_t)st_popc(a[k] ^ dr[k]);
        const uint32_t key = (d << 16) | (uint32_t)j;
        if (key < best) best = key;
    }
    const int bestDist = (int)(best >> 16), bestIdxR = (int)(best & 0xffffu);
    if (!(bestDist < 75)) return;             // thOrbDist = (TH_HIGH + TH_LOW) / 2
    const float uR0 = R.x[bestIdxR];
    const StLevel& G = lv[octL];
    const float sf = G.inv_scale;
    const float scaleduL = roundf(fmul(uL, sf)), scaledvL = roundf(fmul(vL, sf)), scaleduR0 = roundf(fmul(uR0, sf));
    const float iniu = scaleduR0, endu = fadd(scaleduR0, 11.0f);   // scaleduR0 + L - w, scaleduR0 + L + w + 1  (w = 5, L = 5)
    if (iniu < 0 || endu >= (float)G.wR) return;
    const int cy = (int)scaledvL, cxL = (int)scaleduL, cxR = (int)scaleduR0;
    // 11 x 11 SAD at 11 shifts, four pixels per instruction: a row of the left patch is three words (11 bytes, the twelfth masked),
    // the 21 bytes of the right row six; the window of shift s is three funnel shifts of those.  (Round 2 until here: 1331 scalar
    // |l - r| per keypoint, 61 % of the kernel's instructions.)  The rows are read as aligned words around the patch: the patch is
    // >= 9 columns inside the level (keypoints keep EDGE_THRESHOLD = 19 px from the border), so the <= 3 extra bytes exist.
    uint32_t dist[11];
    for (int s = 0; s < 11; ++s) dist[s] = 0u;
    for (int row = 0; row < 11; ++row) {
        const int y = cy + row - 5;
        const uint8_t* pl = G.L + (size_t)y * G.pitchL + (cxL - 5);
        const uint8_t* pr = G.R + (size_t)y * G.pitchR + (cxR - 10);
        const uint32_t al = (uint32_t)(reinterpret_cast<uintptr_t>(pl) & 3u), ar = (uint32_t)(reinterpret_cast<uintptr_t>(pr) & 3u);
        const uint32_t* wl = reinterpret_cast<const uint32_t*>(pl - al);
        const uint32_t* wr = reinterpret_cast<const uint32_t*>(pr - ar);
        const uint32_t a0 = wl[0], a1 = wl[1], a2 = wl[2], a3 = wl[3];
        const uint32_t L0 = st_funnel(a0, a1, 8u * al), L1 = st_funnel(a1, a2, 8u * al), L2 = st_funnel(a2, a3, 8u * al) & 0x00ffffffu;
        uint32_t b[7], Rw[6];
#pragma unroll
        for (int k = 0; k < 7; ++k) b[k] = wr[k];
#pragma unroll
        for (int k = 0; k < 6; ++k) Rw[k] = st_funnel(b[k], b[k + 1], 8u * ar);
#pragma unroll
        for (int s = 0; s < 11; ++s) {   // s is a compile-time constant after unrolling: Rw[] stays in registers, the shifts are immediates
            const int q = s >> 2;
            const uint32_t sh = 8u * (uint32_t)(s & 3);
            const uint32_t w0 = st_funnel(Rw[q], Rw[q + 1], sh), w1 = st_funnel(Rw[q + 1], Rw[q + 2], sh),
                           w2 = st_funnel(Rw[q + 2], Rw[q + 3], sh) & 0x00ffffffu;
            dist[s] = st_sad4(L2, w2, st_sad4(L1, w1, st_sad4(L0, w0, dist[s])));
        }
    }
    int bestSad = 0x7fffffff, bestinc = 0;
    for (int s = 0; s < 11; ++s)
        if ((int)dist[s] < bestSad) { bestSad = (int)dist[s]; bestinc = s - 5; }
    if (bestinc == -5 || bestinc == 5) return;
    const float d1 = (float)dist[5 + bestinc - 1], d2 = (float)dist[5 + bestinc], d3 = (float)dist[5 + bestinc + 1];
    const float deltaR = fdiv(fsub(d1, d3), fmul(2.0f, fsub(fadd(d1, d3), fmul(2.0f, d2))));
    if (deltaR < -1 || deltaR > 1) return;
    float bestuR = fmul(G.scale, fadd(fadd(scaleduR0, (float)bestinc), deltaR));
    float disparity = fsub(uL, bestuR);
    if (!(disparity >= 0 && disparity < maxD)) return;
    if (disparity <= 0) {
        disparity = 0.01f;
        bestuR = (float)((double)uL - 0.01);
    }
    *out_d = fdiv(bf, disparity);
    *out_u = bestuR;
    *out_sad = bestSad;
}

}  // namespace orbdev
