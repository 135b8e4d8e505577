// devmath.cuh -- per-element arithmetic of the ORB hot path, written once for the sm_90a kernels.
// Every function is ORB_HD so that tests/host_emul can compile this header with g++ (no GPU in the
// build container) and compare it against the oracle before a kernel ever runs on the GPU.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define ORB_HD __host__ __device__ __forceinline__
#define ORB_D __device__ __forceinline__
#else
#define ORB_HD inline
#define ORB_D inline
#include <cmath>
#include <cstring>
#endif

namespace orbdev {

// ------------------------------------------------------------------------------------------
// packed 16x2 helpers.  On the device these are single DPX instructions (VIMNMX3.U16x2); the host
// versions exist only for the emulation tests.
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
ORB_D uint32_t min3_u16x2(uint32_t a, uint32_t b, uint32_t c) { return __vimin3_u16x2(a, b, c); }
ORB_D uint32_t max3_u16x2(uint32_t a, uint32_t b, uint32_t c) { return __vimax3_u16x2(a, b, c); }
ORB_D uint32_t min_u16x2(uint32_t a, uint32_t b) { return __vminu2(a, b); }
ORB_D uint32_t max_u16x2(uint32_t a, uint32_t b) { return __vmaxu2(a, b); }
ORB_D uint32_t byte_perm(uint32_t a, uint32_t b, uint32_t s) { return __byte_perm(a, b, s); }
#else
inline uint32_t min_u16x2(uint32_t a, uint32_t b) {
    uint32_t lo = ((a & 0xffff) < (b & 0xffff)) ? (a & 0xffff) : (b & 0xffff);
    uint32_t hi = ((a >> 16) < (b >> 16)) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
}
inline uint32_t max_u16x2(uint32_t a, uint32_t b) {
    uint32_t lo = ((a & 0xffff) > (b & 0xffff)) ? (a & 0xffff) : (b & 0xffff);
    uint32_t hi = ((a >> 16) > (b >> 16)) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
}
inline uint32_t min3_u16x2(uint32_t a, uint32_t b, uint32_t c) { return min_u16x2(min_u16x2(a, b), c); }
inline uint32_t max3_u16x2(uint32_t a, uint32_t b, uint32_t c) { return max_u16x2(max_u16x2(a, b), c); }
inline uint32_t byte_perm(uint32_t a, uint32_t b, uint32_t s) {
    uint64_t v = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) {
        uint32_t sel = (s >> (4 * i)) & 7;
        r |= (uint32_t)((v >> (8 * sel)) & 0xff) << (8 * i);
    }
    return r;
}
#endif

// ------------------------------------------------------------------------------------------
// FAST-9/16 score of two horizontally adjacent pixels at once (SURVEY App. A.3;
// cv::FAST response as used at /root/reference/src/ORBextractor.cc:1135-1148).
//   c2   = centre pixels, packed (px0 | px1<<16), values 0..255
//   r[k] = ring pixel k of both centres, packed the same way
// returns packed scores biased by +256 per lane: lane = score + 256 (score in [-256, 254]).
// score = max over the 16 arcs of 9 consecutive ring pixels of max(min d, -max d) - 1, d = c - r.
// ------------------------------------------------------------------------------------------
ORB_HD uint32_t fast_score_x2(uint32_t c2, const uint32_t r[16]) {
    // D[k] = d + 256 per lane in [1, 511]: no borrow crosses the lanes
    uint32_t D[16];
    const uint32_t cb = c2 + 0x01000100u;
#pragma unroll
    for (int k = 0; k < 16; ++k) D[k] = cb - r[k];
    uint32_t lo3[16], hi3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        lo3[k] = min3_u16x2(D[k], D[(k + 1) & 15], D[(k + 2) & 15]);
        hi3[k] = max3_u16x2(D[k], D[(k + 1) & 15], D[(k + 2) & 15]);
    }
    // min / max over each of the 16 arcs of 9, then max-of-min / min-of-max over the arcs (3-input ops)
    uint32_t mn9[16], mx9[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        mn9[k] = min3_u16x2(lo3[k], lo3[(k + 3) & 15], lo3[(k + 6) & 15]);
        mx9[k] = max3_u16x2(hi3[k], hi3[(k + 3) & 15], hi3[(k + 6) & 15]);
    }
    uint32_t a0 = max3_u16x2(mn9[0], mn9[1], mn9[2]), a1 = max3_u16x2(mn9[3], mn9[4], mn9[5]);
    uint32_t a2 = max3_u16x2(mn9[6], mn9[7], mn9[8]), a3 = max3_u16x2(mn9[9], mn9[10], mn9[11]);
    uint32_t a4 = max3_u16x2(mn9[12], mn9[13], mn9[14]);
    const uint32_t best_min = max3_u16x2(max3_u16x2(a0, a1, a2), max3_u16x2(a3, a4, mn9[15]), 0u);
    uint32_t b0 = min3_u16x2(mx9[0], mx9[1], mx9[2]), b1 = min3_u16x2(mx9[3], mx9[4], mx9[5]);
    uint32_t b2 = min3_u16x2(mx9[6], mx9[7], mx9[8]), b3 = min3_u16x2(mx9[9], mx9[10], mx9[11]);
    uint32_t b4 = min3_u16x2(mx9[12], mx9[13], mx9[14]);
    const uint32_t best_max = min3_u16x2(min3_u16x2(b0, b1, b2), min3_u16x2(b3, b4, mx9[15]), 0xffffffffu);
    // bright = best_min - 256 ; dark = 256 - best_max ; score = max(bright, dark) - 1 ; return +256
    // => lane = max(best_min, 512 - best_max) - 1
    const uint32_t dark = 0x02000200u - best_max;  // per lane in [1, 511], no borrow
    return max_u16x2(best_min, dark) - 0x00010001u;
}

// The same score from the RAW ring values (no per-sample subtraction): with A = max over the arcs of (min of the arc) and
// B = min over the arcs of (max of the arc), score = max(A - c, c - B) - 1.  Returns the same +256-biased lanes as fast_score_x2.
ORB_HD uint32_t fast_score_raw_x2(uint32_t c2, const uint32_t r[16]) {
    uint32_t lo3[16], hi3[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        lo3[k] = min3_u16x2(r[k], r[(k + 1) & 15], r[(k + 2) & 15]);
        hi3[k] = max3_u16x2(r[k], r[(k + 1) & 15], r[(k + 2) & 15]);
    }
    uint32_t mn9[16], mx9[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) {
        mn9[k] = min3_u16x2(lo3[k], lo3[(k + 3) & 15], lo3[(k + 6) & 15]);
        mx9[k] = max3_u16x2(hi3[k], hi3[(k + 3) & 15], hi3[(k + 6) & 15]);
    }
    const uint32_t a0 = max3_u16x2(mn9[0], mn9[1], mn9[2]), a1 = max3_u16x2(mn9[3], mn9[4], mn9[5]);
    const uint32_t a2 = max3_u16x2(mn9[6], mn9[7], mn9[8]), a3 = max3_u16x2(mn9[9], mn9[10], mn9[11]);
    const uint32_t a4 = max3_u16x2(mn9[12], mn9[13], mn9[14]);
    const uint32_t A = max_u16x2(max3_u16x2(a0, a1, a2), max3_u16x2(a3, a4, mn9[15]));
    const uint32_t b0 = min3_u16x2(mx9[0], mx9[1], mx9[2]), b1 = min3_u16x2(mx9[3], mx9[4], mx9[5]);
    const uint32_t b2 = min3_u16x2(mx9[6], mx9[7], mx9[8]), b3 = min3_u16x2(mx9[9], mx9[10], mx9[11]);
    const uint32_t b4 = min3_u16x2(mx9[12], mx9[13], mx9[14]);
    const uint32_t B = min_u16x2(min3_u16x2(b0, b1, b2), min3_u16x2(b3, b4, mx9[15]));
    const uint32_t t1 = (A + 0x01000100u) - c2;   // ring brighter than the centre: A - c + 256 per lane, in [1, 511]
    const uint32_t t2 = (c2 + 0x01000100u) - B;   // ring darker:                   c - B + 256
    return max_u16x2(t1, t2) - 0x00010001u;
}

// cv::FAST's high-speed test in packed form: a 9-arc of the 16-ring contains at least one pixel of each antipodal pair,
// so a pixel can only be a corner at threshold T if min over the 4 pairs (k, k+8), k = 0, 2, 4, 6, of max(r_k, r_k+8)
// exceeds c + T (bright arc), or max over the pairs of min(r_k, r_k+8) is below c - T (dark arc).
// hi / lo = that min-of-max / max-of-min for two adjacent pixels (16x2 lanes, raw 0..255); returns a mask with bit 15 /
// bit 31 set for the lane(s) that pass.
ORB_HD uint32_t fast_pretest_x2(uint32_t c2, uint32_t hi, uint32_t lo, uint32_t T2p1) {
    const uint32_t H = 0x80008000u;
    const uint32_t x = (hi | H) - (c2 + T2p1);      // lane >= 0x8000  <=>  hi >= c + T + 1   (no borrow crosses the lanes)
    const uint32_t y = (c2 | H) - (lo + T2p1);      //                 <=>  c >= lo + T + 1
    return (x | y) & H;
}

// hi / lo of fast_pretest_x2 from the 8 even ring samples r[0], r[2], ..., r[14] (packed like the centre)
ORB_HD void fast_pretest_bounds_x2(const uint32_t r[16], uint32_t* hi, uint32_t* lo) {
    *hi = min_u16x2(min3_u16x2(max_u16x2(r[0], r[8]), max_u16x2(r[2], r[10]), max_u16x2(r[4], r[12])), max_u16x2(r[6], r[14]));
    *lo = max_u16x2(max3_u16x2(min_u16x2(r[0], r[8]), min_u16x2(r[2], r[10]), min_u16x2(r[4], r[12])), min_u16x2(r[6], r[14]));
}

// scalar reference form of the same score (used by the emulation test and the slow paths)
ORB_HD int fast_score_scalar(int c, const int ring[16]) {
    int best = -256;
    for (int s = 0; s < 16; ++s) {
        int mn = 255, mx = -255;
        for (int j = 0; j < 9; ++j) {
            const int d = c - ring[(s + j) & 15];
            mn = d < mn ? d : mn;
            mx = d > mx ? d : mx;
        }
        const int v = mn > -mx ? mn : -mx;
        best = v > best ? v : best;
    }
    return best - 1;
}

// ------------------------------------------------------------------------------------------
// float32 helpers with contraction forbidden (SURVEY App. A.4 / A.5 / D)
// ------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
ORB_D float fmul(float a, float b) { return __fmul_rn(a, b); }
ORB_D float fadd(float a, float b) { return __fadd_rn(a, b); }
ORB_D float fsub(float a, float b) { return __fsub_rn(a, b); }
ORB_D float fdiv(float a, float b) { return __fdiv_rn(a, b); }
ORB_D float fsqrt(float a) { return __fsqrt_rn(a); }
ORB_D double dmul(double a, double b) { return __dmul_rn(a, b); }
ORB_D double dadd(double a, double b) { return __dadd_rn(a, b); }
ORB_D int round_half_even(float v) { return __float2int_rn(v); }
#else
// host build must use -ffp-contract=off
inline float fmul(float a, float b) { return a * b; }
inline float fadd(float a, float b) { return a + b; }
inline float fsub(float a, float b) { return a - b; }
inline float fdiv(float a, float b) { return a / b; }
inline float fsqrt(float a) { return sqrtf(a); }
inline double dmul(double a, double b) { return a * b; }
inline double dadd(double a, double b) { return a + b; }
inline int round_half_even(float v) { return (int)lrintf(v); }
#endif

// cv::fastAtan2 scalar path (degrees, [0,360)), SURVEY App. A.4; called from IC_Angle,
// /root/reference/src/ORBextractor.cc:137.
ORB_HD float fast_atan2_deg(float y, float x) {
    const float sc = (float)(180.0 / 3.14159265358979323846);
    const float p1 = fmul(0.9997878412794807f, sc), p3 = fmul(-0.3258083974640975f, sc),
                p5 = fmul(0.1555786518463281f, sc), p7 = fmul(-0.04432655554792128f, sc);
    const float eps = 2.2204460492503131e-16f;
    const float ax = x < 0 ? -x : x, ay = y < 0 ? -y : y;
    float a, c, c2;
    if (ax >= ay) {
        c = fdiv(ay, fadd(ax, eps));
        c2 = fmul(c, c);
        a = fmul(fadd(fmul(fadd(fmul(fadd(fmul(p7, c2), p5), c2), p3), c2), p1), c);
    } else {
        c = fdiv(ax, fadd(ay, eps));
        c2 = fmul(c, c);
        a = fsub(90.f, fmul(fadd(fmul(fadd(fmul(fadd(fmul(p7, c2), p5), c2), p3), c2), p1), c));
    }
    if (x < 0) a = fsub(180.f, a);
    if (y < 0) a = fsub(360.f, a);
    return a;
}

// ---- glibc 2.39 logf (sysdeps/ieee754/flt-32/e_logf.c + e_logf_data.c, the ARM optimized-routines logf):
// x = 2^k z with z in [OFF, 2 OFF), 16-entry table of (1/c, log c), degree-3 polynomial in fp64, one rounding
// to float.  Validated against the host's logf over EVERY positive normal float (2 130 706 432 values, 0
// mismatches, with and without FMA contraction) and sampled in tests/test_host_emul.py.  MapPoint::PredictScale
// (/root/reference/src/MapPoint.cc:688-721) calls std::log(float) == logf.
ORB_HD float glibc_logf(float x) {
    const double T[16][2] = {
        {0x1.661ec79f8f3bep+0, -0x1.57bf7808caadep-2}, {0x1.571ed4aaf883dp+0, -0x1.2bef0a7c06ddbp-2},
        {0x1.49539f0f010bp+0, -0x1.01eae7f513a67p-2},  {0x1.3c995b0b80385p+0, -0x1.b31d8a68224e9p-3},
        {0x1.30d190c8864a5p+0, -0x1.6574f0ac07758p-3}, {0x1.25e227b0b8eap+0, -0x1.1aa2bc79c81p-3},
        {0x1.1bb4a4a1a343fp+0, -0x1.a4e76ce8c0e5ep-4}, {0x1.12358f08ae5bap+0, -0x1.1973c5a611cccp-4},
        {0x1.0953f419900a7p+0, -0x1.252f438e10c1ep-5}, {0x1p+0, 0x0p+0},
        {0x1.e608cfd9a47acp-1, 0x1.aa5aa5df25984p-5},  {0x1.ca4b31f026aap-1, 0x1.c5e53aa362eb4p-4},
        {0x1.b2036576afce6p-1, 0x1.526e57720db08p-3},  {0x1.9c2d163a1aa2dp-1, 0x1.bc2860d22477p-3},
        {0x1.886e6037841edp-1, 0x1.1058bc8a07ee1p-2},  {0x1.767dcf5534862p-1, 0x1.4043057b6ee09p-2}};
    const double Ln2 = 0x1.62e42fefa39efp-1;
    const double A0 = -0x1.00ea348b88334p-2, A1 = 0x1.5575b0be00b6ap-2, A2 = -0x1.ffffef20a4123p-2;
    uint32_t ix;
#if defined(__CUDA_ARCH__)
    ix = __float_as_uint(x);
#else
    memcpy(&ix, &x, 4);
#endif
    if (ix == 0x3f800000u) return 0.0f;
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {   // x < 2^-126, inf or nan
        if (ix * 2 == 0) return -INFINITY;
        if (ix == 0x7f800000u) return x;
        if ((ix & 0x80000000u) || ix * 2 >= 0xff000000u) return NAN;
        const float xs = x * 0x1p23f;                       // subnormal: normalise (exact)
#if defined(__CUDA_ARCH__)
        ix = __float_as_uint(xs);
#else
        memcpy(&ix, &xs, 4);
#endif
        ix -= 23u << 23;
    }
    const uint32_t tmp = ix - 0x3f330000u;
    const int i = (int)((tmp >> 19) & 15u);
    const int k = (int32_t)tmp >> 23;
    const uint32_t iz = ix - (tmp & (0x1ffu << 23));
    float zf;
#if defined(__CUDA_ARCH__)
    zf = __uint_as_float(iz);
#else
    memcpy(&zf, &iz, 4);
#endif
    const double z = (double)zf;
    const double r = dadd(dmul(z, T[i][0]), -1.0);
    const double y0 = dadd(T[i][1], dmul((double)k, Ln2));
    const double r2 = dmul(r, r);
    double y = dadd(dmul(A1, r), A2);
    y = dadd(dmul(A0, r2), y);
    y = dadd(dmul(y, r2), dadd(y0, r));
    return (float)y;
}


// glibc 2.39 sinf/cosf for x in [0, 2*pi] (sysdeps/ieee754/flt-32/s_sincosf.h algorithm: double
// range reduction by pi/2 and degree-7/8 double polynomials).  Validated exhaustively against the
// host's sinf/cosf over every float in [0, 6.3] (tests/test_host_emul.py); that is the definition
// computeOrbDescriptor uses (/root/reference/src/ORBextractor.cc:155-157, SURVEY App. A.4b).
ORB_HD void glibc_sincosf(float y, float* sp, float* cp) {
    const double HPI_INV = 0x1.45F306DC9C883p+23, HPI = 0x1.921FB54442D18p0;
    const double C0 = 0x1p0, C1 = -0x1.ffffffd0c621cp-2, C2 = 0x1.55553e1068f19p-5,
                 C3 = -0x1.6c087e89a359dp-10, C4 = 0x1.99343027bf8c3p-16;
    const double S1 = -0x1.555545995a603p-3, S2 = 0x1.1107605230bc4p-7, S3 = -0x1.994eb3774cf24p-13;
    double x = (double)y;
    uint32_t iy;
#if defined(__CUDA_ARCH__)
    iy = __float_as_uint(y);
#else
    memcpy(&iy, &y, 4);
#endif
    const uint32_t top = (iy >> 20) & 0x7ff;
    int n = 0;
    double sgn = 1.0, cs = 1.0;  // cs = sign applied to the cosine-polynomial coefficients
    if (top < 0x3f4) {           // |y| < pi/4
        if (top < 0x398) {       // |y| < 2^-12
            *sp = y;
            *cp = 1.0f;
            return;
        }
    } else {
        const double r = dmul(x, HPI_INV);
        n = ((int32_t)r + 0x800000) >> 24;
        x = dadd(x, -dmul((double)n, HPI));
        // sign[] = {1,-1,-1,1}[n&3]
        sgn = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
        cs = (n & 2) ? -1.0 : 1.0;
    }
    const double xs = dmul(x, sgn), x2 = dmul(x, x);
    // sine polynomial on xs, cosine polynomial with coefficient sign cs
    const double x3 = dmul(xs, x2);
    const double s1 = dadd(S2, dmul(x2, S3));
    const double x7 = dmul(x3, x2);
    const double s = dadd(xs, dmul(x3, S1));
    const float sinp = (float)dadd(s, dmul(x7, s1));
    const double x4 = dmul(x2, x2);
    const double c2 = dadd(dmul(cs, C3), dmul(x2, dmul(cs, C4)));
    const double c1 = dadd(dmul(cs, C0), dmul(x2, dmul(cs, C1)));
    const double x6 = dmul(x4, x2);
    const double c = dadd(c1, dmul(x4, dmul(cs, C2)));
    const float cosp = (float)dadd(c, dmul(x6, c2));
    if ((n & 1) == 0) {
        *sp = sinp;
        *cp = cosp;
    } else {
        *sp = cosp;
        *cp = sinp;
    }
}

// ------------------------------------------------------------------------------------------
// libstdc++ 13 std::sort (introsort) transcribed for the quadtree's ordered phase
// (/root/reference/src/ORBextractor.cc:950 sorts (count, node) pairs with compareNodes :676-697;
// ties are resolved by the exact sequence of swaps of bits/stl_algo.h, SURVEY App. B item 5).
// Elements are 32-bit keys (count << 16 | ulx) paired with a payload; the comparator is
// "key less-than" -- equal keys are the ties whose final order this reproduces.
// ------------------------------------------------------------------------------------------
struct SortItem {
    uint32_t key;
    uint32_t val;
};

ORB_HD bool si_less(const SortItem& a, const SortItem& b) { return a.key < b.key; }
ORB_HD void si_swap(SortItem& a, SortItem& b) {
    SortItem t = a;
    a = b;
    b = t;
}

ORB_HD void std_adjust_heap(SortItem* first, int hole, int len, SortItem value) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (si_less(first[child], first[child - 1])) --child;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    // __push_heap
    int parent = (hole - 1) / 2;
    while (hole > top && si_less(first[parent], value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}

ORB_HD void std_heap_sort(SortItem* first, int len) {  // __partial_sort(first,last,last)
    if (len >= 2) {                                     // __make_heap
        int parent = (len - 2) / 2;
        while (true) {
            SortItem v = first[parent];
            std_adjust_heap(first, parent, len, v);
            if (parent == 0) break;
            --parent;
        }
    }
    int last = len;
    while (last > 1) {  // __sort_heap / __pop_heap
        --last;
        SortItem v = first[last];
        first[last] = first[0];
        std_adjust_heap(first, 0, last, v);
    }
}

ORB_HD void std_unguarded_linear_insert(SortItem* a, int last) {
    SortItem v = a[last];
    int next = last - 1;
    while (si_less(v, a[next])) {
        a[last] = a[next];
        last = next;
        --next;
    }
    a[last] = v;
}

ORB_HD void std_insertion_sort(SortItem* a, int first, int last) {
    if (first == last) return;
    for (int i = first + 1; i != last; ++i) {
        if (si_less(a[i], a[first])) {
            SortItem v = a[i];
            for (int j = i; j > first; --j) a[j] = a[j - 1];
            a[first] = v;
        } else {
            std_unguarded_linear_insert(a, i);
        }
    }
}

// iterative form of __introsort_loop: the recursion on [cut,last) becomes an explicit stack
ORB_HD void std_sort(SortItem* a, int n) {
    if (n <= 1) return;
    int lg = 0;
    for (int t = n; t > 1; t >>= 1) ++lg;
    int stack_first[64], stack_last[64], stack_depth[64];
    int sp = 0;
    stack_first[0] = 0;
    stack_last[0] = n;
    stack_depth[0] = 2 * lg;
    sp = 1;
    while (sp > 0) {
        --sp;
        int first = stack_first[sp], last = stack_last[sp], depth = stack_depth[sp];
        // the reference recurses on the right part first and loops on the left part: the right
        // part is fully sorted (down to 16-element runs) before the left part is touched.  The
        // two parts are disjoint, so processing order does not change the result.
        while (last - first > 16) {
            if (depth == 0) {
                std_heap_sort(a + first, last - first);
                break;
            }
            --depth;
            const int mid = first + (last - first) / 2;
            {   // __move_median_to_first(first, first+1, mid, last-1)
                const int A = first + 1, B = mid, C = last - 1;
                if (si_less(a[A], a[B])) {
                    if (si_less(a[B], a[C])) si_swap(a[first], a[B]);
                    else if (si_less(a[A], a[C])) si_swap(a[first], a[C]);
                    else si_swap(a[first], a[A]);
                } else if (si_less(a[A], a[C])) si_swap(a[first], a[A]);
                else if (si_less(a[B], a[C])) si_swap(a[first], a[C]);
                else si_swap(a[first], a[B]);
            }
            int lo = first + 1, hi = last;
            while (true) {  // __unguarded_partition(first+1, last, first)
                while (si_less(a[lo], a[first])) ++lo;
                --hi;
                while (si_less(a[first], a[hi])) --hi;
                if (!(lo < hi)) break;
                si_swap(a[lo], a[hi]);
                ++lo;
            }
            const int cut = lo;
            stack_first[sp] = cut;
            stack_last[sp] = last;
            stack_depth[sp] = depth;
            ++sp;
            last = cut;
        }
    }
    // __final_insertion_sort
    if (n > 16) {
        std_insertion_sort(a, 0, 16);
        for (int i = 16; i < n; ++i) std_unguarded_linear_insert(a, i);
    } else {
        std_insertion_sort(a, 0, n);
    }
}

// ------------------------------------------------------------------------------------------
// Quadtree path key (DistributeOctTree / DivideNode, /root/reference/src/ORBextractor.cc:602-674,
// :718-764).  A candidate's descent through the tree depends only on its own coordinates, so its
// whole path can be computed independently: 2 bits per depth (child n1..n4 = 0..3), root index in
// the top bits.  QT_DEPTH levels cover any level up to 8192 px on a side.
// ------------------------------------------------------------------------------------------
#define ORB_QT_DEPTH 13
#define ORB_QT_ROOT_SHIFT (2 * ORB_QT_DEPTH)

struct QtBox {
    int ulx, uly, urx, bry;
};

ORB_HD QtBox qt_root_box(int root, float hX, int regionH) {
    QtBox b;
    b.ulx = (int)fmul(hX, (float)root);
    b.urx = (int)fmul(hX, (float)(root + 1));
    b.uly = 0;
    b.bry = regionH;
    return b;
}

// child q of box b (n1=0: x<mx,y<my; n2=1: x>=mx,y<my; n3=2: x<mx,y>=my; n4=3)
ORB_HD QtBox qt_child_box(const QtBox& b, int q) {
    const int mx = b.ulx + ((b.urx - b.ulx + 1) >> 1);  // ceil(float(w)/2), w >= 0
    const int my = b.uly + ((b.bry - b.uly + 1) >> 1);
    QtBox c;
    c.ulx = (q & 1) ? mx : b.ulx;
    c.urx = (q & 1) ? b.urx : mx;
    c.uly = (q & 2) ? my : b.uly;
    c.bry = (q & 2) ? b.bry : my;
    return c;
}

ORB_HD uint32_t qt_path_key(int x, int y, float hX, int regionH) {
    const int root = (int)fdiv((float)x, hX);
    QtBox b = qt_root_box(root, hX, regionH);
    uint32_t key = (uint32_t)root;
    for (int d = 0; d < ORB_QT_DEPTH; ++d) {
        const int mx = b.ulx + ((b.urx - b.ulx + 1) >> 1);
        const int my = b.uly + ((b.bry - b.uly + 1) >> 1);
        const int q = (x < mx ? 0 : 1) | (y < my ? 0 : 2);
        key = (key << 2) | (uint32_t)q;
        b = qt_child_box(b, q);
    }
    return key;
}

}  // namespace orbdev
