// tests/host_emul/emul.cpp -- compiles the kernels' per-element math (csrc/devmath.cuh) for the HOST so
// the CPU-only test tier can check it against the oracle / glibc / libstdc++ before any GPU run.
// Build: g++ -O2 -ffp-contract=off -shared -fPIC (see tests/test_host_emul.py).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <thread>
#include <vector>

#include "../../orb_slam3_detailed_comments_b200/csrc/devmath.cuh"

using namespace orbdev;

extern "C" {

// scores of pixels (x, x+1) at row y of img (pitch w); returns packed biased lanes
uint32_t emul_fast_x2(const uint8_t* img, int w, int x, int y) {
    static const int RX[16] = {0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3, -3, -3, -2, -1};
    static const int RY[16] = {-3, -3, -2, -1, 0, 1, 2, 3, 3, 3, 2, 1, 0, -1, -2, -3};
    uint32_t r[16];
    for (int k = 0; k < 16; ++k) {
        const uint8_t* p = img + (size_t)(y + RY[k]) * w + x + RX[k];
        r[k] = (uint32_t)p[0] | ((uint32_t)p[1] << 16);
    }
    const uint8_t* c = img + (size_t)y * w + x;
    return fast_score_x2((uint32_t)c[0] | ((uint32_t)c[1] << 16), r);
}

// fast_score_raw_x2 (k_fast_cells_v2) against fast_score_x2 on n random centre / ring sets (extremes and planted arcs included):
// returns the number of sets on which they differ.
long emul_fast_raw_mismatch(uint32_t seed, long n) {
    uint64_t s = seed * 6364136223846793005ull + 1442695040888963407ull;
    auto rnd = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
    long bad = 0;
    for (long it = 0; it < n; ++it) {
        const int mode = rnd() % 4;
        const uint32_t base = rnd() & 0xff, contrast = mode == 0 ? 255 : (mode == 1 ? 40 : 8);
        auto px = [&]() {
            if (mode == 3) return (uint32_t)((rnd() & 1) ? 255 : 0);
            int v = (int)base + (int)(rnd() % (2 * contrast + 1)) - (int)contrast;
            return (uint32_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
        };
        uint32_t r[16];
        const uint32_t c2 = px() | (px() << 16);
        for (int k = 0; k < 16; ++k) r[k] = px() | (px() << 16);
        if (fast_score_raw_x2(c2, r) != fast_score_x2(c2, r)) ++bad;
    }
    return bad;
}

float emul_atan2(float y, float x) { return fast_atan2_deg(y, x); }

// FAST high-speed test vs the full score on random pixel pairs: returns the number of lanes where the score reaches T but
// the test rejects (must be 0: the test is a necessary condition), and through *passed the lanes that pass the test.
long emul_pretest_violations(uint32_t seed, long n, int T, int contrast, long* passed) {
    uint64_t s = seed * 6364136223846793005ull + 1442695040888963407ull;
    auto rnd = [&]() { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
    long bad = 0, pass = 0;
    for (long it = 0; it < n; ++it) {
        const uint32_t base = rnd() & 0xff;
        auto px = [&]() { int v = (int)base + (int)(rnd() % (2 * contrast + 1)) - contrast; v = v < 0 ? 0 : (v > 255 ? 255 : v); return (uint32_t)v; };
        uint32_t r[16];
        const uint32_t c2 = px() | (px() << 16);
        for (int k = 0; k < 16; ++k) r[k] = px() | (px() << 16);
        if ((rnd() & 3) == 0) {               // plant a bright or dark arc so that real corners occur
            const int start = rnd() & 15, len = 9 + (rnd() % 5), sign = (rnd() & 1) ? 1 : -1;
            for (int j = 0; j < len; ++j) {
                const int k = (start + j) & 15;
                int v0 = (int)(c2 & 0xff) + sign * (T + 1 + (int)(rnd() % 40)), v1 = (int)(c2 >> 16) + sign * (T + 1 + (int)(rnd() % 40));
                v0 = v0 < 0 ? 0 : (v0 > 255 ? 255 : v0); v1 = v1 < 0 ? 0 : (v1 > 255 ? 255 : v1);
                r[k] = (uint32_t)v0 | ((uint32_t)v1 << 16);
            }
        }
        uint32_t hi, lo;
        fast_pretest_bounds_x2(r, &hi, &lo);
        const uint32_t m = fast_pretest_x2(c2, hi, lo, (uint32_t)(T + 1) * 0x00010001u);
        const uint32_t sc = fast_score_x2(c2, r);
        const int s0 = (int)(sc & 0xffff) - 256, s1 = (int)(sc >> 16) - 256;
        if (s0 >= T && !(m & 0x8000u)) ++bad;
        if (s1 >= T && !(m & 0x80000000u)) ++bad;
        pass += ((m & 0x8000u) != 0) + ((m & 0x80000000u) != 0);
    }
    *passed = pass;
    return bad;
}

// number of floats in [lo_bits, hi_bits] whose emulated sin or cos differs from glibc's
long emul_sincos_mismatch(uint32_t lo_bits, uint32_t hi_bits, int nthreads) {
    std::atomic<long> bad(0);
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t)
        th.emplace_back([&, t] {
            long b = 0;
            for (uint64_t i = (uint64_t)lo_bits + t; i <= hi_bits; i += nthreads) {
                uint32_t u = (uint32_t)i;
                float f, s, c;
                memcpy(&f, &u, 4);
                glibc_sincosf(f, &s, &c);
                float rs = sinf(f), rc = cosf(f);
                if (memcmp(&s, &rs, 4) || memcmp(&c, &rc, 4)) ++b;
            }
            bad += b;
        });
    for (auto& x : th) x.join();
    return bad.load();
}

void emul_sincos(float a, float* s, float* c) { glibc_sincosf(a, s, c); }

// number of floats in [lo_bits, hi_bits] (stride `step`) whose emulated logf differs from glibc's
long emul_logf_mismatch(uint32_t lo_bits, uint32_t hi_bits, uint32_t step, int nthreads) {
    std::atomic<long> bad(0);
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; ++t)
        th.emplace_back([&, t] {
            long b = 0;
            for (uint64_t i = (uint64_t)lo_bits + (uint64_t)t * step; i <= hi_bits; i += (uint64_t)nthreads * step) {
                uint32_t u = (uint32_t)i;
                float f;
                memcpy(&f, &u, 4);
                const float a = glibc_logf(f), r = logf(f);
                if (memcmp(&a, &r, 4)) ++b;
            }
            bad += b;
        });
    for (auto& x : th) x.join();
    return bad.load();
}

// sorts (key,val) with the transcribed introsort; caller compares against std::sort
void emul_std_sort(uint32_t* keys, uint32_t* vals, int n) {
    std::vector<SortItem> v(n);
    for (int i = 0; i < n; ++i) v[i] = {keys[i], vals[i]};
    std_sort(v.data(), n);
    for (int i = 0; i < n; ++i) { keys[i] = v[i].key; vals[i] = v[i].val; }
}
void emul_heap_sort(uint32_t* keys, uint32_t* vals, int n) {
    std::vector<SortItem> v(n);
    for (int i = 0; i < n; ++i) v[i] = {keys[i], vals[i]};
    std_heap_sort(v.data(), n);
    for (int i = 0; i < n; ++i) { keys[i] = v[i].key; vals[i] = v[i].val; }
}
static bool ref_less(std::pair<uint32_t, uint32_t>& a, std::pair<uint32_t, uint32_t>& b) { return a.first < b.first; }
void ref_std_sort(uint32_t* keys, uint32_t* vals, int n) {
    std::vector<std::pair<uint32_t, uint32_t>> v(n);
    for (int i = 0; i < n; ++i) v[i] = {keys[i], vals[i]};
    std::sort(v.begin(), v.end(), ref_less);
    for (int i = 0; i < n; ++i) { keys[i] = v[i].first; vals[i] = v[i].second; }
}
void ref_heap_sort(uint32_t* keys, uint32_t* vals, int n) {
    std::vector<std::pair<uint32_t, uint32_t>> v(n);
    for (int i = 0; i < n; ++i) v[i] = {keys[i], vals[i]};
    std::partial_sort(v.begin(), v.end(), v.end(), ref_less);
    for (int i = 0; i < n; ++i) { keys[i] = v[i].first; vals[i] = v[i].second; }
}

uint32_t emul_path_key(int x, int y, float hX, int regionH) { return qt_path_key(x, y, hX, regionH); }
}

// ---- quadtree (csrc/quadtree_core.cuh compiled as sequential host code) -----------------------
#include "../../orb_slam3_detailed_comments_b200/csrc/quadtree_core.cuh"
static int emul_distribute_variant(int variant, const int32_t* cand3, int n, int regionW, int regionH, int N, int wCell, int hCell,
                                   int nCols, int32_t* out3, int cap_out) {
    QtGeom g;
    g.regionW = regionW; g.regionH = regionH;
    g.nIni = (int)std::round((float)regionW / (float)regionH);
    if (g.nIni < 1 || g.nIni > 4) return -2;
    g.hX = (float)regionW / (float)g.nIni;
    g.N = N; g.wCell = wCell; g.hCell = hCell; g.nCols = nCols;
    int npow = 2;
    while (npow < n) npow <<= 1;
    std::vector<uint32_t> arr(npow, 0xffffffffu);
    for (int i = 0; i < n; ++i) arr[i] = qt_element(qt_pack_cand(cand3[3 * i], cand3[3 * i + 1], cand3[3 * i + 2]), g);
    if (variant == 0) qt_bitonic_sort(arr.data(), npow); else qt_bitonic_sort_r8(arr.data(), npow);
    const int cap = N + 20;
    std::vector<char> ws(qt_work_bytes(cap));
    QtWork w;
    qt_work_carve(w, ws.data(), cap);
    std::vector<uint32_t> out(cap + 4);
    const int S = variant == 0 ? qt_distribute(arr.data(), n, g, w, out.data()) : qt_distribute_v<1>(arr.data(), n, g, w, out.data());
    for (int i = 0; i < S && i < cap_out; ++i) {
        out3[3 * i] = out[i] & 0xfff;
        out3[3 * i + 1] = (out[i] >> 12) & 0xfff;
        out3[3 * i + 2] = out[i] >> 24;
    }
    return S;
}

extern "C" int emul_distribute(const int32_t* cand3, int n, int regionW, int regionH, int N, int wCell, int hCell, int nCols,
                               int32_t* out3, int cap_out) {
    return emul_distribute_variant(0, cand3, n, regionW, regionH, N, wCell, hCell, nCols, out3, cap_out);
}
extern "C" int emul_distribute_v1(const int32_t* cand3, int n, int regionW, int regionH, int N, int wCell, int hCell, int nCols,
                                  int32_t* out3, int cap_out) {
    return emul_distribute_variant(1, cand3, n, regionW, regionH, N, wCell, hCell, nCols, out3, cap_out);
}

// std::sort(vSizeAndPointerToNode, compareNodes) three ways: libstdc++ itself, the one-thread transcription, the CTA-parallel form.
// items: n x (cnt, ulx, payload); which = 0 libstdc++, 1 qt_std_sort_items, 2 qt_std_sort_items_par.  out: payloads in sorted order.
extern "C" void emul_sort_items(const uint32_t* items3, int n, int which, uint32_t* out_payload) {
    std::vector<QtItem> abuf(n + 9), tmp(n + 1);      // four items of padding either side: the partition's scans read ahead
    QtItem* a = abuf.data() + 4;
    for (int i = 0; i < n; ++i) { a[i].cnt = items3[3 * i]; a[i].ulx_pos = (items3[3 * i + 1] << 16) | (items3[3 * i + 2] & 0xffffu); }
    if (which == 0) {
        std::sort(a, a + n, [](const QtItem& x, const QtItem& y) { return qt_item_less(x, y); });
    } else if (which == 1) {
        qt_std_sort_items(a, n);
    } else {
        std::vector<int> seg(n + 64), nxt(4 * n + 64), flag(n + 64), st(64);
        qt_std_sort_items_par(a, n, tmp.data(), seg.data(), nxt.data(), flag.data(), st.data(), 4 * n + 64);
    }
    for (int i = 0; i < n; ++i) out_payload[i] = a[i].ulx_pos & 0xffffu;
}

extern "C" void emul_bitonic(uint32_t* arr, int npow, int variant) {
    if (variant == 0) qt_bitonic_sort(arr, npow); else if (variant == 1) qt_bitonic_sort_r4(arr, npow); else qt_bitonic_sort_r8(arr, npow);
}

// ---- LocalInertialBA: the device algorithm (csrc/liba_core.cuh) run by one host "thread" ---------------------------------------
#include "../../orb_slam3_detailed_comments_b200/csrc/liba_pack.h"

extern "C" int emul_liba(const liba_problem* p, liba_result* r) {
    const orb::LibaLayout lay = orb::liba_pack(*p, nullptr, nullptr, nullptr);
    if (lay.total == 0) return -1;
    std::vector<uint8_t> blob(lay.total + 16, 0);
    orb::LibaDev dev;
    orb::liba_pack(*p, blob.data(), blob.data(), &dev);
    orb::liba_optimize(dev);
    orb::liba_unpack(*p, blob.data(), dev, blob.data(), r);
    return r->iterations;
}

// one EdgeInertial through the device code: e9, J[9][24]
extern "C" void emul_liba_inertial(const double* state2x21, const liba_link* link, double* e9, double* J216) {
    orb::LibaDev dev;
    memset(&dev, 0, sizeof(dev));
    dev.state = const_cast<double*>(state2x21);
    orb::LibaLink L;
    memcpy(&L, link, sizeof(L));
    L.k1 = 0; L.k2 = 1;
    orb::liba_inertial(dev, L, e9, J216);
}

extern "C" size_t emul_liba_layout_total(const liba_problem* p) { return orb::liba_pack(*p, nullptr, nullptr, nullptr).total; }

// ---- LocalBundleAdjustment: the index structures and the batch layout of csrc/lba_pack.h ----------------------------------------
#include "../../orb_slam3_detailed_comments_b200/csrc/lba_pack.h"

#define EMUL_LBA_POINTERS(X) X(pose0) X(point0) X(pidx) X(ekf) X(emp) X(obs) X(invs2) X(mpStart) X(mpEdge) X(poseStart) X(poseEdge) \
    X(pairStart) X(ptItemStart) X(ptItem) X(taskStart) X(blockTask) X(taskSum) X(BD) X(poseSlot) X(blockP1) X(blockP2) X(pose)      \
    X(point) X(poseSave) X(pointSave) X(Hpl) X(W) X(Prod) X(Hll) X(bl) X(Dinv) X(db) X(Hpp) X(bp) X(xl) X(HsGlobal) X(posePart)       \
    X(HsBlocks) X(bs) X(xp) X(partials) X(flags) X(err) X(depthPos) X(stats)
#define EMUL_LBA_INTS(X) X(nKF) X(nMP) X(nE) X(nP) X(n) X(nItems) X(nTasks) X(nFreeEdges) X(nPairBlocks)
#define EMUL_LBA_NAME(m) #m " "

// the descriptor members emul_lba_pack exports, in its order
extern "C" const char* emul_lba_fields() { return EMUL_LBA_POINTERS(EMUL_LBA_NAME) EMUL_LBA_INTS(EMUL_LBA_NAME); }

// lba_prepare + lba_pack of n problems with blob as both the host mirror and the device block: blob == nullptr measures.
// sizes = in, desc, work bytes; fields[n][emul_lba_fields]: the blob offset a pointer member points at (-1: null), then the ints.
// Returns lba_prepare's status of the first problem it refuses.
extern "C" int emul_lba_pack(const lba_problem* p, int n, uint8_t* blob, int64_t* sizes, int64_t* fields) {
    std::vector<orb::LbaPrep> prep(n);
    for (int i = 0; i < n; ++i) {
        const char* why = nullptr;
        const orb_status s = orb::lba_prepare(p[i], prep[i], &why);
        if (s != ORB_OK) return s;
    }
    const orb::LbaLayout lay = orb::lba_pack(n, p, prep.data(), nullptr, blob, blob);
    sizes[0] = (int64_t)lay.in_bytes; sizes[1] = (int64_t)lay.desc_bytes; sizes[2] = (int64_t)lay.work_bytes;
    if (!blob) return ORB_OK;
    const orb::LbaDev* D = reinterpret_cast<const orb::LbaDev*>(blob + lay.in_bytes);
    int64_t* f = fields;
    for (int i = 0; i < n; ++i) {
#define EMUL_LBA_PTR(m) *f++ = D[i].m ? (int64_t)((const uint8_t*)D[i].m - blob) : -1;
#define EMUL_LBA_INT(m) *f++ = D[i].m;
        EMUL_LBA_POINTERS(EMUL_LBA_PTR)
        EMUL_LBA_INTS(EMUL_LBA_INT)
    }
    return ORB_OK;
}

// ---- Frame::ComputeStereoMatches, variant 1: csrc/stereo_core.cuh (the body of k_stereo_match_v1's threads) on the host ----------------
#include "../../orb_slam3_detailed_comments_b200/csrc/stereo_core.cuh"

// levelsL / levelsR: nlevels pointers to the raw pyramid levels (tightly packed, pitch = width); wl / wr: their widths.
// Outputs per left keypoint BEFORE the median-SAD filter (Frame.cc:1338-1357): uright, depth, sad (-1 = none).
extern "C" void emul_stereo_v1(const orbx_keypoint* kL, const uint8_t* dL, int nL, const orbx_keypoint* kR, const uint8_t* dR, int nR,
                               int nlevels, const uint8_t* const* levelsL, const uint8_t* const* levelsR, const int* wl, const int* wr,
                               const float* scale, const float* inv_scale, int H, float bf, float b, float* out_u, float* out_d,
                               int* out_sad) {
    std::vector<float> x(nR + 1);
    std::vector<int> band(nR + 1), off(H + 2, 0), ent(nR + 1);
    std::vector<signed char> oct(nR + 1);
    for (int j = 0; j < nR; ++j) {
        const float r = fmul(2.0f, scale[kR[j].octave]);
        const int maxr = (int)ceilf(fadd(kR[j].y, r)), minr = (int)floorf(fsub(kR[j].y, r));
        x[j] = kR[j].x;
        band[j] = (minr & 0xffff) | (maxr << 16);
        oct[j] = (signed char)kR[j].octave;
        ++off[st_row_bucket(kR[j].y, H) + 1];
    }
    for (int i = 0; i < H; ++i) off[i + 1] += off[i];
    {
        std::vector<int> cur(off.begin(), off.begin() + H);
        for (int j = nR - 1; j >= 0; --j) ent[cur[st_row_bucket(kR[j].y, H)]++] = j;     // reversed on purpose: bucket order must not matter
    }
    std::vector<StLevel> lv(nlevels);
    for (int l = 0; l < nlevels; ++l) {
        lv[l].L = levelsL[l]; lv[l].R = levelsR[l];
        lv[l].pitchL = wl[l]; lv[l].pitchR = wr[l]; lv[l].wR = wr[l];
        lv[l].scale = scale[l]; lv[l].inv_scale = inv_scale[l];
    }
    StRight R;
    R.x = x.data(); R.band = band.data(); R.oct = oct.data(); R.row_off = off.data(); R.row_ent = ent.data();
    R.H = H; R.W = st_scan_window(scale[nlevels - 1]);
    for (int i = 0; i < nL; ++i)
        stereo_match_one(kL[i].x, kL[i].y, kL[i].octave, reinterpret_cast<const uint32_t*>(dL + 32 * (size_t)i), R, dR, lv.data(), bf, b,
                         &out_u[i], &out_d[i], &out_sad[i]);
}

// ---- ComputePyramid, one level transition: csrc/resize_core.cuh (the body of k_resize_v3's threads) on the host ------------------------
#include "../../orb_slam3_detailed_comments_b200/csrc/resize_core.cuh"

// src: sh rows of spitch bytes (src_avail readable bytes from src: the word loads stop there); dst: dh rows of dpitch bytes.
extern "C" void emul_resize_v3(const uint8_t* src, int sw, int sh, int spitch, long src_avail, uint8_t* dst, int dw, int dh, int dpitch) {
    std::vector<int> tx(2 * dw), ty(2 * dh);
    rs_linear_taps(sw, dw, tx.data());
    rs_linear_taps(sh, dh, ty.data());
    for (int dy0 = 0; dy0 < dh; dy0 += 4)
        for (int dx4 = 0; dx4 < dw; dx4 += 4)
            rs_thread<4>(src, sw, sh, spitch, src + src_avail, dst, dw, dh, dpitch, tx.data(), ty.data(), dx4, dy0);
}
