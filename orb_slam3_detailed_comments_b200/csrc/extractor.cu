// extractor.cu -- host side of the batched ORB extractor + its C ABI (include/orbslam3_b200.h).
// Replaces ORBextractor::ORBextractor / operator() / ComputePyramid / ComputeKeyPointsOctTree
// (/root/reference/src/ORBextractor.cc:468-571, 1557-1682, 1687-1738, 1061-1208).
#include <math.h>
#include <string.h>

#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "extractor.h"
#include "extractor_kernels.cuh"
#include "blur_mma.cuh"

namespace orb {
thread_local std::string g_last_error;
std::atomic<long long> g_launches{0};
}  // namespace orb

using namespace orb;

static inline int round_up(int v, int a) { return (v + a - 1) / a * a; }
static inline int pow2_ceil(int v) {
    int p = 2;
    while (p < v) p <<= 1;
    return p;
}

// ------------------------------------------------------------------------------------------
// constructor tables -- ORBextractor.cc:478-570 (float32 arithmetic mirrored operation by operation)
// ------------------------------------------------------------------------------------------
static void build_tables(orbx_handle* h) {
    const int nl = h->cfg.n_levels;
    const float sf = h->cfg.scale_factor;
    h->scale.assign(nl, 1.f);
    h->sigma2.assign(nl, 1.f);
    for (int i = 1; i < nl; ++i) {
        h->scale[i] = (float)(h->scale[i - 1] * (double)sf);   // the member is `double scaleFactor` (ORBextractor.h:99)
        h->sigma2[i] = h->scale[i] * h->scale[i];
    }
    h->inv_scale.resize(nl);
    h->inv_sigma2.resize(nl);
    for (int i = 0; i < nl; ++i) {
        h->inv_scale[i] = 1.0f / h->scale[i];
        h->inv_sigma2[i] = 1.0f / h->sigma2[i];
    }
    h->quota.resize(nl);
    const float factor = (float)(1.0f / (double)sf);
    float per = h->cfg.n_features * (1 - factor) / (1 - (float)pow((double)factor, (double)nl));
    int sum = 0;
    for (int l = 0; l < nl - 1; ++l) {
        h->quota[l] = (int)lrintf(per);
        sum += h->quota[l];
        per *= factor;
    }
    h->quota[nl - 1] = std::max(h->cfg.n_features - sum, 0);
    h->umax.assign(16, 0);
    const int vmax = (int)floor(15 * sqrt(2.f) / 2 + 1), vmin = (int)ceil(15 * sqrt(2.f) / 2);
    for (int v = 0; v <= vmax; ++v) h->umax[v] = (int)lrint(sqrt(225.0 - v * v));
    for (int v = 15, v0 = 0; v >= vmin; --v) {
        while (h->umax[v0] == h->umax[v0 + 1]) ++v0;
        h->umax[v] = v0;
        ++v0;
    }
}

// cv::resize INTER_LINEAR tap table: resize_core.cuh (shared with the host emulation of k_resize_v3)
static void linear_taps(int ssize, int dsize, int2* out) { orbdev::rs_linear_taps(ssize, dsize, reinterpret_cast<int*>(out)); }

// DistributeOctTree's sort element of a level (quadtree_core.cuh QtForm): the 64-bit, 12-depth form when a side of the region
// (maxBorder - minBorder) exceeds 2048 px, the 32-bit, 11-depth form otherwise
static bool qt_level_k64(const LevelGeom& L) {
    return L.maxBX - 16 > orbdev::QtForm<uint32_t>::max_dim || L.maxBY - 16 > orbdev::QtForm<uint32_t>::max_dim;
}

// the region of level 0 (side - 32) must fit the 12-bit candidate coordinates and the 12-depth quadtree element
static orb_status check_image_side(int w, int hh) {
    const int lim = orbdev::QtForm<uint64_t>::max_dim + 32;
    if (w > lim || hh > lim) return set_error(ORB_ERR_UNSUPPORTED, "image side > 4128 px is not supported (12-bit candidate coordinates)");
    return ORB_OK;
}

// geometry for images of (w,h); (re)allocates nothing -- buffers are sized for max_width/max_height
static orb_status plan_geometry(orbx_handle* h, int w, int hh) {
    if (check_image_side(w, hh) != ORB_OK) return ORB_ERR_UNSUPPORTED;
    const int nl = h->cfg.n_levels;
    ExtractGeom& g = h->geom;
    memset(&g, 0, sizeof(g));
    g.nlevels = nl;
    g.iniTh = h->cfg.ini_th_fast;
    g.minTh = h->cfg.min_th_fast;
    std::vector<int2> taps;
    int cells = 0, tiles = 0, cand = 0, kp = 0, sortOff = 0;
    for (int l = 0; l < nl; ++l) {
        LevelGeom& L = g.lv[l];
        L.w = (int)lrintf((float)w * h->inv_scale[l]);   // ORBextractor.cc:1691-1692
        L.h = (int)lrintf((float)hh * h->inv_scale[l]);
        L.pitch = round_up(L.w, 16);
        L.blur_pitch = L.pitch;
        L.img_stride = (int64_t)L.pitch * L.h;
        L.blur_stride = L.img_stride;
        L.base = nullptr;  // assigned by apply_geometry
        L.blur = nullptr;
        // FAST cells, ORBextractor.cc:1076-1095
        L.maxBX = L.w - 16;
        L.maxBY = L.h - 16;
        const float width = (float)(L.maxBX - 16), height = (float)(L.maxBY - 16);
        L.nCols = (int)(width / 35.f);
        L.nRows = (int)(height / 35.f);
        if (L.nCols < 1 || L.nRows < 1)
            return set_error(ORB_ERR_UNSUPPORTED, "pyramid level smaller than one FAST cell (reference divides by zero)");
        L.wCell = (int)ceilf(width / L.nCols);
        L.hCell = (int)ceilf(height / L.nRows);
        L.cellBase = cells;
        cells += L.nCols * L.nRows;
        g.fastRows = std::max(g.fastRows, L.hCell + 6);
        L.tilesX = (L.w + BLUR_TW - 1) / BLUR_TW;
        L.tilesY = (L.h + BLUR_TH - 1) / BLUR_TH;
        L.tileBase = tiles;
        tiles += L.tilesX * L.tilesY;
        // quadtree, ORBextractor.cc:715-716
        L.quota = h->quota[l];
        L.nIni = (int)roundf(width / height);
        if (L.nIni < 1 || L.nIni > 4)
            return set_error(ORB_ERR_UNSUPPORTED, "aspect ratio outside [0.5, 4.5): nIni must be 1..4");
        L.hX = width / (float)L.nIni;
        // worst case of strict 3x3 local maxima: one per 2x2 block of every cell's tested area
        int cap = 0;
        for (int i = 0; i < L.nRows; ++i) {
            const int y0 = 16 + i * L.hCell;
            if (y0 >= L.maxBY - 3) continue;
            const int th = std::min(y0 + L.hCell + 6, L.maxBY) - y0 - 6;
            for (int j = 0; j < L.nCols; ++j) {
                const int x0 = 16 + j * L.wCell;
                if (x0 >= L.maxBX - 6) continue;
                const int tw = std::min(x0 + L.wCell + 6, L.maxBX) - x0 - 6;
                if (tw > 0 && th > 0) cap += ((tw + 1) / 2) * ((th + 1) / 2);
            }
        }
        L.candCap = round_up(std::max(cap, 4), 4);
        L.candOff = cand;
        cand += L.candCap;
        L.kpCap = qt_node_cap(L.quota);   // the node list never exceeds N + 3 (quadtree_core.cuh)
        L.kpOff = kp;
        kp += L.kpCap;
        L.sortOff = sortOff;   // uint32 slots; every block is a power of two >= 4 slots, so 64-bit blocks stay 16-byte aligned
        sortOff += pow2_ceil(L.candCap) * (qt_level_k64(L) ? 2 : 1);
        L.scale = h->scale[l];
        L.inv_scale = h->inv_scale[l];
        L.patch = (float)(int)(31 * h->scale[l]);   // ORBextractor.cc:1184
        L.tapOff = (int)taps.size();
        L.area2x = 0;
        if (l > 0) {
            const LevelGeom& P = g.lv[l - 1];
            L.area2x = (P.w == 2 * L.w && P.h == 2 * L.h) ? 1 : 0;
            taps.resize(taps.size() + L.w + L.h);
            linear_taps(P.w, L.w, taps.data() + L.tapOff);
            linear_taps(P.h, L.h, taps.data() + L.tapOff + L.w);
        }
    }
    if (g.fastRows > FAST_ROWS) return set_error(ORB_ERR_UNSUPPORTED, "FAST cell taller than the staging arrays");
    {   // k_fast_cells_v2: table of the cells cv::FAST actually tests (ORBextractor.cc:1098-1126), staging sizes from the geometry
        h->cells_host.clear();
        int maxCh = 7, maxPairs = 8, maxTask = 1;
        for (int l = 0; l < nl; ++l) {
            const LevelGeom& L = g.lv[l];
            for (int i = 0; i < L.nRows; ++i)
                for (int j = 0; j < L.nCols; ++j) {
                    const int x0 = 16 + j * L.wCell, y0 = 16 + i * L.hCell;
                    if (x0 >= L.maxBX - 6 || y0 >= L.maxBY - 3) continue;
                    const int cw = std::min(x0 + L.wCell + 6, L.maxBX) - x0, ch = std::min(y0 + L.hCell + 6, L.maxBY) - y0;
                    if (cw < 7 || ch < 7) continue;
                    if (cw > 255 || ch > 255) return set_error(ORB_ERR_UNSUPPORTED, "FAST cell wider than 255 px");
                    if (x0 > 0xfff || y0 > 0xfff) return set_error(ORB_ERR_UNSUPPORTED, "FAST cell origin beyond the 12-bit cell table");
                    h->cells_host.push_back(make_uint2((uint32_t)x0 | ((uint32_t)y0 << 12) | ((uint32_t)l << 24), (uint32_t)cw | ((uint32_t)ch << 8)));
                    const int tx0 = x0 + 3, tx1 = x0 + cw - 3;
                    const int gx0 = ((tx0 & ~3) - 4) & ~7, wd0 = ((tx0 & ~3) - gx0) >> 2, ngrp = ((tx1 - 1) >> 2) - (tx0 >> 2) + 1;
                    const int nC8 = (wd0 + ngrp + 2) >> 1;
                    maxCh = std::max(maxCh, ch);
                    maxPairs = std::max(maxPairs, 4 * nC8);
                    maxTask = std::max(maxTask, (ch - 6) * ngrp);
                }
        }
        h->fast_R = maxCh;
        h->fast_PW = maxPairs | 1;   // odd row stride: the lanes of a warp work on consecutive rows (bank-conflict-free)
        h->fast_LW = 64 * ((round_up(maxTask, 32) + FAST2_THREADS - 1) / FAST2_THREADS);   // per warp: both pairs of every task it tests
        if (h->fast_PW > 64) return set_error(ORB_ERR_UNSUPPORTED, "FAST cell wider than the pair index of k_fast_cells_v2");
    }
    g.totalCells = cells;
    g.totalTiles = tiles;
    g.candTotal = cand;
    g.kpTotal = kp;
    g.sortTotal = sortOff;
    h->taps_host = taps;
    h->cur_w = w;
    h->cur_h = hh;
    return ORB_OK;
}

// Places the levels of the planned geometry in the two pyramid blocks, each level base 256-byte aligned (the ORB_FAST_TMA path needs
// 16): returns the bytes the levels take.  On null blocks (orbx_create's sizing) it only measures.
static size_t place_levels(orbx_handle* h) {
    Carve pyr{h->d_pyr}, blur{h->d_blur};
    for (int l = 0; l < h->cfg.n_levels; ++l) {
        LevelGeom& L = h->geom.lv[l];
        L.base = pyr.take<uint8_t>((size_t)L.img_stride * h->cfg.max_batch);
        L.blur = blur.take<uint8_t>((size_t)L.img_stride * h->cfg.max_batch);
    }
    return (pyr.off + 255) / 256 * 256;
}

// One (image, level)'s quadtree node workspace: qt_node_cap(N) nodes for the largest quota N (quadtree_core.cuh)
static size_t qt_node_bytes(const orbx_handle* h) { return (qt_work_bytes(h->qt_node_cap) + 15) / 16 * 16; }

extern "C" const char* orb_last_error(void) { return g_last_error.c_str(); }
extern "C" int orb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}
extern "C" int64_t orb_kernel_launches(void) { return (int64_t)g_launches.load(); }

// upper bound of the keypoints one image can produce (sum over the levels of quota + 20): the row stride of the per-image
// outputs of orbv_transform
extern "C" int32_t orbx_max_features(const orbx_handle* h) {
    if (!h) return 0;
    int t = 0;
    for (int l = 0; l < h->cfg.n_levels; ++l) t += qt_node_cap(h->quota[l]);
    return t;
}

static orb_status apply_geometry(orbx_handle* h, int w, int hh) {
    if (w == h->cur_w && hh == h->cur_h) return ORB_OK;
    if (check_image_side(w, hh) != ORB_OK) return ORB_ERR_UNSUPPORTED;   // before the handle's size: a refusal, not a usage error
    if (w > h->cfg.max_width || hh > h->cfg.max_height || w < 1 || hh < 1)
        return set_error(ORB_ERR_INVALID, "image larger than the handle's max_width/max_height");
    // pyramid base pointers are laid out for the CURRENT size inside the max-size allocation
    orb_status s = plan_geometry(h, w, hh);
    if (s != ORB_OK) {
        h->cur_w = h->cur_h = -1;
        return s;
    }
    if (place_levels(h) + 4096 > h->pyr_bytes) return set_error(ORB_ERR_CAPACITY, "pyramid allocation too small");
    if ((size_t)h->geom.candTotal > h->cand_slots || (size_t)h->geom.kpTotal > h->kp_slots ||
        (size_t)h->geom.sortTotal > h->sort_slots || h->taps_host.size() > h->taps_slots || h->cells_host.size() > h->cells_slots)
        return set_error(ORB_ERR_CAPACITY, "workspace sized for max image is too small for this size");
    ORB_CUDA(cudaMemcpyAsync(h->d_taps, h->taps_host.data(), h->taps_host.size() * sizeof(int2), cudaMemcpyHostToDevice,
                             h->stream));
    ORB_CUDA(cudaMemcpyAsync(h->d_cells, h->cells_host.data(), h->cells_host.size() * sizeof(uint2), cudaMemcpyHostToDevice, h->stream));
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    const size_t nodeBytes = qt_node_bytes(h);
    // Sort capacity in shared memory per level: a texture-rich level yields about one FAST candidate
    // per 37 tested pixels; provision area/24 and fall back to the global scratch beyond that.
    // Consecutive levels with the same capacity form a group (<= 4 groups, one launch each on its own stream).
    {
        // Levels whose region side exceeds 2048 px (a prefix of the pyramid) sort 64-bit elements: they form one group of their own, run by
        // k_quadtree_v1_k64; the other levels are grouped as before and keep their kernels.
        int capOf[ORB_MAX_LEVELS];
        bool k64Of[ORB_MAX_LEVELS];
        for (int l = 0; l < h->cfg.n_levels; ++l) k64Of[l] = qt_level_k64(h->geom.lv[l]);
        if (k64Of[0] && (h->qt_variant == 0 || h->qt_max_groups == 4))
            return set_error(ORB_ERR_UNSUPPORTED, "regions over 2048 px need k_quadtree_v1's 64-bit form: ORB_QT_VARIANT=0 and ORB_QT_GROUPS=4 "
                                                  "support images up to 2080 px only");
        for (int l = 0; l < h->cfg.n_levels; ++l) {
            const LevelGeom& L = h->geom.lv[l];
            const size_t esz = k64Of[l] ? 8 : 4;
            const int est = (int)((int64_t)(L.maxBX - 16) * (L.maxBY - 16) / 24);
            int c = pow2_ceil(std::max(est, 1024));
            c = std::min(c, 32768);
            if (c > 8192) c = std::max(c, 16384);
            else if (c > 4096 || (c > 2048 && h->qt_max_groups < 4)) c = 8192;
            else if (c > 2048) c = 4096;     // ORB_QT_GROUPS=4 only: levels 2-4 of a 640x480 pyramid sort <= 4096 keys
            else c = 2048;
            while ((size_t)c * esz + (h->qt_nodes_in_smem ? nodeBytes : 0) > 200 * 1024 && c > 2048) c >>= 1;
            capOf[l] = c;
        }
        for (int l = 1; l < h->cfg.n_levels; ++l)
            if (k64Of[l] == k64Of[l - 1]) capOf[l] = std::min(capOf[l], capOf[l - 1]);  // monotone within a form
        const int k64Groups = k64Of[0] ? 1 : 0;
        h->qt_ngroups = 0;
        for (int l = 0; l < h->cfg.n_levels; ++l) {
            const orbx_handle::QtGroup* P = h->qt_ngroups > 0 ? &h->qt_groups[h->qt_ngroups - 1] : nullptr;
            if (P && P->k64 == k64Of[l] &&
                (k64Of[l] || capOf[l] == P->sort_cap || h->qt_ngroups - k64Groups == h->qt_max_groups)) {
                h->qt_groups[h->qt_ngroups - 1].level_end = l + 1;
            } else {
                orbx_handle::QtGroup& G = h->qt_groups[h->qt_ngroups++];
                G.level_begin = l;
                G.level_end = l + 1;
                G.sort_cap = capOf[l];
                G.k64 = k64Of[l];
            }
        }
        size_t maxSmem = 0, maxSmem64 = 0;
        for (int i = 0; i < h->qt_ngroups; ++i) {
            // a group that absorbed smaller levels keeps its (larger) capacity: always sufficient
            orbx_handle::QtGroup& G = h->qt_groups[i];
            G.smem = (size_t)G.sort_cap * (G.k64 ? 8 : 4) + (h->qt_nodes_in_smem ? nodeBytes : 0);
            (G.k64 ? maxSmem64 : maxSmem) = std::max(G.k64 ? maxSmem64 : maxSmem, G.smem);
        }
        ORB_CUDA(cudaFuncSetAttribute(k_quadtree, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxSmem));
        ORB_CUDA(cudaFuncSetAttribute(k_quadtree_v1<QT_THREADS, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxSmem));
        ORB_CUDA(cudaFuncSetAttribute(k_quadtree_v1<1024, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxSmem));
        if (k64Groups)
            ORB_CUDA(cudaFuncSetAttribute(k_quadtree_v1_k64<QT_K64_THREADS, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)maxSmem64));
    }
    const size_t ordBytes = ((size_t)h->geom.kpTotal + 64) * 4;
    static const size_t orderStatic = static_smem(k_order);
    if ((s = check_smem(h, ordBytes, orderStatic, "k_order")) != ORB_OK) {
        h->cur_w = h->cur_h = -1;
        return s;
    }
    ORB_CUDA(cudaFuncSetAttribute(k_order, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(ordBytes, (size_t)1024)));
    h->order_smem_bytes = ordBytes;
    return ORB_OK;
}

extern "C" orb_status orbx_create(const orbx_config* cfg, orbx_handle** out) {
    if (!cfg || !out) return set_error(ORB_ERR_INVALID, "null argument");
    *out = nullptr;
    if (cfg->n_levels < 1 || cfg->n_levels > ORB_MAX_LEVELS || cfg->n_features < 1 || cfg->scale_factor <= 1.0f ||
        cfg->min_th_fast < 1 || cfg->ini_th_fast < cfg->min_th_fast || cfg->ini_th_fast > 254 || cfg->max_batch < 1 ||
        cfg->max_width < 1 || cfg->max_height < 1)
        return set_error(ORB_ERR_INVALID, "bad extractor configuration");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= cfg->device || cfg->device < 0)
        return set_error(ORB_ERR_NO_DEVICE, "no usable CUDA device (this library has no CPU fallback)");
    ORB_CUDA(cudaSetDevice(cfg->device));
    orbx_handle* h = new orbx_handle();
    h->cfg = *cfg;
    if (const char* v = getenv("ORB_FAST_VARIANT")) h->fast_variant = atoi(v) == 0 ? 0 : 1;   // 0 selects the round-1 kernel
    if (const char* v = getenv("ORB_QT_VARIANT")) h->qt_variant = atoi(v) == 0 ? 0 : 1;   // 0 selects the round-1 kernel (k_quadtree)
    if (const char* v = getenv("ORB_BLUR_VARIANT")) h->blur_variant = atoi(v);       // 1: k_blur<true> (IDP.4A), 0: k_blur<false> (packed 16x2 multiply-adds)
    if (const char* v = getenv("ORB_RESIZE_VARIANT")) h->resize_variant = atoi(v);   // 0: k_resize (4 px of one row per thread)
    if (const char* v = getenv("ORB_FAST_TMA")) h->fast_tma = atoi(v) != 0;   // window rows of k_fast_cells_v2 staged by TMA bulk copies
    if (const char* v = getenv("ORB_QT_GROUPS")) h->qt_max_groups = atoi(v) == 4 ? 4 : 3;
    build_tables(h);
    static const int kUmax[16] = {15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3};
    for (int i = 0; i < 16; ++i)
        if (h->umax[i] != kUmax[i]) {
            delete h;
            return set_error(ORB_ERR_INVALID, "umax table mismatch");
        }
    orb_status s = ORB_OK;
    auto fail = [&](orb_status st) {
        orbx_destroy(h);
        return st;
    };
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess)
        return fail(set_error(ORB_ERR_CUDA, "cudaStreamCreate failed"));
    for (int r = 0; r < orbx_handle::kProfRing; ++r)
        for (int i = 0; i < 8; ++i) cudaEventCreate(&h->evr[r][i]);
    for (int i = 0; i < 3; ++i) {
        cudaStreamCreateWithFlags(&h->aux_stream[i], cudaStreamNonBlocking);
        cudaEventCreateWithFlags(&h->ev_join[i], cudaEventDisableTiming);
    }
    cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming);
    // size every buffer for the largest image: the capacities of the max-size plan bound every size the handle accepts
    h->d_pyr = h->d_blur = nullptr;
    s = plan_geometry(h, cfg->max_width, cfg->max_height);
    if (s != ORB_OK) return fail(s);
    h->cur_w = h->cur_h = -1;
    const int B = cfg->max_batch;
    h->pyr_bytes = place_levels(h) + 4096;   // slack after the last level: k_resize_v3 reads own levels up to d_pyr + pyr_bytes
    h->cand_slots = h->geom.candTotal + 64;
    h->kp_slots = h->geom.kpTotal + 64;
    h->sort_slots = h->geom.sortTotal + 64;
    h->taps_slots = h->taps_host.size() + 4 * (cfg->max_width + cfg->max_height) + 64;
    h->cells_slots = h->geom.totalCells;   // monotone in the image's width and height
    h->out_rows = (size_t)h->kp_slots * B;
    // the quadtree node workspace depends on the quotas only: in shared memory when it fits, else one block per (image, level)
    for (int l = 0; l < cfg->n_levels; ++l) h->qt_node_cap = std::max(h->qt_node_cap, qt_node_cap(h->quota[l]));
    h->qt_nodes_in_smem = qt_node_bytes(h) <= 96 * 1024 ? 1 : 0;
    h->qt_node_stride = (qt_node_bytes(h) + 255) / 256 * 256;
    uint32_t frag[256], pat_w[256];
    orbdev::bm_fragments(frag);
    {   // the rBRIEF pattern as 256 packed words (xa, ya, xb, yb), transposed to [pair % 8][pair / 8] for k_orient_describe
        static const int8_t pat[1024] = {
#include "orb_pattern.inc"
        };
        for (int i = 0; i < 256; ++i)
            pat_w[(i & 7) * 32 + (i >> 3)] = (uint32_t)(uint8_t)pat[4 * i] | ((uint32_t)(uint8_t)pat[4 * i + 1] << 8) |
                                             ((uint32_t)(uint8_t)pat[4 * i + 2] << 16) | ((uint32_t)(uint8_t)pat[4 * i + 3] << 24);
    }
    auto layout = [&](Carve& c) {
        h->d_pyr = c.take<uint8_t>(h->pyr_bytes);
        h->d_blur = c.take<uint8_t>(h->pyr_bytes);
        h->d_cand = c.take<uint32_t>(h->cand_slots * B);
        h->d_sort = c.take<uint32_t>(h->sort_slots * B);
        h->d_lvl_kp = c.take<uint32_t>(h->kp_slots * B);
        h->d_slot = c.take<int>(h->kp_slots * B);
        h->d_cand_cnt = c.take<int>((size_t)B * ORB_MAX_LEVELS);
        h->d_lvl_cnt = c.take<int>((size_t)B * ORB_MAX_LEVELS);
        h->d_nkp = c.take<int>(3 * B + 8);
        h->d_err = c.take<int>(8);
        h->d_taps = c.take<int2>(h->taps_slots);
        h->d_kps = c.take<orbx_keypoint>(h->out_rows);
        h->d_desc = c.take<uint8_t>(h->out_rows * 32);
        h->d_uright = c.take<float>(h->out_rows);
        h->d_depth = c.take<float>(h->out_rows);
        h->d_sad = c.take<int>(h->out_rows);
        h->d_pat = stage_in(c, pat_w, 256, false);
        h->d_blur_frag = stage_in(c, frag, 256, false);
        h->d_cells = c.take<uint2>(h->cells_slots);
        if (!h->qt_nodes_in_smem) h->d_node_scratch = c.take<uint8_t>(h->qt_node_stride * B * cfg->n_levels);
    };
    if ((s = carve_exact(h->d_ws, h->stream, layout).status) != ORB_OK) return fail(s);
    h->d_mono = h->d_nkp + B;
    h->d_offsets = h->d_nkp + 2 * B;
    cudaMemsetAsync(h->d_err, 0, sizeof(int) * 8, h->stream);
    cudaMemsetAsync(h->d_pyr, 0, h->pyr_bytes, h->stream);
    cudaMemsetAsync(h->d_blur, 0, h->pyr_bytes, h->stream);
    if (cudaMallocHost((void**)&h->h_counts, sizeof(int) * (3 * B + 16)) != cudaSuccess)
        return fail(set_error(ORB_ERR_CUDA, "cudaMallocHost failed"));
    s = apply_geometry(h, cfg->max_width, cfg->max_height);
    if (s != ORB_OK) return fail(s);
    *out = h;
    return ORB_OK;
}

extern "C" void orbx_destroy(orbx_handle* h) {
    if (!h) return;
    cudaSetDevice(h->cfg.device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    orbr_release(h);
    for (void* p : {h->d_ws, h->d_stage, h->d_po, h->d_xl, h->d_src, h->d_dmap})
        if (p) cudaFree(p);
    if (h->h_counts) cudaFreeHost(h->h_counts);
    for (int r = 0; r < orbx_handle::kProfRing; ++r)
        for (int i = 0; i < 8; ++i)
            if (h->evr[r][i]) cudaEventDestroy(h->evr[r][i]);
    for (int i = 0; i < 3; ++i) {
        if (h->aux_stream[i]) cudaStreamDestroy(h->aux_stream[i]);
        if (h->ev_join[i]) cudaEventDestroy(h->ev_join[i]);
    }
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

extern "C" orb_status orbx_get_tables(const orbx_handle* h, float* scale, float* inv_scale, float* sigma2,
                                      float* inv_sigma2, int32_t* fpl, int32_t* umax16) {
    if (!h) return set_error(ORB_ERR_INVALID, "null handle");
    const int nl = h->cfg.n_levels;
    for (int i = 0; i < nl; ++i) {
        if (scale) scale[i] = h->scale[i];
        if (inv_scale) inv_scale[i] = h->inv_scale[i];
        if (sigma2) sigma2[i] = h->sigma2[i];
        if (inv_sigma2) inv_sigma2[i] = h->inv_sigma2[i];
        if (fpl) fpl[i] = h->quota[i];
    }
    if (umax16)
        for (int i = 0; i < 16; ++i) umax16[i] = h->umax[i];
    return ORB_OK;
}

// the kernel sequence of one batch; level 0 must already be in place (or aliased)
static orb_status run_pipeline(orbx_handle* h, int batch, int lap0, int lap1) {
    const ExtractGeom& g = h->geom;
    cudaStream_t st = h->stream;
    const bool prof = h->profiling;
    if (prof) cudaEventRecord(h->ev[1], st);
    ORB_CUDA(cudaMemsetAsync(h->d_cand_cnt, 0, sizeof(int) * batch * g.nlevels, st));
    for (int l = 1; l < g.nlevels; ++l) {
        if (h->resize_variant == 3 && !g.lv[l].area2x) {   // as variant 1, source rows by word loads + PRMT + IDP.2A
            const LevelGeom& S = g.lv[l - 1];
            const uint8_t* src_end = S.base + (int64_t)(batch - 1) * S.img_stride + (int64_t)(S.h - 1) * S.pitch + S.w;   // a caller-owned level 0 ends here
            if (S.base >= h->d_pyr && S.base < h->d_pyr + h->pyr_bytes) src_end = h->d_pyr + h->pyr_bytes;               // own levels: the allocation has slack
            dim3 grid((g.lv[l].w + 127) / 128, (g.lv[l].h + 31) / 32, batch);
            k_resize_v3<<<grid, 256, 0, st>>>(g, l, h->d_taps, src_end);
        } else if (h->resize_variant >= 1 && !g.lv[l].area2x) {   // 4 px x 4 (or 8) rows per thread, source-row interpolations shared between rows
            const int rows = h->resize_variant == 2 ? 8 : 4;
            dim3 grid((g.lv[l].w + 127) / 128, (g.lv[l].h + 8 * rows - 1) / (8 * rows), batch);
            if (rows == 8) k_resize_v2<8><<<grid, 256, 0, st>>>(g, l, h->d_taps);
            else k_resize_v2<4><<<grid, 256, 0, st>>>(g, l, h->d_taps);
        } else {
            dim3 grid((g.lv[l].w + 127) / 128, (g.lv[l].h + 7) / 8, batch), block(32, 8);
            k_resize<<<grid, block, 0, st>>>(g, l, h->d_taps);
        }
        ORB_LAUNCHED();
    }
    if (prof) cudaEventRecord(h->ev[2], st);
    if (h->fast_variant == 1) {   // pe / po rows, the byte score map, one list of pixel pairs per warp
        FastPlan fp;
        fp.cells = h->d_cells; fp.nCells = (int)h->cells_host.size(); fp.R = h->fast_R; fp.PW = h->fast_PW; fp.LW = h->fast_LW;
        const int ws = ((fp.PW - 1) >> 1) | 1;
        const size_t fsm = (size_t)round_up(fp.R * fp.PW, 4) * 8 + (size_t)round_up(fp.R * ws * 4, 16) + (size_t)2 * (FAST2_THREADS / 32) * fp.LW * 2;
        // ORB_FAST_TMA=1: the window rows by TMA bulk copies -- needs 64-byte rows to cover the staged columns (PW == 29: the 35-37 px
        // cells of the usual geometries) and 16-byte aligned level images (own levels always; an aliased level 0 is checked here)
        bool tma = h->fast_tma && fp.PW == 29;
        for (int l = 0; l < g.nlevels && tma; ++l)
            tma = (g.lv[l].pitch % 16 == 0) && (g.lv[l].img_stride % 16 == 0) && ((uintptr_t)g.lv[l].base % 16 == 0);
        if (tma) {
            const size_t fsmT = fsm + (size_t)fp.R * 64;
            ORB_CUDA(cudaFuncSetAttribute(k_fast_cells_v2<29, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmT));
            if (fp.nCells > 0) k_fast_cells_v2<29, true><<<dim3(fp.nCells, batch), FAST2_THREADS, fsmT, st>>>(g, fp, h->d_cand, h->d_cand_cnt, h->d_err);
        } else {
            auto kern = fp.PW == 29 ? k_fast_cells_v2<29> : k_fast_cells_v2<0>;
            ORB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsm));
            if (fp.nCells > 0) kern<<<dim3(fp.nCells, batch), FAST2_THREADS, fsm, st>>>(g, fp, h->d_cand, h->d_cand_cnt, h->d_err);
        }
    } else {   // pe / po / se rows + the NMS tile (which also holds the list of pixel pairs that pass the high-speed test)
        const size_t fsm = (size_t)g.fastRows * (3 * FAST_PW + FAST_TW) * 4;
        ORB_CUDA(cudaFuncSetAttribute(k_fast_cells, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsm));
        k_fast_cells<<<dim3(g.totalCells, batch), FAST_THREADS, fsm, st>>>(g, h->d_cand, h->d_cand_cnt, h->d_err);
    }
    ORB_LAUNCHED();
    if (prof) cudaEventRecord(h->ev[3], st);
    // DistributeOctTree: level groups on parallel streams (fork from / join into the handle's stream)
    cudaEventRecord(h->ev_fork, st);
    for (int gi = 0; gi < h->qt_ngroups; ++gi) {
        const orbx_handle::QtGroup& Q = h->qt_groups[gi];
        cudaStream_t qs = gi == 0 ? st : h->aux_stream[gi - 1];
        if (gi > 0) cudaStreamWaitEvent(qs, h->ev_fork, 0);
        // 1024 threads per CTA for the group with level 0 and, after a 64-bit group, for the first 32-bit group (the largest levels of
        // each form).  The 64-bit group always holds level 0.
        const bool wide = h->qt_variant == 1 && (gi == 0 || (gi == 1 && h->qt_groups[0].k64));
        launch_p(Q.k64 ? k_quadtree_v1_k64<QT_K64_THREADS, 1>
                       : h->qt_variant == 0 ? k_quadtree : wide ? k_quadtree_v1<1024, 1> : k_quadtree_v1<QT_THREADS, 4>,
                 dim3(batch * (Q.level_end - Q.level_begin)), dim3(Q.k64 ? QT_K64_THREADS : wide ? 1024 : QT_THREADS), Q.smem, qs,
                 g, batch, Q.level_begin, h->d_cand, h->d_cand_cnt, h->d_sort, (char*)h->d_node_scratch,
                 (int64_t)h->qt_node_stride, Q.sort_cap, h->qt_nodes_in_smem, h->qt_node_cap, h->d_lvl_kp, h->d_lvl_cnt, h->d_err);
        ORB_LAUNCHED();
        if (gi > 0) {
            cudaEventRecord(h->ev_join[gi - 1], qs);
            cudaStreamWaitEvent(st, h->ev_join[gi - 1], 0);
        }
    }
    launch_p(k_order, dim3(batch), dim3(256), h->order_smem_bytes, st, g, h->d_lvl_kp, h->d_lvl_cnt, lap0, lap1, h->d_slot, h->d_nkp, h->d_mono);
    ORB_LAUNCHED();
    launch_p(k_offsets, dim3(1), dim3(32), 0, st, h->d_nkp, batch, h->d_offsets);
    ORB_LAUNCHED();
    if (prof) cudaEventRecord(h->ev[4], st);
    if (h->blur_variant == 2) {   // both passes on the tensor cores (blur_mma.cuh), 128 x 96 tiles
        BlurMmaPlan bp;
        bp.frag = h->d_blur_frag;
        int tiles = 0;
        for (int l = 0; l < g.nlevels; ++l) {
            bp.tileBase[l] = tiles;
            bp.tilesX[l] = (g.lv[l].w + BM_TW - 1) / BM_TW;
            tiles += bp.tilesX[l] * ((g.lv[l].h + BM_TH - 1) / BM_TH);
        }
        bp.tileBase[g.nlevels] = tiles;
        k_blur_mma<<<dim3(tiles, batch), 256, 0, st>>>(g, bp);
    } else if (h->blur_variant == 1) k_blur<true><<<dim3(g.totalTiles, batch), 256, 0, st>>>(g);    // horizontal pass by IDP.4A
    else k_blur<false><<<dim3(g.totalTiles, batch), 256, 0, st>>>(g);
    ORB_LAUNCHED();
    if (prof) cudaEventRecord(h->ev[5], st);
    k_orient_describe<<<dim3((g.kpTotal + OD_WARPS - 1) / OD_WARPS, batch), OD_WARPS * 32, 0, st>>>(
        g, h->d_lvl_kp, h->d_lvl_cnt, h->d_slot, h->d_offsets, h->d_pat, h->d_kps, h->d_desc);
    ORB_LAUNCHED();
    if (prof) cudaEventRecord(h->ev[6], st);
    ORB_CUDA(cudaGetLastError());
    h->last_batch = batch;
    h->counts_valid = false;
    h->stereo_valid = false;
    return ORB_OK;
}

static orb_status check_batch_args(orbx_handle* h, const void* imgs, int batch, int w, int hh, int stride) {
    if (!h) return set_error(ORB_ERR_INVALID, "null handle");
    if (!imgs || w <= 0 || hh <= 0) return set_error(ORB_ERR_EMPTY, "empty image");
    if (batch < 1 || batch > h->cfg.max_batch || stride < w) return set_error(ORB_ERR_INVALID, "bad batch/stride");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    return apply_geometry(h, w, hh);
}

// The profiling ring: the next slot's stage events, the batch's first one recorded now
static void profile_batch(orbx_handle* h) {
    if (!h->profiling) return;
    h->ev = h->evr[h->prof_count % orbx_handle::kProfRing];
    ++h->prof_count;
    cudaEventRecord(h->ev[0], h->stream);
}

// Level 0 of w x hh images in the handle's own pyramid block, rows padded to 16 bytes
static const LevelGeom& own_level0(orbx_handle* h, int w, int hh) {
    LevelGeom& L0 = h->geom.lv[0];
    L0.base = h->d_pyr;
    L0.pitch = round_up(w, 16);
    L0.img_stride = (int64_t)L0.pitch * hh;
    return L0;
}

orb_status copy_images(orbx_handle* h, uint8_t* dst, size_t dst_pitch, const uint8_t* src, size_t src_pitch, size_t src_image, size_t row,
                       int rows, int batch, cudaMemcpyKind kind) {
    if (src_image == src_pitch * rows)
        ORB_CUDA(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, row, (size_t)rows * batch, kind, h->stream));
    else
        for (int b = 0; b < batch; ++b)
            ORB_CUDA(cudaMemcpy2DAsync(dst + b * dst_pitch * rows, dst_pitch, src + b * src_image, src_pitch, row, rows, kind, h->stream));
    return ORB_OK;
}

extern "C" orb_status orbx_extract_batch_device(orbx_handle* h, const uint8_t* d_imgs, int32_t batch, int32_t w,
                                                int32_t hh, int32_t stride, size_t image_stride_bytes, int32_t lap0,
                                                int32_t lap1) {
    orb_status s = check_batch_args(h, d_imgs, batch, w, hh, stride);
    if (s != ORB_OK) return s;
    profile_batch(h);
    const bool aligned = ((uintptr_t)d_imgs % 16 == 0) && (stride % 8 == 0) && (image_stride_bytes % 8 == 0);   // k_fast_cells_v2 stages with 64-bit loads
    if (aligned) {
        LevelGeom& L0 = h->geom.lv[0];
        L0.base = const_cast<uint8_t*>(d_imgs);
        L0.pitch = stride;
        L0.img_stride = (int64_t)image_stride_bytes;
    } else {
        const LevelGeom& L0 = own_level0(h, w, hh);
        s = copy_images(h, L0.base, L0.pitch, d_imgs, stride, image_stride_bytes, w, hh, batch, cudaMemcpyDeviceToDevice);
        if (s != ORB_OK) return s;
    }
    return run_pipeline(h, batch, lap0, lap1);
}

// ---- camera images of any format and size (k_ingest) ----------------------------------------------------------------------------
static int format_channels(int format) { return format == ORB_FORMAT_GRAY ? 1 : format <= ORB_FORMAT_BGR ? 3 : 4; }

namespace orb {

// colour conversion and resize of a batch of camera images into level 0 (resize_core.cuh ig_pixels4).  256 threads cover 1024 px x
// 1 row; blockIdx.z is the image.
__global__ void __launch_bounds__(256) k_ingest(const __grid_constant__ orbdev::IngestPlan P) {
    const int dx4 = 4 * (blockIdx.x * 256 + threadIdx.x), dy = blockIdx.y;
    if (dx4 >= P.dw) return;
    const uint32_t v = orbdev::ig_pixels4(P, P.src + (int64_t)blockIdx.z * P.src_image, dx4, dy);
    *reinterpret_cast<uint32_t*>(P.dst + (int64_t)blockIdx.z * P.dst_image + (int64_t)dy * P.dpitch + dx4) = v;
}

}  // namespace orb

orb_status check_source(ImageSource& src, int w, int hh) {
    if (src.format < ORB_FORMAT_GRAY || src.format > ORB_FORMAT_BGRA) return set_error(ORB_ERR_INVALID, "unknown image format");
    if (src.w == 0 && src.h == 0) { src.w = w; src.h = hh; }
    const int64_t row = (int64_t)src.w * format_channels(src.format);
    if (src.stride == 0) src.stride = row;
    if (src.image_stride == 0) src.image_stride = (size_t)src.stride * src.h;
    if (src.w < 1 || src.h < 1 || src.stride < row || src.stride > INT32_MAX) return set_error(ORB_ERR_INVALID, "bad source size or stride");
    return ORB_OK;
}

extern "C" orb_status orbx_extract_batch_device_format(orbx_handle* h, const uint8_t* d_imgs, int32_t batch, int32_t w, int32_t hh,
                                                       int32_t stride, size_t image_stride_bytes, int32_t lap0, int32_t lap1,
                                                       int32_t format, int32_t src_width, int32_t src_height) {
    ImageSource src{format, src_width, src_height, stride, image_stride_bytes};
    if (!h) return set_error(ORB_ERR_INVALID, "null handle");
    orb_status s = check_source(src, w, hh);
    if (s == ORB_OK) s = check_batch_args(h, d_imgs, batch, w, hh, w);
    if (s != ORB_OK) return s;
    const LevelGeom& L0 = own_level0(h, w, hh);
    profile_batch(h);
    const orbdev::IngestPlan P = orbdev::ig_plan(d_imgs, (int64_t)src.image_stride, format, src.w, src.h, (int)src.stride, L0.base, L0.img_stride,
                                                 w, hh, L0.pitch);
    k_ingest<<<dim3((P.dw + 1023) / 1024, P.dh, batch), 256, 0, h->stream>>>(P);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(ORB_ERR_CUDA, std::string("k_ingest: ") + cudaGetErrorString(e));
    ORB_LAUNCHED();
    return run_pipeline(h, batch, lap0, lap1);
}

orb_status extract_batch_source(orbx_handle* h, const uint8_t* imgs, int batch, int w, int hh, const ImageSource& src, int lap0, int lap1) {
    if (!imgs || batch < 1 || batch > h->cfg.max_batch) return set_error(ORB_ERR_INVALID, "bad batch");
    if (w < 1 || hh < 1 || w > h->cfg.max_width || hh > h->cfg.max_height)
        return set_error(ORB_ERR_INVALID, "image larger than the handle's max_width/max_height");
    const size_t row = (size_t)src.w * format_channels(src.format), img = row * src.h;
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    orb_status s = grow_device(h->src_bytes, h->d_src, img * batch, h->capturing);
    if (s == ORB_OK) s = copy_images(h, h->d_src, row, imgs, src.stride, src.image_stride, row, src.h, batch, cudaMemcpyHostToDevice);
    if (s != ORB_OK) return s;
    return orbx_extract_batch_device_format(h, h->d_src, batch, w, hh, (int)row, img, lap0, lap1, src.format, src.w, src.h);
}

extern "C" orb_status orbx_extract_batch(orbx_handle* h, const uint8_t* imgs, int32_t batch, int32_t w, int32_t hh,
                                         int32_t stride, size_t image_stride_bytes, int32_t lap0, int32_t lap1,
                                         int32_t* n_out, int32_t* mono_index) {
    orb_status s = check_batch_args(h, imgs, batch, w, hh, stride);
    if (s != ORB_OK) return s;
    const LevelGeom& L0 = own_level0(h, w, hh);
    profile_batch(h);
    s = copy_images(h, L0.base, L0.pitch, imgs, stride, image_stride_bytes, w, hh, batch, cudaMemcpyHostToDevice);
    if (s == ORB_OK) s = run_pipeline(h, batch, lap0, lap1);
    if (s != ORB_OK) return s;
    if (n_out || mono_index) {
        s = orbx_counts(h, n_out, mono_index, nullptr);
    }
    return s;
}

// ---- the batch count table ------------------------------------------------------------------------------------------------
// d_nkp holds [max_batch] features per image (k_order), [max_batch] mono indices (k_order) and [max_batch + 1] first rows
// (k_offsets).  h_counts mirrors those words, then holds the first four words of d_err at 3 max_batch + 4: [0] FAST candidate
// overflow, [1] quadtree node overflow.
orb_status queue_counts(orbx_handle* h) {
    const int MB = h->cfg.max_batch;
    ORB_CUDA(cudaMemcpyAsync(h->h_counts, h->d_nkp, sizeof(int) * (3 * MB + 1), cudaMemcpyDeviceToHost, h->stream));
    ORB_CUDA(cudaMemcpyAsync(h->h_counts + 3 * MB + 4, h->d_err, sizeof(int) * 4, cudaMemcpyDeviceToHost, h->stream));
    return ORB_OK;
}

orb_status latch_counts(orbx_handle* h) {
    if (!h->counts_valid) {
        h->counts_valid = true;
        const int* e = h->h_counts + 3 * h->cfg.max_batch + 4;
        h->batch_status = (e[0] || e[1]) ? (e[0] ? 1 : 2) : 0;   // latched until the next extract: every accessor keeps reporting it
        if (h->batch_status) cudaMemsetAsync(h->d_err, 0, sizeof(int) * 8, h->stream);
    }
    if (h->batch_status)
        return set_error(ORB_ERR_CAPACITY, h->batch_status == 1 ? "FAST candidate capacity exceeded" : "quadtree node capacity exceeded");
    return ORB_OK;
}

extern "C" orb_status orbx_counts(orbx_handle* h, int32_t* n, int32_t* mono_index, int32_t* offsets) {
    if (!h || h->last_batch < 1) return set_error(ORB_ERR_INVALID, "no batch has been extracted");
    const int B = h->last_batch, MB = h->cfg.max_batch;
    if (!h->counts_valid) {
        orb_status s = queue_counts(h);
        if (s != ORB_OK) return s;
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    }
    const orb_status s = latch_counts(h);
    if (s != ORB_OK) return s;
    for (int b = 0; b < B; ++b) {
        if (n) n[b] = image_features(h, b);
        if (mono_index) mono_index[b] = h->h_counts[MB + b];
        if (offsets) offsets[b] = image_row0(h, b);
    }
    if (offsets) offsets[B] = image_row0(h, B);
    return ORB_OK;
}

orb_status batch_rows(orbx_handle* h, int* rows) {
    const orb_status s = orbx_counts(h, nullptr, nullptr, nullptr);
    if (s == ORB_OK) *rows = batch_total_rows(h);
    return s;
}

extern "C" orb_status orbx_download(orbx_handle* h, orbx_keypoint* kps, uint8_t* desc, int32_t cap_rows) {
    int total = 0;
    orb_status s = batch_rows(h, &total);
    if (s != ORB_OK) return s;
    const int rows = std::min(total, (int)cap_rows);
    if (rows > 0) {
        if (kps) ORB_CUDA(cudaMemcpyAsync(kps, h->d_kps, sizeof(orbx_keypoint) * (size_t)rows, cudaMemcpyDeviceToHost, h->stream));
        if (desc) ORB_CUDA(cudaMemcpyAsync(desc, h->d_desc, 32 * (size_t)rows, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    }
    return total > cap_rows ? set_error(ORB_ERR_CAPACITY, "output buffer smaller than the batch result") : ORB_OK;
}

extern "C" orb_status orbx_extract(orbx_handle* h, const uint8_t* img, int32_t w, int32_t hh, int32_t stride,
                                   int32_t lap0, int32_t lap1, orbx_keypoint* kps, uint8_t* desc, int32_t cap,
                                   int32_t* n_out, int32_t* mono_index) {
    if (n_out) *n_out = 0;
    if (mono_index) *mono_index = -1;
    int n = 0, mono = 0;
    orb_status s = orbx_extract_batch(h, img, 1, w, hh, stride, (size_t)stride * hh, lap0, lap1, &n, &mono);
    if (s != ORB_OK) return s;
    if (n_out) *n_out = n;
    if (mono_index) *mono_index = mono;
    s = orbx_download(h, kps, desc, cap);
    return s;
}

extern "C" orb_status orbx_level_size(const orbx_handle* h, int32_t level, int32_t* w, int32_t* hh) {
    if (!h || level < 0 || level >= h->cfg.n_levels || h->cur_w < 0) return set_error(ORB_ERR_INVALID, "bad level");
    if (w) *w = h->geom.lv[level].w;
    if (hh) *hh = h->geom.lv[level].h;
    return ORB_OK;
}

extern "C" orb_status orbx_download_level(orbx_handle* h, int32_t b, int32_t level, int32_t blurred, uint8_t* dst,
                                          int32_t dst_stride) {
    if (!h || !dst || level < 0 || level >= h->cfg.n_levels || b < 0 || b >= h->last_batch)
        return set_error(ORB_ERR_INVALID, "bad level/batch index");
    const LevelGeom& L = h->geom.lv[level];
    const uint8_t* src = blurred ? L.blur + (int64_t)b * L.blur_stride : L.base + (int64_t)b * L.img_stride;
    ORB_CUDA(cudaMemcpy2DAsync(dst, dst_stride, src, blurred ? L.blur_pitch : L.pitch, L.w, L.h, cudaMemcpyDeviceToHost, h->stream));
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    return ORB_OK;
}

// ---- CUDA-graph capture of whatever the caller queues on the handle's stream between begin and end ----------------------
struct orbx_graph {
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    int kernels = 0;
};

extern "C" orb_status orbx_graph_begin(orbx_handle* h) {
    if (!h || h->capturing) return set_error(ORB_ERR_INVALID, "null handle or capture already open");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    if (h->profiling) return set_error(ORB_ERR_INVALID, "switch profiling off before capturing");
    ORB_CUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    h->capturing = true;
    return ORB_OK;
}

extern "C" orb_status orbx_graph_end(orbx_handle* h, orbx_graph** out) {
    if (!h || !out || !h->capturing) return set_error(ORB_ERR_INVALID, "no capture is open on this handle");
    h->capturing = false;
    orbx_graph* g = new orbx_graph();
    cudaError_t e = cudaStreamEndCapture(h->stream, &g->graph);
    if (e != cudaSuccess || !g->graph) {
        delete g;
        cudaGetLastError();
        return set_error(ORB_ERR_CUDA, "cudaStreamEndCapture failed (a captured call synchronised or allocated)");
    }
    size_t n = 0;
    cudaGraphGetNodes(g->graph, nullptr, &n);
    std::vector<cudaGraphNode_t> nodes(n);
    if (n) cudaGraphGetNodes(g->graph, nodes.data(), &n);
    for (size_t i = 0; i < n; ++i) {
        cudaGraphNodeType t;
        if (cudaGraphNodeGetType(nodes[i], &t) == cudaSuccess && t == cudaGraphNodeTypeKernel) ++g->kernels;
    }
    e = cudaGraphInstantiate(&g->exec, g->graph, 0);
    if (e != cudaSuccess) {
        cudaGraphDestroy(g->graph);
        delete g;
        return set_error(ORB_ERR_CUDA, "cudaGraphInstantiate failed");
    }
    *out = g;
    return ORB_OK;
}

extern "C" orb_status orbx_graph_launch(orbx_handle* h, orbx_graph* g) {
    if (!h || !g || !g->exec) return set_error(ORB_ERR_INVALID, "null handle or graph");
    ORB_CUDA(cudaGraphLaunch(g->exec, h->stream));
    g_launches += g->kernels;
    h->counts_valid = false;    // a replay produces new results
    return ORB_OK;
}

extern "C" int32_t orbx_graph_kernels(const orbx_graph* g) { return g ? g->kernels : 0; }

extern "C" void orbx_graph_destroy(orbx_graph* g) {
    if (!g) return;
    if (g->exec) cudaGraphExecDestroy(g->exec);
    if (g->graph) cudaGraphDestroy(g->graph);
    delete g;
}

extern "C" orb_status orbx_download_pyramid(orbx_handle* h, int32_t b, int32_t blurred, uint8_t* const* dst, const int32_t* dst_stride) {
    if (!h || !dst || !dst_stride || b < 0 || b >= h->last_batch) return set_error(ORB_ERR_INVALID, "bad batch index / null arrays");
    for (int l = 0; l < h->cfg.n_levels; ++l) {
        const LevelGeom& L = h->geom.lv[l];
        if (!dst[l] || dst_stride[l] < L.w) return set_error(ORB_ERR_INVALID, "bad destination for a pyramid level");
        const uint8_t* src = blurred ? L.blur + (int64_t)b * L.blur_stride : L.base + (int64_t)b * L.img_stride;
        ORB_CUDA(cudaMemcpy2DAsync(dst[l], dst_stride[l], src, blurred ? L.blur_pitch : L.pitch, L.w, L.h, cudaMemcpyDeviceToHost, h->stream));
    }
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    return ORB_OK;
}

extern "C" orb_status orbx_download_candidates(orbx_handle* h, int32_t b, int32_t level, int32_t* xys, int32_t cap,
                                               int32_t* n_out) {
    if (!h || !n_out || level < 0 || level >= h->cfg.n_levels || b < 0 || b >= h->last_batch)
        return set_error(ORB_ERR_INVALID, "bad level/batch index");
    const ExtractGeom& g = h->geom;
    const LevelGeom& L = g.lv[level];
    int n = 0;
    ORB_CUDA(cudaMemcpyAsync(&n, h->d_cand_cnt + b * g.nlevels + level, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    n = std::min(n, L.candCap);
    std::vector<uint32_t> raw(n);
    if (n)
        ORB_CUDA(cudaMemcpy(raw.data(), h->d_cand + (size_t)b * g.candTotal + L.candOff, 4 * (size_t)n, cudaMemcpyDeviceToHost));
    // reference order: cell row, cell column, then row-major inside the cell
    std::vector<std::pair<uint64_t, uint32_t>> v(n);
    for (int i = 0; i < n; ++i) {
        const int x = raw[i] & 0xfff, y = (raw[i] >> 12) & 0xfff;
        const uint64_t key = ((uint64_t)(((y - 3) / L.hCell) * L.nCols + (x - 3) / L.wCell) << 24) | ((uint64_t)y << 12) | x;
        v[i] = {key, raw[i]};
    }
    std::sort(v.begin(), v.end());
    *n_out = n;
    for (int i = 0; i < n && i < cap; ++i) {
        xys[3 * i] = v[i].second & 0xfff;
        xys[3 * i + 1] = (v[i].second >> 12) & 0xfff;
        xys[3 * i + 2] = v[i].second >> 24;
    }
    return ORB_OK;
}

extern "C" orb_status orbx_download_level_keypoints(orbx_handle* h, int32_t b, int32_t level, int32_t* xys, int32_t cap,
                                                    int32_t* n_out) {
    if (!h || !n_out || level < 0 || level >= h->cfg.n_levels || b < 0 || b >= h->last_batch)
        return set_error(ORB_ERR_INVALID, "bad level/batch index");
    const ExtractGeom& g = h->geom;
    const LevelGeom& L = g.lv[level];
    int n = 0;
    ORB_CUDA(cudaMemcpyAsync(&n, h->d_lvl_cnt + b * g.nlevels + level, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    std::vector<uint32_t> raw(std::max(n, 1));
    if (n)
        ORB_CUDA(cudaMemcpy(raw.data(), h->d_lvl_kp + (size_t)b * g.kpTotal + L.kpOff, 4 * (size_t)n, cudaMemcpyDeviceToHost));
    *n_out = n;
    for (int i = 0; i < n && i < cap; ++i) {
        xys[3 * i] = (raw[i] & 0xfff) + 16;
        xys[3 * i + 1] = ((raw[i] >> 12) & 0xfff) + 16;
        xys[3 * i + 2] = raw[i] >> 24;
    }
    return ORB_OK;
}

extern "C" orb_status orbx_set_profiling(orbx_handle* h, int32_t on) {
    if (!h) return set_error(ORB_ERR_INVALID, "null handle");
    h->profiling = on != 0;
    h->prof_count = 0;
    return ORB_OK;
}

// averages over the batches recorded since orbx_set_profiling (at most the last kProfRing)
extern "C" orb_status orbx_last_timings(orbx_handle* h, float* ms7) {
    if (!h || !ms7 || !h->profiling || h->prof_count < 1) return set_error(ORB_ERR_INVALID, "profiling is off or no batch ran");
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    const int n = std::min(h->prof_count, (int)orbx_handle::kProfRing);
    static const int a[7] = {0, 1, 2, 3, 4, 5, 0}, b[7] = {6, 2, 3, 4, 5, 6, 1};
    for (int k = 0; k < 7; ++k) ms7[k] = 0.f;
    for (int r = 0; r < n; ++r)
        for (int k = 0; k < 7; ++k) {
            float t = 0;
            cudaEventElapsedTime(&t, h->evr[r][a[k]], h->evr[r][b[k]]);
            ms7[k] += t / n;
        }
    return ORB_OK;
}

#if defined(QT_PROFILE)
// profile build only (tools/qt_phases.py): the quadtree phase clocks, summed over the CTAs since the last reset
extern "C" void orbx_debug_qt_profile(long long* out32, int reset) {
    cudaDeviceSynchronize();
    if (out32) cudaMemcpyFromSymbol(out32, orbdev::g_qt_prof, sizeof(long long) * 32);
    if (reset) {
        long long z[32] = {};
        cudaMemcpyToSymbol(orbdev::g_qt_prof, z, sizeof(z));
    }
}
#endif

extern "C" void* orbx_cuda_stream(orbx_handle* h) { return h ? (void*)h->stream : nullptr; }
