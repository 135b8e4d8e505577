// matcher_core.cuh -- the device code of the ORBmatcher searches (matcher.cu), written once for both places the searched frame's
// features can live:
//   * SmemFrame: each CTA stages the frame into its own shared memory (FrameFeat 23 B, GridFeat 17 B per feature).  The kernels
//     k_proj_candidates[_grp], k_proj_resolve_par and k_proj_resolve of matcher.cu.
//   * GlobalFrame: k_stage_frames_xl writes the same FrameFeat / GridFeat blocks once per frame into global scratch and the kernels
//     read them from there (L2-resident: ~650 KB per frame at 16 384 features); only the per-feature resolve state stays in shared
//     memory.  The *_xl kernels of matcher.cu.
// launch_proj (matcher.cu) runs the shared-memory form whenever a call's shared-memory need fits the device's opt-in limit.
#pragma once
#include "common.cuh"
#include "devmath.cuh"

namespace orb {
using namespace orbdev;

#define PM_K 8            // stored candidates per query
#define PM_WARPS 8
#define PM_QPB 64         // queries per CTA in the candidate kernel
#define GRID_COLS 64      // include/Frame.h:46-47
#define GRID_ROWS 48

struct FrameFeat {   // shared-memory staging of one frame's features
    float* x;
    float* y;
    float* ur;
    float* ang;
    uint16_t* cell;   // ix * 48 + iy, 0xffff = not in the grid (PosInGrid false)
    uint8_t* oct;
    int* node;        // mode 2: vocabulary node of the feature (F.mFeatVec), -1 = none
};

struct ProjParams {
    // frame side (an extractor handle's last batch)
    const orbx_keypoint* kps;
    const uint8_t* desc;
    const float* uright;      // null => monocular (mvuRight = -1)
    const int* offsets;
    const int* nkp;
    int maxFeat;
    float minX, maxX, minY, maxY, invW, invH;
    float fx, fy, cx, cy, bf;
    float scale[ORB_MAX_LEVELS];
    // query side
    int mode;                 // 0 = local map points, 1 = last frame, 2 = bag of words (same vocabulary node),
                              // 3 = projection into a keyframe, 4 = monocular initialisation (a0/a1 = vbPrevMatched, level = octave)
    const int* feat_node;     // mode 2: per compact feature row
    const int* frame_image;   // [n_frames]
    const int* qoff;          // [n_frames + 1]
    const float* a0;          // mode 0: projX      mode 1: world pos (3 per query)
    const float* a1;          // mode 0: projY
    const float* a2;          // mode 0: projXR
    const int* level;         // mode 0: predicted level   mode 1: last octave
    const float* f0;          // mode 0: viewCos    mode 1: last angle
    const float* f1;          // mode 0: trackDepth or null
    const uint8_t* qdesc;
    const uint8_t* flag;      // mode 0: initial claim mask per compact feature row (or null); mode 1: obs>0 per query
    const float* Tcw;         // mode 1: [n_frames][7] qx qy qz qw tx ty tz
    const int* direction;     // mode 1: [n_frames] 0 none, 1 forward, 2 backward
    float th, nnratio, thFar;
    int bFar, checkOri;
    // mode 3 (projection into a keyframe): a0 = world pos, f0 = query angle (variant 3), Tcw per target
    int variant;              // 0 Fuse(pose), 1 Fuse(Scw), 2 SearchByProjection(KF, Scw), 3 SearchByProjection(F, KF, set),
                              // 4 one direction of SearchBySim3
    const float* Ow;          // [n_frames][3]
    const float* S;           // variant 4: [n_frames][8] Sim3 quaternion (non-unit) x y z w, translation, scale
    const float* normal;      // [nq][3] MapPoint::GetNormal (variants 0-2)
    const float* maxD;        // mfMaxDistance (raw member)
    const float* minD;
    float logScale, thr;
    int nLevels;
    float invSigma2[ORB_MAX_LEVELS];
    // per-frame feature grid (Frame::mGrid as CSR), built by k_frame_grid for modes 0 / 1
    uint16_t* gridOrder;       // [n_frames][maxFeat] feature ids sorted by (cell, id)
    uint16_t* gridStart;       // [n_frames][GRID_COLS * GRID_ROWS + 1]
    // scratch + outputs
    unsigned long long* topk;  // [nq][PM_K]
    int* cnt;                  // [nq] candidates passing the order-free gates
    float* quv;                // mode 1: [nq][4] u, v, radius, invzc
    int* match;                // mode 0: [nq] feature index or -1;  mode 1: per compact feature row: query or -1
    int* nmatches;             // [n_frames]
    const uint8_t* qvalid;     // mode 0: mbTrackInView per query (Frame::isInFrustum), null = all
    int* seqFlag;              // [n_frames] modes 0 / 1: set by the parallel resolve when a frame must take the sequential kernel; null = always sequential
    int qpb;                   // queries per CTA of k_proj_candidates_grp
};

// the FrameFeat arrays of M features from `base` (frame_smem_bytes(M) bytes)
__device__ __forceinline__ void frame_view(unsigned char* base, size_t M, FrameFeat& F) {
    F.x = reinterpret_cast<float*>(base);
    F.y = F.x + M;
    F.ur = F.y + M;
    F.ang = F.ur + M;
    F.node = reinterpret_cast<int*>(F.ang + M);
    F.cell = reinterpret_cast<uint16_t*>(F.node + M);
    F.oct = reinterpret_cast<uint8_t*>(F.cell + M);
}

// the frame's features into FrameFeat at `smem` (shared memory, or a global block in k_stage_frames_xl), strided over the CTA
__device__ __forceinline__ void stage_frame(const ProjParams& P, int img, unsigned char* smem, FrameFeat& F, int& N, int& row0) {
    N = min(P.nkp[img], P.maxFeat);
    row0 = P.offsets[img];
    frame_view(smem, (size_t)P.maxFeat, F);
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        const orbx_keypoint k = P.kps[row0 + i];
        F.x[i] = k.x;
        F.y[i] = k.y;
        F.ur[i] = P.uright ? P.uright[row0 + i] : -1.0f;
        F.ang[i] = k.angle;
        F.node[i] = P.feat_node ? P.feat_node[row0 + i] : -1;
        // Frame::PosInGrid, Frame.cc:962-978 (C round(): half away from zero)
        const int px = (int)roundf(fmul(fsub(k.x, P.minX), P.invW)), py = (int)roundf(fmul(fsub(k.y, P.minY), P.invH));
        F.cell[i] = (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) ? (uint16_t)0xffff : (uint16_t)(px * GRID_ROWS + py);
        F.oct[i] = (uint8_t)k.octave;
    }
}

__device__ __forceinline__ size_t frame_smem_bytes(int maxFeat) { return (size_t)maxFeat * 23 + 16; }

struct Window {   // Frame::GetFeaturesInArea arguments resolved to cell ranges
    int node;         // >= 0: bag-of-words query, candidates = features of this vocabulary node (no window)
    float x, y, r;
    int c0, c1, r0, r1, minLevel, maxLevel;
    bool empty;
};

__device__ __forceinline__ Window make_window(const ProjParams& P, float x, float y, float r, int minLevel, int maxLevel) {
    Window w;
    w.node = -1;
    w.x = x; w.y = y; w.r = r; w.minLevel = minLevel; w.maxLevel = maxLevel;
    w.c0 = max(0, (int)floorf(fmul(fsub(fsub(x, P.minX), r), P.invW)));
    w.c1 = min(GRID_COLS - 1, (int)ceilf(fmul(fadd(fsub(x, P.minX), r), P.invW)));
    w.r0 = max(0, (int)floorf(fmul(fsub(fsub(y, P.minY), r), P.invH)));
    w.r1 = min(GRID_ROWS - 1, (int)ceilf(fmul(fadd(fsub(y, P.minY), r), P.invH)));
    w.empty = (w.c0 >= GRID_COLS) || (w.c1 < 0) || (w.r0 >= GRID_ROWS) || (w.r1 < 0);
    return w;
}

// is feature i a candidate of the window (all gates of GetFeaturesInArea)?
__device__ __forceinline__ bool in_window(const FrameFeat& F, const Window& w, int i) {
    if (w.node >= 0) return F.node[i] == w.node;
    const int cell = F.cell[i];
    if (cell == 0xffff) return false;
    const int ix = cell / GRID_ROWS, iy = cell - ix * GRID_ROWS;
    if (ix < w.c0 || ix > w.c1 || iy < w.r0 || iy > w.r1) return false;
    const int oc = F.oct[i];
    if ((w.minLevel > 0) || (w.maxLevel >= 0)) {
        if (oc < w.minLevel) return false;
        if (w.maxLevel >= 0 && oc > w.maxLevel) return false;
    }
    const float dx = fsub(F.x[i], w.x), dy = fsub(F.y[i], w.y);
    return fabsf(dx) < w.r && fabsf(dy) < w.r;
}

__device__ __forceinline__ uint32_t hamming256(const uint4& a0, const uint4& a1, const uint8_t* d) {
    const uint4* p = reinterpret_cast<const uint4*>(d);
    const uint4 b0 = __ldg(p), b1 = __ldg(p + 1);
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
        v = u < v ? u : v;
    }
    return v;
}

// Fuse's reprojection gate (ORBmatcher.cc:1465-1500): stereo keypoints 3-dof chi2 > 7.8, monocular 2-dof > 5.99
__device__ __forceinline__ bool fuse_chi2_ok(const ProjParams& P, float u, float v, float ur_pred, float kx, float ky, float kur, int oc) {
    const float ex = fsub(u, kx), ey = fsub(v, ky);
    if (kur >= 0) {
        const float er = fsub(ur_pred, kur);
        const float e2 = fadd(fadd(fmul(ex, ex), fmul(ey, ey)), fmul(er, er));
        return !((double)fmul(e2, P.invSigma2[oc]) > 7.8);
    }
    const float e2 = fadd(fmul(ex, ex), fmul(ey, ey));
    return !((double)fmul(e2, P.invSigma2[oc]) > 5.99);
}

// Candidate test shared by the two scans below: window / vocabulary node, optional claim mask, then the gate --
// gate 0: stereo window |ur_pred - mvuRight[i]| <= er_max when mvuRight[i] > 0 (modes 0 / 1); gate 1: none;
// gate 2: Fuse's reprojection chi2.
__device__ __forceinline__ bool scan_accepts(const ProjParams& P, const FrameFeat& F, const Window& w, int i, float ur_pred,
                                             float er_max, const uint8_t* claimed, int gate) {
    if (!in_window(F, w, i)) return false;
    if (claimed && claimed[i]) return false;
    const float ur = F.ur[i];
    if (gate == 0) {
        if (ur > 0) {
            const float er = fabsf(fsub(ur_pred, ur));
            if (er > er_max) return false;
        }
    } else if (gate == 2) {
        if (!fuse_chi2_ok(P, w.x, w.y, ur_pred, F.x[i], F.y[i], ur, F.oct[i])) return false;
    }
    return true;
}

// Bag-of-words scan of one query (mode 2): the candidates are the frame features of the query's vocabulary node in
// feature order, so (distance << 16 | id) in 32 bits is the reference order and the K smallest come out of K REDUX.MIN.
// Returns the number of candidates; out[k] = distance << 32 | id.
__device__ __forceinline__ int warp_scan_query(const ProjParams& P, const FrameFeat& F, int N, int row0, const Window& w,
                                               const uint8_t* qd, unsigned long long out[PM_K]) {
    const int lane = threadIdx.x & 31;
    uint32_t loc[PM_K];
#pragma unroll
    for (int k = 0; k < PM_K; ++k) loc[k] = 0xffffffffu;
    int count = 0;
    if (!w.empty) {
        const uint4* q4 = reinterpret_cast<const uint4*>(qd);
        const uint4 a0 = __ldg(q4), a1 = __ldg(q4 + 1);
        for (int base = 0; base < N; base += 32) {
            const int i = base + lane;
            if (i >= N || !scan_accepts(P, F, w, i, 0.f, 3.0e38f, nullptr, 1)) continue;
            ++count;
            uint32_t key = (hamming256(a0, a1, P.desc + (size_t)(row0 + i) * 32) << 16) | (uint32_t)i;
#pragma unroll
            for (int k = 0; k < PM_K; ++k)   // sorted insert
                if (key < loc[k]) {
                    const uint32_t t = loc[k];
                    loc[k] = key;
                    key = t;
                }
        }
    }
    count = __reduce_add_sync(0xffffffffu, count);
#pragma unroll
    for (int k = 0; k < PM_K; ++k) out[k] = ~0ull;
#pragma unroll
    for (int k = 0; k < PM_K; ++k) {
        const uint32_t m = __reduce_min_sync(0xffffffffu, loc[0]);
        if (m == 0xffffffffu) break;   // warp-uniform
        out[k] = ((unsigned long long)(m >> 16) << 32) | (unsigned long long)(m & 0xffffu);
        if (loc[0] == m) {             // ids are unique => exactly one owner
#pragma unroll
            for (int q = 0; q + 1 < PM_K; ++q) loc[q] = loc[q + 1];
            loc[PM_K - 1] = 0xffffffffu;
        }
    }
    return count;
}

// Exact rescan of one query with the claim mask applied (resolve slow path): only the best and the second best
// (distance, reference candidate order = cell, id) keys are needed.  Each lane keeps its own two smallest keys; the
// warp minimum is b1, the minimum of what remains is b2.
__device__ __forceinline__ void warp_rescan_best2(const ProjParams& P, const FrameFeat& F, int N, int row0, const Window& w,
                                                  const uint8_t* qd, float ur_pred, float er_max, const uint8_t* claimed, int gate,
                                                  unsigned long long& b1, unsigned long long& b2, const int* md = nullptr,
                                                  const int* claimMin = nullptr, int ql = 0) {
    const int lane = threadIdx.x & 31;
    unsigned long long l1 = ~0ull, l2 = ~0ull;
    if (!w.empty) {
        const uint4* q4 = reinterpret_cast<const uint4*>(qd);
        const uint4 a0 = __ldg(q4), a1 = __ldg(q4 + 1);
        for (int base = 0; base < N; base += 32) {
            const int i = base + lane;
            if (i >= N || !scan_accepts(P, F, w, i, ur_pred, er_max, claimed, gate)) continue;
            if (claimMin && claimMin[i] < ql) continue;   // parallel resolve: claimed by an earlier query
            const unsigned long long d = hamming256(a0, a1, P.desc + (size_t)(row0 + i) * 32);
            if (md && md[i] <= (int)d) continue;   // SearchForInitialization: vMatchedDistance[i2] <= dist
            const unsigned long long cell = w.node >= 0 ? 0ull : (unsigned long long)F.cell[i];
            const unsigned long long key = (d << 32) | (cell << 16) | (unsigned long long)i;
            if (key < l1) { l2 = l1; l1 = key; }
            else if (key < l2) l2 = key;
        }
    }
    b1 = warp_min_u64(l1);
    b2 = warp_min_u64(l1 == b1 ? l2 : l1);   // keys are unique (feature id in the low bits)
}

// mode 1 per-query geometry (ORBmatcher.cc:1985-2023): returns false when the query is skipped
__device__ __forceinline__ bool last_frame_window(const ProjParams& P, int frame, int q, Window& w, float& u, float& invzc,
                                                  float& radius) {
    const float* T = P.Tcw + 7 * frame;
    const float* p = P.a0 + 3 * (size_t)q;
    // Sophus::SE3f * Vector3f (so3.hpp:358-367): uv = qv x p; uv += uv; p' = p + w uv + qv x uv; + t
    const float qx = T[0], qy = T[1], qz = T[2], qw = T[3];
    const float uvx = fsub(fmul(qy, p[2]), fmul(qz, p[1])), uvy = fsub(fmul(qz, p[0]), fmul(qx, p[2])),
                uvz = fsub(fmul(qx, p[1]), fmul(qy, p[0]));
    const float ux = fadd(uvx, uvx), uy = fadd(uvy, uvy), uz = fadd(uvz, uvz);
    const float c0 = fsub(fmul(qy, uz), fmul(qz, uy)), c1 = fsub(fmul(qz, ux), fmul(qx, uz)), c2 = fsub(fmul(qx, uy), fmul(qy, ux));
    const float xc = fadd(fadd(fadd(p[0], fmul(qw, ux)), c0), T[4]);
    const float yc = fadd(fadd(fadd(p[1], fmul(qw, uy)), c1), T[5]);
    const float zc = fadd(fadd(fadd(p[2], fmul(qw, uz)), c2), T[6]);
    invzc = (float)(1.0 / (double)zc);
    if (invzc < 0) return false;
    u = fadd(fdiv(fmul(P.fx, xc), zc), P.cx);                 // Pinhole::project, Pinhole.cpp:61-68
    const float v = fadd(fdiv(fmul(P.fy, yc), zc), P.cy);
    if (u < P.minX || u > P.maxX) return false;
    if (v < P.minY || v > P.maxY) return false;
    const int oct = P.level[q];
    radius = fmul(P.th, P.scale[oct]);
    const int dir = P.direction[frame];
    if (dir == 1) w = make_window(P, u, v, radius, oct, -1);
    else if (dir == 2) w = make_window(P, u, v, radius, 0, oct);
    else w = make_window(P, u, v, radius, oct - 1, oct + 1);
    return true;
}

// mode 3 per-query geometry: projection of a map point into a keyframe from a pose, frustum / distance / viewing
// angle gates and MapPoint::PredictScale (MapPoint.cc:688-721, logf).  Vector3f norm and dot in Eigen's unrolled
// order x + (y + z).  ur_pred = u - bf / z (Fuse only).
__device__ __forceinline__ bool kf_window(const ProjParams& P, int frame, int q, Window& w, float& ur_pred) {
    const float* T = P.Tcw + 7 * frame;
    const float* p = P.a0 + 3 * (size_t)q;
    const float qx = T[0], qy = T[1], qz = T[2], qw = T[3];
    const float uvx = fsub(fmul(qy, p[2]), fmul(qz, p[1])), uvy = fsub(fmul(qz, p[0]), fmul(qx, p[2])),
                uvz = fsub(fmul(qx, p[1]), fmul(qy, p[0]));
    const float ux = fadd(uvx, uvx), uy = fadd(uvy, uvy), uz = fadd(uvz, uvz);
    const float c0 = fsub(fmul(qy, uz), fmul(qz, uy)), c1 = fsub(fmul(qz, ux), fmul(qx, uz)), c2 = fsub(fmul(qx, uy), fmul(qy, ux));
    const float xc = fadd(fadd(fadd(p[0], fmul(qw, ux)), c0), T[4]);
    const float yc = fadd(fadd(fadd(p[1], fmul(qw, uy)), c1), T[5]);
    float zc = fadd(fadd(fadd(p[2], fmul(qw, uz)), c2), T[6]);
    float u, v, invz, px, py, pz;
    if (P.variant == 4) {
        // p2 = S * p1 (Sophus rxso3.hpp:265-273, sim3.hpp:227-230): scale p + (w 2(v x p) + v x 2(v x p)) + t
        const float* S = P.S + 8 * frame;
        const float sx = S[0], sy = S[1], sz = S[2], sw = S[3], sc = S[7];
        const float ax = fsub(fmul(sy, zc), fmul(sz, yc)), ay = fsub(fmul(sz, xc), fmul(sx, zc)), az = fsub(fmul(sx, yc), fmul(sy, xc));
        const float bx = fadd(ax, ax), by = fadd(ay, ay), bz = fadd(az, az);
        const float d0 = fsub(fmul(sy, bz), fmul(sz, by)), d1 = fsub(fmul(sz, bx), fmul(sx, bz)), d2 = fsub(fmul(sx, by), fmul(sy, bx));
        px = fadd(fadd(fmul(sc, xc), fadd(fmul(sw, bx), d0)), S[4]);
        py = fadd(fadd(fmul(sc, yc), fadd(fmul(sw, by), d1)), S[5]);
        pz = fadd(fadd(fmul(sc, zc), fadd(fmul(sw, bz), d2)), S[6]);
        if ((double)pz < 0.0) return false;
        invz = (float)(1.0 / (double)pz);
        u = fadd(fmul(P.fx, fmul(px, invz)), P.cx);
        v = fadd(fmul(P.fy, fmul(py, invz)), P.cy);
    } else {
        if (P.variant != 3 && zc < 0.0f) return false;
        invz = fdiv(1.0f, zc);
        u = fadd(fdiv(fmul(P.fx, xc), zc), P.cx);
        v = fadd(fdiv(fmul(P.fy, yc), zc), P.cy);
        const float* O = P.Ow + 3 * frame;
        px = fsub(p[0], O[0]); py = fsub(p[1], O[1]); pz = fsub(p[2], O[2]);
    }
    if (P.variant == 3) {
        if (u < P.minX || u > P.maxX) return false;
        if (v < P.minY || v > P.maxY) return false;
    } else if (!(u >= P.minX && u < P.maxX && v >= P.minY && v < P.maxY)) return false;
    ur_pred = fsub(u, fmul(P.bf, invz));
    const float dist = fsqrt(fadd(fmul(px, px), fadd(fmul(py, py), fmul(pz, pz))));
    // GetMinDistanceInvariance / GetMaxDistanceInvariance (MapPoint.cc:658-672): 0.8f * mfMinDistance, 1.2f * mfMaxDistance; PredictScale
    // (MapPoint.cc:688-721) takes the RAW mfMaxDistance
    if (dist < fmul(0.8f, P.minD[q]) || dist > fmul(1.2f, P.maxD[q])) return false;
    if (P.variant < 3) {
        const float* n = P.normal + 3 * (size_t)q;
        const float d = fadd(fmul(px, n[0]), fadd(fmul(py, n[1]), fmul(pz, n[2])));
        if ((double)d < 0.5 * (double)dist) return false;
    }
    const float ratio = fdiv(P.maxD[q], dist);
    int lvl = (int)ceilf(fdiv(glibc_logf(ratio), P.logScale));
    if (lvl < 0) lvl = 0;
    else if (lvl >= P.nLevels) lvl = P.nLevels - 1;
    const float radius = fmul(P.th, P.scale[lvl]);
    w = make_window(P, u, v, radius, lvl - 1, P.variant == 3 ? lvl + 1 : lvl);
    return true;
}

__device__ __forceinline__ bool local_window(const ProjParams& P, int q, Window& w, float& er_max) {
    if (P.qvalid && !P.qvalid[q]) return false;                 // !pMP->mbTrackInView (ORBmatcher.cc:52-53)
    if (P.bFar && P.f1 && P.f1[q] > P.thFar) return false;
    const int lvl = P.level[q];
    float r = ((double)P.f0[q] > 0.998) ? 2.5f : 4.0f;        // RadiusByViewingCos, ORBmatcher.cc:242-248
    if (P.th != 1.0f) r = fmul(r, P.th);
    er_max = fmul(r, P.scale[lvl]);
    w = make_window(P, P.a0[q], P.a1[q], er_max, lvl - 1, lvl);
    return true;
}

#define PM_NCELL (GRID_COLS * GRID_ROWS)

struct GridFeat {   // a frame's features in (cell, id) order + the CSR cell table, in shared memory
    float* x;
    float* y;
    float* ur;
    uint16_t* cell;
    uint16_t* id;
    uint16_t* start;   // PM_NCELL + 1
    uint8_t* oct;
};

__device__ __forceinline__ size_t grid_smem_bytes(int maxFeat) { return (size_t)maxFeat * 17 + (PM_NCELL + 1) * 2 + 32; }

// the GridFeat arrays of M features from `base` (grid_smem_bytes(M) bytes)
__device__ __forceinline__ void grid_view(unsigned char* base, size_t M, GridFeat& F) {
    F.x = reinterpret_cast<float*>(base);
    F.y = F.x + M;
    F.ur = F.y + M;
    F.cell = reinterpret_cast<uint16_t*>(F.ur + M);
    F.id = F.cell + M;
    F.start = F.id + M;
    F.oct = reinterpret_cast<uint8_t*>(F.start + PM_NCELL + 2);
}

// the frame's features in grid order into GridFeat at `smem` (shared memory, or a global block in k_stage_frames_xl)
__device__ __forceinline__ void stage_grid(const ProjParams& P, int frame, unsigned char* smem, GridFeat& F, int& N, int& row0) {
    const int img = P.frame_image[frame];
    N = min(P.nkp[img], P.maxFeat);
    row0 = P.offsets[img];
    grid_view(smem, (size_t)P.maxFeat, F);
    const uint16_t* order = P.gridOrder + (size_t)frame * P.maxFeat;
    const uint16_t* start = P.gridStart + (size_t)frame * (PM_NCELL + 1);
    for (int j = threadIdx.x; j < N; j += blockDim.x) {
        const int i = order[j];
        const orbx_keypoint k = P.kps[row0 + i];
        F.x[j] = k.x;
        F.y[j] = k.y;
        F.ur[j] = P.uright ? P.uright[row0 + i] : -1.0f;
        const int px = (int)roundf(fmul(fsub(k.x, P.minX), P.invW)), py = (int)roundf(fmul(fsub(k.y, P.minY), P.invH));
        F.cell[j] = (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) ? (uint16_t)0xffff : (uint16_t)(px * GRID_ROWS + py);
        F.id[j] = (uint16_t)i;
        F.oct[j] = (uint8_t)k.octave;
    }
    for (int c = threadIdx.x; c <= PM_NCELL; c += blockDim.x) F.start[c] = start[c];
}

// Where a kernel body finds the searched frame.  frame() / grid() set the view (the caller synchronises the CTA before reading it);
// kShared: the view takes the front of the CTA's dynamic shared memory, and the body's own arrays start after it.
struct SmemFrame {   // staged into the CTA's shared memory
    static constexpr bool kShared = true;
    __device__ __forceinline__ void frame(const ProjParams& P, int img, int, unsigned char* smem, FrameFeat& F, int& N, int& row0) const {
        stage_frame(P, img, smem, F, N, row0);
    }
    __device__ __forceinline__ void grid(const ProjParams& P, int frame, unsigned char* smem, GridFeat& F, int& N, int& row0) const {
        stage_grid(P, frame, smem, F, N, row0);
    }
};

struct GlobalFrame {   // staged once per frame into global scratch by k_stage_frames_xl
    static constexpr bool kShared = false;
    unsigned char* featBlocks;   // [n_frames][featStride]: FrameFeat blocks
    unsigned char* gridBlocks;   // [n_frames][gridStride]: GridFeat blocks (modes 0, 1, 3, 4), null for mode 2
    size_t featStride, gridStride;
    __device__ __forceinline__ void frame(const ProjParams& P, int img, int frame, unsigned char*, FrameFeat& F, int& N, int& row0) const {
        N = min(P.nkp[img], P.maxFeat);
        row0 = P.offsets[img];
        frame_view(featBlocks + (size_t)frame * featStride, (size_t)P.maxFeat, F);
    }
    __device__ __forceinline__ void grid(const ProjParams& P, int frame, unsigned char*, GridFeat& F, int& N, int& row0) const {
        const int img = P.frame_image[frame];
        N = min(P.nkp[img], P.maxFeat);
        row0 = P.offsets[img];
        grid_view(gridBlocks + (size_t)frame * gridStride, (size_t)P.maxFeat, F);
    }
};

// GetFeaturesInArea over the CSR grid: only the cells of the window are visited (Frame.cc:905-947).
// Keys are 32 bits here -- distance << 16 | position in the (cell, id)-sorted feature order, which is the
// reference's candidate order -- so the warp-wide minimum is ONE instruction (REDUX.MIN) instead of a 64-bit
// shuffle tree; they are widened to the (distance, cell, id) form of the resolve pass when stored.
__device__ __forceinline__ int warp_scan_query_grid(const ProjParams& P, const GridFeat& F, int row0, const Window& w, const uint8_t* qd,
                                                    float ur_pred, float er_max, unsigned long long out[PM_K], int gate = 0) {
    const int lane = threadIdx.x & 31;
    uint32_t loc[PM_K];
#pragma unroll
    for (int k = 0; k < PM_K; ++k) loc[k] = 0xffffffffu;
    int count = 0;
    if (!w.empty) {
        const uint4* q4 = reinterpret_cast<const uint4*>(qd);
        const uint4 a0 = __ldg(q4), a1 = __ldg(q4 + 1);
        const bool checkLevels = (w.minLevel > 0) || (w.maxLevel >= 0);
        for (int ix = w.c0; ix <= w.c1; ++ix) {
            const int jb = F.start[ix * GRID_ROWS + w.r0], je = F.start[ix * GRID_ROWS + w.r1 + 1];
            for (int j = jb + lane; j < je; j += 32) {
                const int oc = F.oct[j];
                if (checkLevels) {
                    if (oc < w.minLevel) continue;
                    if (w.maxLevel >= 0 && oc > w.maxLevel) continue;
                }
                const float dx = fsub(F.x[j], w.x), dy = fsub(F.y[j], w.y);
                if (!(fabsf(dx) < w.r && fabsf(dy) < w.r)) continue;
                const float ur = F.ur[j];
                if (gate == 0) {
                    if (ur > 0) {
                        const float er = fabsf(fsub(ur_pred, ur));
                        if (er > er_max) continue;
                    }
                } else if (gate == 2) {
                    if (!fuse_chi2_ok(P, w.x, w.y, ur_pred, F.x[j], F.y[j], ur, oc)) continue;
                }
                ++count;
                const uint32_t d = hamming256(a0, a1, P.desc + (size_t)(row0 + F.id[j]) * 32);
                uint32_t key = (d << 16) | (uint32_t)j;
#pragma unroll
                for (int k = 0; k < PM_K; ++k)
                    if (key < loc[k]) {
                        const uint32_t t = loc[k];
                        loc[k] = key;
                        key = t;
                    }
            }
        }
    }
    count = __reduce_add_sync(0xffffffffu, count);
#pragma unroll
    for (int k = 0; k < PM_K; ++k) out[k] = ~0ull;
#pragma unroll
    for (int k = 0; k < PM_K; ++k) {
        const uint32_t m = __reduce_min_sync(0xffffffffu, loc[0]);
        if (m == 0xffffffffu) break;   // warp-uniform
        const int j = (int)(m & 0xffffu);
        out[k] = ((unsigned long long)(m >> 16) << 32) | ((unsigned long long)F.cell[j] << 16) | (unsigned long long)F.id[j];
        if (loc[0] == m) {             // sorted positions are unique => exactly one owner
#pragma unroll
            for (int q = 0; q + 1 < PM_K; ++q) loc[q] = loc[q + 1];
            loc[PM_K - 1] = 0xffffffffu;
        }
    }
    return count;
}

// ---- kernel A', modes 0 / 1: G lanes per query ----------------------------------------------------
// The windows of the two per-frame searches are small (th = 3: 2-3 grid columns of 2-3 cells, ~0.4 features per cell; th = 15: 4-12
// columns), so a whole warp per query leaves 31 lanes idle on every column run.  Here a query belongs to G adjacent lanes: lane g
// walks the columns c0 + g, c0 + g + G, ... serially, every lane keeps its own sorted top-K and the group merges them with K
// REDUX.MIN rounds.  The candidate SET, the keys and therefore the stored top-K are those of the warp-wide scan (keys are unique).
template <int G>
__device__ __forceinline__ int group_scan_query_grid(const ProjParams& P, const GridFeat& F, int row0, const Window& w, const uint8_t* qd,
                                                     float ur_pred, float er_max, unsigned gmask, int sub, unsigned long long out[PM_K]) {
    uint32_t loc[PM_K];
#pragma unroll
    for (int k = 0; k < PM_K; ++k) loc[k] = 0xffffffffu;
    int count = 0;
    if (!w.empty) {
        const uint4* q4 = reinterpret_cast<const uint4*>(qd);
        const uint4 a0 = __ldg(q4), a1 = __ldg(q4 + 1);
        const bool checkLevels = (w.minLevel > 0) || (w.maxLevel >= 0);
        for (int ix = w.c0 + sub; ix <= w.c1; ix += G) {
            const int jb = F.start[ix * GRID_ROWS + w.r0], je = F.start[ix * GRID_ROWS + w.r1 + 1];
            for (int j = jb; j < je; ++j) {   // one exit per iteration: the gates are a predicate, not branches
                const int oc = F.oct[j];
                const float dx = fsub(F.x[j], w.x), dy = fsub(F.y[j], w.y), ur = F.ur[j];
                bool pass = !(checkLevels && (oc < w.minLevel || (w.maxLevel >= 0 && oc > w.maxLevel)));
                pass = pass && (fabsf(dx) < w.r && fabsf(dy) < w.r);
                pass = pass && !(ur > 0 && fabsf(fsub(ur_pred, ur)) > er_max);
                if (pass) {
                    ++count;
                    const uint32_t d = hamming256(a0, a1, P.desc + (size_t)(row0 + F.id[j]) * 32);
                    uint32_t key = (d << 16) | (uint32_t)j;
#pragma unroll
                    for (int k = 0; k < PM_K; ++k) {   // branch-free sorted insert
                        const uint32_t lo = min(key, loc[k]);
                        key = max(key, loc[k]);
                        loc[k] = lo;
                    }
                }
            }
        }
    }
    count = __reduce_add_sync(gmask, count);
#pragma unroll
    for (int k = 0; k < PM_K; ++k) out[k] = ~0ull;
#pragma unroll
    for (int k = 0; k < PM_K; ++k) {
        const uint32_t m = __reduce_min_sync(gmask, loc[0]);
        if (m == 0xffffffffu) break;   // uniform over the group
        const int j = (int)(m & 0xffffu);
        out[k] = ((unsigned long long)(m >> 16) << 32) | ((unsigned long long)F.cell[j] << 16) | (unsigned long long)F.id[j];
        if (loc[0] == m) {             // sorted positions are unique => exactly one owner
#pragma unroll
            for (int q = 0; q + 1 < PM_K; ++q) loc[q] = loc[q + 1];
            loc[PM_K - 1] = 0xffffffffu;
        }
    }
    return count;
}

template <int G, class Src>
__device__ __forceinline__ void proj_candidates_grp_body(const ProjParams& P, const Src& S) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    const int frame = blockIdx.y;
    const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1];
    const int qbase = q0 + blockIdx.x * P.qpb;
    if (qbase >= q1) return;
    GridFeat GF;
    int N, row0;
    S.grid(P, frame, pm_smem, GF, N, row0);
    __syncthreads();
    const int lane = threadIdx.x & 31, sub = lane & (G - 1);
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane - sub));
    const int qend = min(qbase + P.qpb, q1);
    for (int q = qbase + (int)(threadIdx.x / G); q < qend; q += PM_WARPS * 32 / G) {   // uniform over the G lanes of a query
        Window w;
        float ur_pred = 0.f, er_max = 0.f, u = 0.f, invzc = 0.f, radius = 0.f;
        bool ok;
        if (P.mode == 0) {
            ok = local_window(P, q, w, er_max);
            ur_pred = P.a2[q];
        } else {
            ok = last_frame_window(P, frame, q, w, u, invzc, radius);
            ur_pred = fsub(u, fmul(P.bf, invzc));
            er_max = radius;
        }
        unsigned long long top[PM_K];
        int count = 0;
        if (ok) count = group_scan_query_grid<G>(P, GF, row0, w, P.qdesc + 32 * (size_t)q, ur_pred, er_max, gmask, sub, top);
        if (sub == 0) {
            P.cnt[q] = ok ? count : -1;
#pragma unroll
            for (int k = 0; k < PM_K; ++k) P.topk[(size_t)q * PM_K + k] = ok ? top[k] : ~0ull;
        }
    }
}

// ---- kernel A: order-free candidate scan ----------------------------------------------------------
template <class Src>
__device__ __forceinline__ void proj_candidates_body(const ProjParams& P, const Src& S) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    const int frame = blockIdx.y;
    const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1];
    const int qbase = q0 + blockIdx.x * PM_QPB;
    if (qbase >= q1) return;
    FrameFeat F;
    GridFeat GF;
    int N, row0;
    const bool use_grid = P.mode != 2;
    if (use_grid) S.grid(P, frame, pm_smem, GF, N, row0);
    else S.frame(P, P.frame_image[frame], frame, pm_smem, F, N, row0);
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int q = qbase + warp; q < min(qbase + PM_QPB, q1); q += PM_WARPS) {
        Window w;
        float ur_pred = 0.f, er_max = 0.f, u = 0.f, invzc = 0.f, radius = 0.f;
        bool ok;
        int gate = 0;
        if (P.mode == 0) {
            ok = local_window(P, q, w, er_max);
            ur_pred = P.a2[q];
        } else if (P.mode == 1) {
            ok = last_frame_window(P, frame, q, w, u, invzc, radius);
            ur_pred = fsub(u, fmul(P.bf, invzc));
            er_max = radius;
        } else if (P.mode == 3) {
            ok = kf_window(P, frame, q, w, ur_pred);
            gate = P.variant == 0 ? 2 : 1;
        } else if (P.mode == 4) {
            ok = P.level[q] <= 0;      // level1 > 0: continue (ORBmatcher.cc:758-760)
            if (ok) w = make_window(P, P.a0[q], P.a1[q], P.th, 0, 0);
            gate = 1;
        } else {
            w.node = P.level[q];       // query's vocabulary node
            w.empty = w.node < 0;
            ok = true;
            er_max = 3.0e38f;          // no stereo gate in SearchByBoW
        }
        unsigned long long top[PM_K];
        int count = 0;
        if (ok) count = use_grid ? warp_scan_query_grid(P, GF, row0, w, P.qdesc + 32 * (size_t)q, ur_pred, er_max, top, gate)
                                 : warp_scan_query(P, F, N, row0, w, P.qdesc + 32 * (size_t)q, top);
        if (lane == 0) {
            P.cnt[q] = ok ? count : -1;
#pragma unroll
            for (int k = 0; k < PM_K; ++k) P.topk[(size_t)q * PM_K + k] = ok ? top[k] : ~0ull;
        }
    }
}


// ---- kernel B: ordered resolve, one CTA per frame, warp 0 walks the queries ------------------------
// Its body is matcher_resolve.inc and that of kernel B' matcher_resolve_par.inc, each included inside the kernel's braces with `P`
// (the ProjParams) and `S` (SmemFrame or GlobalFrame) in scope.  Compiled as a function called by the kernel, their static shared
// arrays and early returns come out as different (equivalent) machine code, and k_proj_resolve / k_proj_resolve_par must keep theirs.
#define PM_CHUNK 1024

// ---- kernel B': the ordered resolve as a parallel fixed point (modes 0 and 1, the per-frame tracking searches) -----
// The reference walks the queries in order and a feature taken by query i is skipped by every later query.  Here every
// query first picks from its stored (distance, order)-sorted list as if nothing were taken; then, round after round,
// each query re-decides seeing only the features claimed BY EARLIER QUERIES in the previous round (claim[f] = smallest
// query index whose accepted choice is f).  Query 0 is final after one round, and a query is final one round after all
// the earlier queries it depends on, so the loop ends in (longest dependency chain + 1) rounds -- 2 to 4 in practice --
// and at the fixed point every choice is exactly what the sequential walk produces.  A query whose stored list is
// exhausted by claims (count > PM_K) gets the same exact rescan as in the sequential kernel, with the claim predicate.
#define PR_THREADS 512
#define PR_QCAP 8192
#define PR_LIST 512

__device__ __forceinline__ int pr_decide(const ProjParams& P, const FrameFeat& F, unsigned long long b1, unsigned long long b2) {
    if (b1 == ~0ull) return -1;
    const int bestDist = (int)(b1 >> 32), bestIdx = (int)(b1 & 0xffffu);
    if (bestDist > 100) return -1;   // TH_HIGH
    if (P.mode == 0) {               // ORBmatcher.cc:203-232
        const int bestDist2 = (b2 == ~0ull) ? 256 : (int)(b2 >> 32);
        const int idx2 = (b2 == ~0ull) ? 0 : (int)(b2 & 0xffffu);
        const int bestLevel = F.oct[bestIdx], bestLevel2 = (b2 == ~0ull) ? -1 : (int)F.oct[idx2];
        if (bestLevel == bestLevel2 && (float)bestDist > fmul(P.nnratio, (float)bestDist2)) return -1;
    }
    return bestIdx;
}

}  // namespace orb
