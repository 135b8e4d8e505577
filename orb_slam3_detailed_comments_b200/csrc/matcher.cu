// matcher.cu -- ORBmatcher::SearchByProjection family on the device, for Frame::Nleft == -1
// (pinhole / rectified stereo, the configurations of BASELINE.json):
//   * SearchByProjection(Frame&, const vector<MapPoint*>&, th, bFarPoints, thFarPoints)
//       /root/reference/src/ORBmatcher.cc:45-239      (TrackLocalMap, Tracking.cc:4062)
//   * SearchByProjection(Frame& cur, const Frame& last, th, bMono)
//       /root/reference/src/ORBmatcher.cc:1950-2184   (TrackWithMotionModel, Tracking.cc:3389)
//   * SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>&)
//       /root/reference/src/ORBmatcher.cc:259-493     (TrackReferenceKeyFrame, Tracking.cc:3183)
//   * the projection searches into a KeyFrame (mode 3): Fuse x2 (:1325-1687), SearchByProjection(KF, Scw, ...) x2
//       (:495-732), SearchByProjection(CurrentFrame, KeyFrame, sAlreadyFound, th, ORBdist) (:2196-2330)
//   * SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize) (mode 4, :734-890)
// with Frame::GetFeaturesInArea / PosInGrid (src/Frame.cc:859-951, 962-978) folded in.
//
// The reference is greedy: a feature claimed by query i is skipped by every later query.  Here the
// expensive part is order-free -- one warp per query scans the frame's features (staged in shared
// memory), applies the window / level / stereo gates, takes 256-bit Hamming distances with __popc
// and keeps the K smallest (distance, reference-candidate-order) keys -- and a per-frame resolve pass
// (one warp) replays the queries in order against the claim mask.  If claims eat into a query's
// stored list so that its best / second best can no longer be known, the resolve warp rescans that
// query with the mask applied (exact slow path).
#include <algorithm>
#include <vector>

#include "extractor.h"
#include "devmath.cuh"

using namespace orb;
using namespace orbdev;

namespace orb {

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

__device__ __forceinline__ void stage_frame(const ProjParams& P, int img, unsigned char* smem, FrameFeat& F, int& N, int& row0) {
    N = min(P.nkp[img], P.maxFeat);
    row0 = P.offsets[img];
    const size_t M = (size_t)P.maxFeat;
    F.x = reinterpret_cast<float*>(smem);
    F.y = F.x + M;
    F.ur = F.y + M;
    F.ang = F.ur + M;
    F.node = reinterpret_cast<int*>(F.ang + M);
    F.cell = reinterpret_cast<uint16_t*>(F.node + M);
    F.oct = reinterpret_cast<uint8_t*>(F.cell + M);
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

// ---- Frame::AssignFeaturesToGrid (Frame.cc:469-504) as a CSR table: feature ids sorted by (cell, id) -------------
#define PM_NCELL (GRID_COLS * GRID_ROWS)
// Counting sort: per-cell histogram, exclusive scan (= the CSR table), unordered scatter, then every feature finds its rank among
// the ids of its own cell (runs are a few features long; a run of n costs n steps per feature, so the worst case stays bounded).
// Features outside the grid (PosInGrid false) form the run after the last cell, in id order, as in the sorted-key formulation.
__global__ void __launch_bounds__(256) k_frame_grid(const __grid_constant__ ProjParams P) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    int* cnt = reinterpret_cast<int*>(pm_smem);                         // PM_NCELL + 2: counts, then exclusive starts
    uint16_t* cellOf = reinterpret_cast<uint16_t*>(cnt + PM_NCELL + 2);   // maxFeat
    uint16_t* tmp = cellOf + P.maxFeat;                                  // maxFeat: ids in cell order, unordered inside a cell
    __shared__ int s_warp[8];
    const int frame = blockIdx.x, img = P.frame_image[frame];
    const int N = min(P.nkp[img], P.maxFeat), row0 = P.offsets[img];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int c = tid; c < PM_NCELL + 2; c += 256) cnt[c] = 0;
    __syncthreads();
    for (int i = tid; i < N; i += 256) {
        const orbx_keypoint k = P.kps[row0 + i];
        const int px = (int)roundf(fmul(fsub(k.x, P.minX), P.invW)), py = (int)roundf(fmul(fsub(k.y, P.minY), P.invH));
        const int cell = (px < 0 || px >= GRID_COLS || py < 0 || py >= GRID_ROWS) ? PM_NCELL : (px * GRID_ROWS + py);
        cellOf[i] = (uint16_t)cell;
        atomicAdd(&cnt[cell], 1);
    }
    __syncthreads();
    // exclusive scan of cnt[0 .. PM_NCELL] (3073 entries; 13 per thread covers 3328)
    constexpr int PER = (PM_NCELL + 1 + 255) / 256;
    int loc[PER], sum = 0;
#pragma unroll
    for (int k = 0; k < PER; ++k) {
        const int c = tid * PER + k;
        loc[k] = c <= PM_NCELL ? cnt[c] : 0;
        sum += loc[k];
    }
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
    }
    if (lane == 31) s_warp[wid] = inc;
    __syncthreads();
    int base = inc - sum;
    for (int w = 0; w < wid; ++w) base += s_warp[w];
    uint16_t* start = P.gridStart + (size_t)frame * (PM_NCELL + 1);
#pragma unroll
    for (int k = 0; k < PER; ++k) {
        const int c = tid * PER + k;
        if (c <= PM_NCELL) {
            cnt[c] = base;                       // start of cell c; cnt doubles as the fill cursor below
            if (c < PM_NCELL) start[c] = (uint16_t)base;
            else start[PM_NCELL] = (uint16_t)base;   // first position outside the grid
        }
        base += loc[k];
    }
    if (tid == 0) cnt[PM_NCELL + 1] = N;
    __syncthreads();
    for (int i = tid; i < N; i += 256) tmp[atomicAdd(&cnt[cellOf[i]], 1)] = (uint16_t)i;   // cnt[c] ends at start[c + 1]
    __syncthreads();
    uint16_t* order = P.gridOrder + (size_t)frame * P.maxFeat;
    for (int p = tid; p < N; p += 256) {
        const int id = tmp[p], c = cellOf[id];
        const int b = c > 0 ? cnt[c - 1] : 0, e = cnt[c];   // the cursors after the scatter: cnt[c] = end of cell c = start of cell c + 1
        int rank = 0;
        for (int q = b; q < e; ++q) rank += tmp[q] < id;
        order[b + rank] = (uint16_t)id;
    }
}

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

__device__ __forceinline__ void stage_grid(const ProjParams& P, int frame, unsigned char* smem, GridFeat& F, int& N, int& row0) {
    const int img = P.frame_image[frame];
    N = min(P.nkp[img], P.maxFeat);
    row0 = P.offsets[img];
    const size_t M = (size_t)P.maxFeat;
    F.x = reinterpret_cast<float*>(smem);
    F.y = F.x + M;
    F.ur = F.y + M;
    F.cell = reinterpret_cast<uint16_t*>(F.ur + M);
    F.id = F.cell + M;
    F.start = F.id + M;
    F.oct = reinterpret_cast<uint8_t*>(F.start + PM_NCELL + 2);
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

template <int G>
__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates_grp(const __grid_constant__ ProjParams P) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    const int frame = blockIdx.y;
    const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1];
    const int qbase = q0 + blockIdx.x * P.qpb;
    if (qbase >= q1) return;
    GridFeat GF;
    int N, row0;
    stage_grid(P, frame, pm_smem, GF, N, row0);
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
__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates(const __grid_constant__ ProjParams P) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    const int frame = blockIdx.y;
    const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1];
    const int qbase = q0 + blockIdx.x * PM_QPB;
    if (qbase >= q1) return;
    FrameFeat F;
    GridFeat GF;
    int N, row0;
    const bool use_grid = P.mode != 2;
    if (use_grid) stage_grid(P, frame, pm_smem, GF, N, row0);
    else stage_frame(P, P.frame_image[frame], pm_smem, F, N, row0);
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
#define PM_CHUNK 1024

__global__ void __launch_bounds__(256) k_proj_resolve(const __grid_constant__ ProjParams P) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    const int frame = blockIdx.x;
    if (P.seqFlag && P.seqFlag[frame] == 0) return;   // resolved by k_proj_resolve_par
    const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1];
    FrameFeat F;
    int N, row0;
    stage_frame(P, P.frame_image[frame], pm_smem, F, N, row0);
    unsigned char* extra = pm_smem + ((frame_smem_bytes(P.maxFeat) + 15) / 16) * 16;
    unsigned long long* s_top = reinterpret_cast<unsigned long long*>(extra);           // PM_CHUNK * PM_K
    int* s_cnt = reinterpret_cast<int*>(s_top + PM_CHUNK * PM_K);                        // PM_CHUNK
    int* s_holder = s_cnt + PM_CHUNK;                                                    // maxFeat: mode 1 holder query, mode 0 unused
    uint8_t* s_claimed = reinterpret_cast<uint8_t*>(s_holder + P.maxFeat);               // maxFeat
    __shared__ int s_hist[30];
    __shared__ int s_nm;
    const bool bowKF = P.mode == 2 && P.variant == 1;          // SearchByBoW(KF, KF): per-query output, strict TH_LOW
    const bool init = P.mode == 4;                              // SearchForInitialization: distance-dependent claims
    const bool perQuery = P.mode == 0 || P.mode == 3 || bowKF || init;  // match[q] = feature  (else: match[feature row] = query)
    const bool claims = P.mode == 0 || bowKF || (P.mode == 3 && (P.variant == 2 || P.variant == 3));
    const bool oriHist = P.checkOri && (P.mode == 1 || P.mode == 2 || init || (P.mode == 3 && P.variant == 3));
    for (int i = threadIdx.x; i < N; i += blockDim.x) {
        s_claimed[i] = (claims && P.flag) ? P.flag[row0 + i] : 0;
        s_holder[i] = -1;
    }
    if (threadIdx.x < 30) s_hist[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_nm = 0;
    if (oriHist)
        for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) P.quv[q] = __int_as_float(-1);
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int nmatches = 0;
    float* s_qf = reinterpret_cast<float*>(s_claimed + ((P.maxFeat + 15) / 16) * 16);   // PM_CHUNK: mode 1 last angle
    uint8_t* s_qflag = reinterpret_cast<uint8_t*>(s_qf + PM_CHUNK);                      // PM_CHUNK: mode 1 obs > 0
    int* s_md = reinterpret_cast<int*>(s_qflag + PM_CHUNK);                              // maxFeat (mode 4): vMatchedDistance
    if (init) {
        for (int i = threadIdx.x; i < N; i += blockDim.x) s_md[i] = 0x7fffffff;
        __syncthreads();
    }
    for (int base = q0; base < q1; base += PM_CHUNK) {
        const int nchunk = min(PM_CHUNK, q1 - base);
        for (int i = threadIdx.x; i < nchunk * PM_K; i += blockDim.x) s_top[i] = P.topk[(size_t)base * PM_K + i];
        for (int i = threadIdx.x; i < nchunk; i += blockDim.x) {
            s_cnt[i] = P.cnt[base + i];
            if (perQuery) P.match[base + i] = -1;
            if (P.mode != 0) { s_qf[i] = P.f0 ? P.f0[base + i] : 0.f; s_qflag[i] = (P.mode == 1) ? P.flag[base + i] : (uint8_t)1; }
        }
        __syncthreads();
        if (warp == 0) {
            for (int qi = 0; qi < nchunk; ++qi) {
                const int q = base + qi;
                const int count = s_cnt[qi];
                if (count <= 0) continue;
                // the stored candidates are sorted by (distance, reference order): lane k looks at entry k, the first
                // (two) still-free ones are the best / second best of the reference's sequential scan
                const int stored = min(count, PM_K);
                const unsigned long long key = (lane < stored) ? s_top[qi * PM_K + lane] : ~0ull;
                const int kidx = (lane < stored) ? (int)(key & 0xffffu) : 0;   // in range even if the load is speculated
                const bool is_free = (lane < stored) && (init ? s_md[kidx] > (int)(key >> 32) : !s_claimed[kidx]);
                const unsigned fm = __ballot_sync(0xffffffffu, is_free);
                const int live = __popc(fm);
                const int need = (P.mode == 1 || P.mode == 3) ? 1 : 2;   // modes 0, 2, 4 use the second best
                unsigned long long b1 = ~0ull, b2 = ~0ull;
                if (live < need && count > PM_K) {
                    // claims consumed the stored list: exact rescan with the mask applied (warp-cooperative)
                    Window w;
                    float ur_pred = 0.f, er_max = 0.f, u = 0.f, invzc = 0.f, radius = 0.f;
                    int gate = 0;
                    if (P.mode == 0) {
                        local_window(P, q, w, er_max);
                        ur_pred = P.a2[q];
                    } else if (P.mode == 1) {
                        last_frame_window(P, frame, q, w, u, invzc, radius);
                        ur_pred = fsub(u, fmul(P.bf, invzc));
                        er_max = radius;
                    } else if (P.mode == 3) {
                        kf_window(P, frame, q, w, ur_pred);
                        gate = P.variant == 0 ? 2 : 1;
                    } else if (init) {
                        w = make_window(P, P.a0[q], P.a1[q], P.th, 0, 0);
                        gate = 1;
                    } else {
                        w.node = P.level[q];
                        w.empty = w.node < 0;
                        er_max = 3.0e38f;
                    }
                    warp_rescan_best2(P, F, N, row0, w, P.qdesc + 32 * (size_t)q, ur_pred, er_max, init ? nullptr : s_claimed, gate, b1, b2,
                                      init ? s_md : nullptr);
                } else {
                    if (fm) {
                        const int i1 = __ffs(fm) - 1;
                        b1 = __shfl_sync(0xffffffffu, key, i1);
                        const unsigned fm2 = fm & (fm - 1);
                        if (fm2) b2 = __shfl_sync(0xffffffffu, key, __ffs(fm2) - 1);
                    }
                }
                if (b1 == ~0ull) continue;
                const int bestDist = (int)(b1 >> 32), bestIdx = (int)(b1 & 0xffffu);
                if (P.mode == 0) {
                    const int bestDist2 = (b2 == ~0ull) ? 256 : (int)(b2 >> 32);
                    const int idx2 = (b2 == ~0ull) ? 0 : (int)(b2 & 0xffffu);   // in range even if the load is speculated
                    const int bestLevel = F.oct[bestIdx], bestLevel2 = (b2 == ~0ull) ? -1 : (int)F.oct[idx2];
                    if (bestDist <= 100) {   // TH_HIGH
                        const float lim = fmul(P.nnratio, (float)bestDist2);
                        if (bestLevel == bestLevel2 && (float)bestDist > lim) continue;
                        if (bestLevel != bestLevel2 || (float)bestDist <= lim) {
                            if (lane == 0) {
                                P.match[q] = bestIdx;
                                s_claimed[bestIdx] = 1;
                            }
                            ++nmatches;
                            __syncwarp();
                        }
                    }
                } else if (init) {
                    // ORBmatcher.cc:800-835: TH_LOW, ratio against the second best, a better match steals the feature
                    const float d2f = (b2 == ~0ull) ? 2147483648.0f : (float)(int)(b2 >> 32);
                    if (bestDist <= 50 && (float)bestDist < fmul(d2f, P.nnratio)) {
                        const int old = s_holder[bestIdx];
                        if (lane == 0) {
                            if (old >= 0) P.match[old] = -1;
                            P.match[q] = bestIdx;
                            s_holder[bestIdx] = q;
                            s_md[bestIdx] = bestDist;
                            if (oriHist) {
                                float rot = fsub(s_qf[qi], F.ang[bestIdx]);
                                if (rot < 0.0f) rot = fadd(rot, 360.0f);
                                int bin = (int)roundf(fmul(rot, 1.0f / 30));
                                if (bin == 30) bin = 0;
                                s_hist[bin] += 1;
                                P.quv[q] = __int_as_float((bin << 16) | bestIdx);
                            }
                        }
                        if (old < 0) ++nmatches;
                        __syncwarp();
                    }
                } else if (perQuery) {
                    bool accept = (float)bestDist <= P.thr;
                    if (bowKF) {   // ORBmatcher.cc:978-982: bestDist1 < TH_LOW and the ratio test in float
                        const int bestDist2 = (b2 == ~0ull) ? 256 : (int)(b2 >> 32);
                        accept = bestDist < 50 && (float)bestDist < fmul(P.nnratio, (float)bestDist2);
                    }
                    if (accept) {
                        if (lane == 0) {
                            P.match[q] = bestIdx;
                            if (claims) s_claimed[bestIdx] = 1;
                            if (oriHist) {
                                float rot = fsub(s_qf[qi], F.ang[bestIdx]);
                                if (rot < 0.0f) rot = fadd(rot, 360.0f);
                                int bin = (int)roundf(fmul(rot, 1.0f / 30));
                                if (bin == 30) bin = 0;
                                s_hist[bin] += 1;
                                P.quv[q] = __int_as_float((bin << 16) | bestIdx);
                            }
                        }
                        ++nmatches;
                        __syncwarp();
                    }
                } else {
                    bool accept = bestDist <= 100;
                    if (P.mode == 2) {   // SearchByBoW: TH_LOW and the ratio test in float (ORBmatcher.cc:384-387)
                        const int bestDist2 = (b2 == ~0ull) ? 256 : (int)(b2 >> 32);
                        accept = bestDist <= 50 && (float)bestDist < fmul(P.nnratio, (float)bestDist2);
                    }
                    if (accept) {
                        if (lane == 0) {
                            s_holder[bestIdx] = q;
                            s_claimed[bestIdx] = (P.mode == 2 || s_qflag[qi]) ? 1 : 0;   // mode 1: only map points with observations block
                            if (oriHist) {
                                float rot = fsub(s_qf[qi], F.ang[bestIdx]);
                                if (rot < 0.0f) rot = fadd(rot, 360.0f);
                                int bin = (int)roundf(fmul(rot, 1.0f / 30));
                                if (bin == 30) bin = 0;
                                s_hist[bin] += 1;
                                P.quv[q] = __int_as_float((bin << 16) | bestIdx);   // rotHist entry of this query
                            }
                        }
                        ++nmatches;
                        __syncwarp();
                    }
                }
            }
        }
        __syncthreads();
    }
    if (perQuery && !oriHist) {
        if (threadIdx.x == 0) P.nmatches[frame] = nmatches;
        return;
    }
    // ---- mode 1: rotation-histogram filter (ORBmatcher.cc:2160-2181, ComputeThreeMaxima :2335-2377) ----
    __shared__ int s_keep[30];
    if (threadIdx.x == 0) {
        s_nm = nmatches;
        int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
        for (int i = 0; i < 30; ++i) {
            const int s = s_hist[i];
            if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
            else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
            else if (s > max3) { max3 = s; ind3 = i; }
        }
        if ((float)max2 < fmul(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
        else if ((float)max3 < fmul(0.1f, (float)max1)) { ind3 = -1; }
        for (int i = 0; i < 30; ++i) s_keep[i] = (i == ind1 || i == ind2 || i == ind3) ? 1 : 0;
    }
    __syncthreads();
    if (oriHist) {
        int removed = 0;
        for (int q = q0 + threadIdx.x; q < q1; q += blockDim.x) {
            if (P.cnt[q] <= 0) continue;
            const int e = __float_as_int(P.quv[q]);
            if (e < 0) continue;
            const int bin = e >> 16, idx = e & 0xffff;
            if (!s_keep[bin]) {
                if (init) {                 // ORBmatcher.cc:870-876: only matches that are still alive count
                    if (P.match[q] >= 0) { P.match[q] = -1; ++removed; }
                    continue;
                }
                if (perQuery) P.match[q] = -1;
                else s_holder[idx] = -1;   // every entry of a rejected bin clears its feature (duplicates included)
                ++removed;
            }
        }
        if (removed) atomicSub(&s_nm, removed);
    }
    __syncthreads();
    if (!perQuery)
        for (int i = threadIdx.x; i < N; i += blockDim.x) P.match[row0 + i] = s_holder[i];
    if (threadIdx.x == 0) P.nmatches[frame] = s_nm;
}


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

__global__ void __launch_bounds__(PR_THREADS) k_proj_resolve_par(const __grid_constant__ ProjParams P) {
    extern __shared__ __align__(16) unsigned char pm_smem[];
    const int frame = blockIdx.x, tid = threadIdx.x;
    const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1], nq = q1 - q0;
    if (nq > PR_QCAP) {
        if (tid == 0) P.seqFlag[frame] = 1;
        return;
    }
    FrameFeat F;
    int N, row0;
    stage_frame(P, P.frame_image[frame], pm_smem, F, N, row0);
    unsigned char* extra = pm_smem + ((frame_smem_bytes(P.maxFeat) + 15) / 16) * 16;
    int* s_claim = reinterpret_cast<int*>(extra);            // maxFeat
    int* s_holder = s_claim + P.maxFeat;                       // maxFeat (mode 1: last query holding the feature)
    int* s_choice = s_holder + P.maxFeat;                      // PR_QCAP
    int* s_list = s_choice + PR_QCAP;                          // PR_LIST
    uint8_t* s_static = reinterpret_cast<uint8_t*>(s_list + PR_LIST);   // maxFeat
    __shared__ int s_hist[30], s_keep[30], s_nm, s_nlist, s_over;
    for (int i = tid; i < N; i += PR_THREADS) {
        s_static[i] = (P.mode == 0 && P.flag) ? P.flag[row0 + i] : 0;
        s_holder[i] = -1;
        s_claim[i] = 0x7fffffff;
    }
    for (int i = tid; i < nq; i += PR_THREADS) s_choice[i] = -1;
    if (tid < 30) s_hist[tid] = 0;
    if (tid == 0) { s_nm = 0; s_nlist = 0; s_over = 0; }
    __syncthreads();
    const int need = P.mode == 1 ? 1 : 2;
    const int lane = tid & 31, warp = tid >> 5;
    for (;;) {
        int changed = 0;
        for (int ql = tid; ql < nq; ql += PR_THREADS) {
            const int q = q0 + ql, count = P.cnt[q];
            int choice = -1;
            if (count > 0) {
                const int stored = min(count, PM_K);
                const unsigned long long* top = P.topk + (size_t)q * PM_K;
                unsigned long long b1 = ~0ull, b2 = ~0ull;
                int nfree = 0;
                for (int k = 0; k < stored && nfree < need; ++k) {
                    const unsigned long long key = top[k];
                    const int f = (int)(key & 0xffffu);
                    if (s_static[f] || s_claim[f] < ql) continue;
                    if (nfree == 0) b1 = key; else b2 = key;
                    ++nfree;
                }
                if (nfree < need && count > PM_K) {   // exhausted by claims: exact rescan below
                    const int slot = atomicAdd(&s_nlist, 1);
                    if (slot < PR_LIST) s_list[slot] = ql; else s_over = 1;
                    continue;
                }
                choice = pr_decide(P, F, b1, b2);
            }
            if (choice != s_choice[ql]) { s_choice[ql] = choice; changed = 1; }
        }
        __syncthreads();
        const int nl = min(s_nlist, PR_LIST);
        for (int i = warp; i < nl; i += PR_THREADS / 32) {
            const int ql = s_list[i], q = q0 + ql;
            Window w;
            float ur_pred = 0.f, er_max = 0.f, u = 0.f, invzc = 0.f, radius = 0.f;
            if (P.mode == 0) {
                local_window(P, q, w, er_max);
                ur_pred = P.a2[q];
            } else {
                last_frame_window(P, frame, q, w, u, invzc, radius);
                ur_pred = fsub(u, fmul(P.bf, invzc));
                er_max = radius;
            }
            unsigned long long b1, b2;
            warp_rescan_best2(P, F, N, row0, w, P.qdesc + 32 * (size_t)q, ur_pred, er_max, s_static, 0, b1, b2, nullptr, s_claim, ql);
            const int choice = pr_decide(P, F, b1, b2);
            if (lane == 0 && choice != s_choice[ql]) { s_choice[ql] = choice; changed = 1; }
        }
        const int any = __syncthreads_or(changed);
        if (s_over) {                                  // more exhausted lists than the rescan list holds: sequential kernel
            if (tid == 0) P.seqFlag[frame] = 1;
            return;
        }
        if (!any) break;
        for (int i = tid; i < N; i += PR_THREADS) s_claim[i] = 0x7fffffff;
        if (tid == 0) s_nlist = 0;
        __syncthreads();
        for (int ql = tid; ql < nq; ql += PR_THREADS) {
            const int c = s_choice[ql];
            if (c >= 0 && (P.mode == 0 || P.flag[q0 + ql])) atomicMin(&s_claim[c], ql);   // mode 1: only map points with observations block
        }
        __syncthreads();
    }
    // ---- outputs ---------------------------------------------------------------------------------------------------
    int acc = 0;
    for (int ql = tid; ql < nq; ql += PR_THREADS) {
        const int q = q0 + ql, c = s_choice[ql];
        if (P.mode == 0) {
            P.match[q] = c;
        } else {
            int e = -1;
            if (c >= 0) {
                atomicMax(&s_holder[c], q);              // the last query that takes a feature holds it
                if (P.checkOri) {
                    float rot = fsub(P.f0[q], F.ang[c]);
                    if (rot < 0.0f) rot = fadd(rot, 360.0f);
                    int bin = (int)roundf(fmul(rot, 1.0f / 30));
                    if (bin == 30) bin = 0;
                    atomicAdd(&s_hist[bin], 1);
                    e = (bin << 16) | c;
                }
            }
            if (P.checkOri) P.quv[q] = __int_as_float(e);
        }
        acc += c >= 0;
    }
    acc = __reduce_add_sync(0xffffffffu, acc);
    if (lane == 0 && acc) atomicAdd(&s_nm, acc);
    __syncthreads();
    if (P.mode == 0) {
        if (tid == 0) P.nmatches[frame] = s_nm;
        return;
    }
    // rotation-histogram filter (ORBmatcher.cc:2160-2181, ComputeThreeMaxima :2335-2377)
    if (tid == 0) {
        int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
        for (int i = 0; i < 30; ++i) {
            const int s = s_hist[i];
            if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
            else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
            else if (s > max3) { max3 = s; ind3 = i; }
        }
        if ((float)max2 < fmul(0.1f, (float)max1)) { ind2 = -1; ind3 = -1; }
        else if ((float)max3 < fmul(0.1f, (float)max1)) { ind3 = -1; }
        for (int i = 0; i < 30; ++i) s_keep[i] = (i == ind1 || i == ind2 || i == ind3) ? 1 : 0;
    }
    __syncthreads();
    if (P.checkOri) {
        int removed = 0;
        for (int ql = tid; ql < nq; ql += PR_THREADS) {
            const int e = __float_as_int(P.quv[q0 + ql]);
            if (e < 0) continue;
            if (!s_keep[e >> 16]) {
                s_holder[e & 0xffff] = -1;   // every entry of a rejected bin clears its feature (duplicates included)
                ++removed;
            }
        }
        if (removed) atomicSub(&s_nm, removed);
    }
    __syncthreads();
    for (int i = tid; i < N; i += PR_THREADS) P.match[row0 + i] = s_holder[i];
    if (tid == 0) P.nmatches[frame] = s_nm;
}


// ---- Frame::isInFrustum (src/Frame.cc:667-720): one thread per candidate map point ------------------------------------
struct FrustumParams {
    const int* poff;           // [n_frames + 1]
    const float* Rcw;          // [n_frames][9] row-major mRcw
    const float* tcw;          // [n_frames][3] mtcw
    const float* Ow;           // [n_frames][3] mOw
    const float* xw;           // [np][3]
    const float* normal;
    const float* maxD;
    const float* minD;
    float fx, fy, cx, cy, bf, minX, maxX, minY, maxY, logScale, cosLimit;
    int nLevels;
    uint8_t* in_view;
    float *px, *py, *pxr, *vc, *depth;
    int* level;
};

__global__ void __launch_bounds__(256) k_in_frustum(const __grid_constant__ FrustumParams P) {
    const int frame = blockIdx.y;
    const int p0 = P.poff[frame], p1 = P.poff[frame + 1];
    const int i = p0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p1) return;
    const float* R = P.Rcw + 9 * frame;
    const float* t = P.tcw + 3 * frame;
    const float* O = P.Ow + 3 * frame;
    const float X = P.xw[3 * (size_t)i], Y = P.xw[3 * (size_t)i + 1], Z = P.xw[3 * (size_t)i + 2];
    uint8_t vis = 0;
    float u = -1.f, v = -1.f, ur = -1.f, viewCos = 0.f, dep = 0.f;
    int lvl = -1;
    // Eigen's fixed-size product / norm / dot: a0 b0 + (a1 b1 + a2 b2)
    const float xc = fadd(fadd(fmul(R[0], X), fadd(fmul(R[1], Y), fmul(R[2], Z))), t[0]);
    const float yc = fadd(fadd(fmul(R[3], X), fadd(fmul(R[4], Y), fmul(R[5], Z))), t[1]);
    const float zc = fadd(fadd(fmul(R[6], X), fadd(fmul(R[7], Y), fmul(R[8], Z))), t[2]);
    const float pcDist = fsqrt(fadd(fmul(xc, xc), fadd(fmul(yc, yc), fmul(zc, zc))));
    const float invz = fdiv(1.0f, zc);
    do {
        if (zc < 0.0f) break;
        const float uu = fadd(fdiv(fmul(P.fx, xc), zc), P.cx), vv = fadd(fdiv(fmul(P.fy, yc), zc), P.cy);
        if (uu < P.minX || uu > P.maxX) break;
        if (vv < P.minY || vv > P.maxY) break;
        u = uu;
        v = vv;
        const float ox = fsub(X, O[0]), oy = fsub(Y, O[1]), oz = fsub(Z, O[2]);
        const float dist = fsqrt(fadd(fmul(ox, ox), fadd(fmul(oy, oy), fmul(oz, oz))));
        if (dist < fmul(0.8f, P.minD[i]) || dist > fmul(1.2f, P.maxD[i])) break;   // Get{Min,Max}DistanceInvariance, MapPoint.cc:658-672
        const float* n = P.normal + 3 * (size_t)i;
        const float c = fdiv(fadd(fmul(ox, n[0]), fadd(fmul(oy, n[1]), fmul(oz, n[2]))), dist);
        if (c < P.cosLimit) break;
        int l = (int)ceilf(fdiv(glibc_logf(fdiv(P.maxD[i], dist)), P.logScale));   // MapPoint::PredictScale
        if (l < 0) l = 0;
        else if (l >= P.nLevels) l = P.nLevels - 1;
        vis = 1;
        ur = fsub(uu, fmul(P.bf, invz));
        dep = pcDist;
        lvl = l;
        viewCos = c;
    } while (false);
    P.in_view[i] = vis; P.px[i] = u; P.py[i] = v; P.pxr[i] = ur; P.level[i] = lvl; P.vc[i] = viewCos; P.depth[i] = dep;
}

}  // namespace orb

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static orb_status launch_proj(orbx_handle* h, ProjParams& P, int n_frames, int max_q_per_frame) {
    cudaStream_t st = h->stream;
    const size_t fsm = ((size_t)P.maxFeat * 23 + 16 + 15) / 16 * 16;
    const size_t gsm = ((size_t)P.maxFeat * 17 + (PM_NCELL + 1) * 2 + 32 + 15) / 16 * 16;
    const size_t csm = std::max(fsm, gsm);
    if (P.mode != 2) {   // modes 0, 1, 3 search a window of the feature grid
        const size_t gridSm = (size_t)(PM_NCELL + 2) * 4 + (size_t)P.maxFeat * 4 + 16;
        ORB_CUDA(cudaFuncSetAttribute(k_frame_grid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(gridSm, (size_t)1024)));
        launch_p(k_frame_grid, dim3(n_frames), dim3(256), gridSm, st, P);
        ORB_LAUNCHED();
    }
    // modes 0 / 1 (the two per-frame searches): G lanes per query (ORB_PROJ_LANES = 4 | 8 | 16; 32 = the warp-per-query kernel)
    const char* vLanes = getenv("ORB_PROJ_LANES");
    const char* vQpb = getenv("ORB_PROJ_QPB");
    const int envLanes = vLanes ? atoi(vLanes) : 0, envQpb = vQpb ? atoi(vQpb) : 0;
    const int lanes = P.mode > 1 ? 32 : (envLanes ? envLanes : (P.mode == 0 ? 4 : 8));
    if (lanes == 4 || lanes == 8 || lanes == 16) {
        P.qpb = envQpb > 0 ? envQpb : (P.mode == 0 ? 128 : 64);
        auto kern = lanes == 4 ? k_proj_candidates_grp<4> : (lanes == 8 ? k_proj_candidates_grp<8> : k_proj_candidates_grp<16>);
        ORB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(csm, (size_t)1024)));
        dim3 grid((max_q_per_frame + P.qpb - 1) / P.qpb, n_frames);
        if (grid.x > 0) {
            launch_p(kern, grid, dim3(PM_WARPS * 32), csm, st, P);
            ORB_LAUNCHED();
        }
    } else {
        ORB_CUDA(cudaFuncSetAttribute(k_proj_candidates, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(csm, (size_t)1024)));
        dim3 grid((max_q_per_frame + PM_QPB - 1) / PM_QPB, n_frames);
        if (grid.x > 0) {
            k_proj_candidates<<<grid, PM_WARPS * 32, csm, st>>>(P);
            ORB_LAUNCHED();
        }
    }
    if (P.seqFlag) {   // modes 0 / 1: parallel fixed-point resolve; frames it cannot finish are flagged for the sequential kernel
        const size_t psm = fsm + (size_t)P.maxFeat * 9 + (size_t)(PR_QCAP + PR_LIST) * 4 + 64;
        ORB_CUDA(cudaFuncSetAttribute(k_proj_resolve_par, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psm));
        launch_p(k_proj_resolve_par, dim3(n_frames), dim3(PR_THREADS), psm, st, P);
        ORB_LAUNCHED();
    }
    const size_t rsm = fsm + (size_t)PM_CHUNK * PM_K * 8 + (size_t)PM_CHUNK * 4 + (size_t)P.maxFeat * (P.mode == 4 ? 9 : 5) + (size_t)PM_CHUNK * 5 + 256;
    ORB_CUDA(cudaFuncSetAttribute(k_proj_resolve, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rsm));
    launch_p(k_proj_resolve, dim3(n_frames), dim3(256), rsm, st, P);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return ORB_OK;
}

static void fill_frame_side(orbx_handle* h, const orbm_camera* cam, ProjParams& P) {
    P.kps = h->d_kps;
    P.desc = h->d_desc;
    P.uright = h->stereo_valid ? h->d_uright : nullptr;
    P.offsets = h->d_offsets;
    P.nkp = h->d_nkp;
    P.maxFeat = h->geom.kpTotal;
    P.minX = cam->min_x; P.maxX = cam->max_x; P.minY = cam->min_y; P.maxY = cam->max_y;
    P.invW = (float)GRID_COLS / (cam->max_x - cam->min_x);   // Frame.cc:187-188
    P.invH = (float)GRID_ROWS / (cam->max_y - cam->min_y);
    P.fx = cam->fx; P.fy = cam->fy; P.cx = cam->cx; P.cy = cam->cy; P.bf = cam->bf;
    for (int l = 0; l < ORB_MAX_LEVELS; ++l) P.scale[l] = l < h->cfg.n_levels ? h->scale[l] : 1.f;
}

// Query counts of a per-frame search (total, largest frame) and the rows of the batch.  Host tables are read in place, device
// tables are read back; bounded (orbm_set_device_query_bounds), the bounds stand in and nothing is read back.
static orb_status frame_table(orbx_handle* h, int nf, const int32_t* frame_image, const int32_t* query_offset, bool dev, bool bounded,
                              int& nq, int& maxq, int& rows) {
    rows = h->rows_bound > 0 ? h->rows_bound : (int)h->out_rows;
    orb_status s;
    if (!bounded && (s = batch_rows(h, &rows)) != ORB_OK) return s;
    std::vector<int> qoff_h(nf + 1, 0), fimg_h(nf, 0);
    if (dev && !bounded) {
        ORB_CUDA(cudaMemcpyAsync(qoff_h.data(), query_offset, sizeof(int) * (nf + 1), cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaMemcpyAsync(fimg_h.data(), frame_image, sizeof(int) * nf, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    } else if (!dev) {
        std::copy(query_offset, query_offset + nf + 1, qoff_h.begin());
        std::copy(frame_image, frame_image + nf, fimg_h.begin());
    }
    nq = qoff_h[nf];
    maxq = 0;
    for (int f = 0; f < nf; ++f) {
        maxq = std::max(maxq, qoff_h[f + 1] - qoff_h[f]);
        if (fimg_h[f] < 0 || fimg_h[f] >= h->last_batch || qoff_h[f + 1] < qoff_h[f]) return set_error(ORB_ERR_INVALID, "bad frame table");
    }
    if (bounded) { nq = h->q_total_bound; maxq = h->q_frame_bound; }   // upper bounds: the kernels take the real counts from the device tables
    return ORB_OK;
}

extern "C" orb_status orbm_set_device_query_bounds(orbx_handle* h, int32_t total_queries, int32_t max_queries_per_frame, int32_t total_rows) {
    if (!h || total_queries < 0 || max_queries_per_frame < 0 || total_rows < 0) return set_error(ORB_ERR_INVALID, "bad bounds");
    h->q_total_bound = total_queries; h->q_frame_bound = max_queries_per_frame;
    h->rows_bound = std::min(total_rows, (int)h->out_rows);   // a batch never has more rows than the handle's result capacity
    return ORB_OK;
}

extern "C" orb_status orbm_search_local_points(orbx_handle* h, const orbm_camera* cam, const orbm_local_queries* Q,
                                               float th, float nnratio, int32_t far_points, float th_far,
                                               int32_t* match_out, int32_t* nmatches_out) {
    if (!h || !cam || !Q || !match_out || Q->n_frames < 1 || !Q->frame_image || !Q->query_offset)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const bool dev = Q->on_device != 0;
    const bool bounded = dev && h->q_total_bound > 0;   // orbm_set_device_query_bounds: nothing is read back, no synchronisation
    const int nf = Q->n_frames;
    int nq, maxq, rows;
    orb_status s = frame_table(h, nf, Q->frame_image, Q->query_offset, dev, bounded, nq, maxq, rows);
    if (s != ORB_OK) return s;
    ProjParams P{};
    fill_frame_side(h, cam, P);
    P.mode = 0;
    P.th = th; P.nnratio = nnratio; P.bFar = far_points; P.thFar = th_far;
    auto layout = [&](Carve& c) {
        P.frame_image = stage_in(c, Q->frame_image, nf, dev); P.qoff = stage_in(c, Q->query_offset, nf + 1, dev);
        P.a0 = stage_in(c, Q->proj_x, nq, dev); P.a1 = stage_in(c, Q->proj_y, nq, dev); P.a2 = stage_in(c, Q->proj_xr, nq, dev);
        P.level = stage_in(c, Q->level, nq, dev); P.f0 = stage_in(c, Q->view_cos, nq, dev); P.f1 = stage_in(c, Q->track_depth, nq, dev);
        P.qdesc = stage_in(c, Q->desc, (size_t)nq * 32, dev); P.flag = stage_in(c, Q->feature_claimed, rows, dev);
        P.qvalid = stage_in(c, Q->in_view, nq, dev);
        P.gridOrder = c.take<uint16_t>((size_t)nf * P.maxFeat);
        P.gridStart = c.take<uint16_t>((size_t)nf * (GRID_COLS * GRID_ROWS + 1));
        P.topk = c.take<unsigned long long>((size_t)nq * PM_K);
        P.cnt = c.take<int>(nq);
        P.match = dev ? match_out : c.take<int>(nq);
        P.nmatches = (dev && nmatches_out) ? nmatches_out : c.take<int>(nf);
        P.seqFlag = c.take<int>(nf);
    };
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    ORB_CUDA(cudaMemsetAsync(P.seqFlag, 0, sizeof(int) * nf, h->stream));
    if (nq > 0 && (s = launch_proj(h, P, nf, maxq)) != ORB_OK) return s;
    if (dev && nq == 0 && nmatches_out) ORB_CUDA(cudaMemsetAsync(nmatches_out, 0, sizeof(int) * nf, h->stream));   // no kernel ran: a consumer must not see the previous step's counts
    if (!dev) {
        if (nq > 0) ORB_CUDA(cudaMemcpyAsync(match_out, P.match, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToHost, h->stream));
        if (nmatches_out && nq > 0) ORB_CUDA(cudaMemcpyAsync(nmatches_out, P.nmatches, sizeof(int) * nf, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaStreamSynchronize(h->stream));
        if (nmatches_out && nq == 0) std::fill(nmatches_out, nmatches_out + nf, 0);
    }
    return ORB_OK;
}

extern "C" orb_status orbm_search_last_frame(orbx_handle* h, const orbm_camera* cam, const orbm_last_queries* Q, float th,
                                             int32_t check_orientation, int32_t* feature_match_out, int32_t* nmatches_out) {
    if (!h || !cam || !Q || !feature_match_out || Q->n_frames < 1 || !Q->frame_image || !Q->query_offset || !Q->Tcw ||
        !Q->direction)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const bool dev = Q->on_device != 0;
    const bool bounded = dev && h->q_total_bound > 0;   // orbm_set_device_query_bounds: nothing is read back, no synchronisation
    const int nf = Q->n_frames;
    int nq, maxq, total_rows;
    orb_status s = frame_table(h, nf, Q->frame_image, Q->query_offset, dev, bounded, nq, maxq, total_rows);
    if (s != ORB_OK) return s;
    ProjParams P{};
    fill_frame_side(h, cam, P);
    P.mode = 1;
    P.th = th; P.checkOri = check_orientation;
    auto layout = [&](Carve& c) {
        P.frame_image = stage_in(c, Q->frame_image, nf, dev); P.qoff = stage_in(c, Q->query_offset, nf + 1, dev);
        P.Tcw = stage_in(c, Q->Tcw, (size_t)nf * 7, dev); P.direction = stage_in(c, Q->direction, nf, dev);
        P.a0 = stage_in(c, Q->world_pos, (size_t)nq * 3, dev); P.level = stage_in(c, Q->last_octave, nq, dev);
        P.f0 = stage_in(c, Q->last_angle, nq, dev); P.qdesc = stage_in(c, Q->desc, (size_t)nq * 32, dev);
        P.flag = stage_in(c, Q->obs_positive, nq, dev);
        P.gridOrder = c.take<uint16_t>((size_t)nf * P.maxFeat);
        P.gridStart = c.take<uint16_t>((size_t)nf * (GRID_COLS * GRID_ROWS + 1));
        P.topk = c.take<unsigned long long>((size_t)nq * PM_K);
        P.cnt = c.take<int>(nq);
        P.quv = c.take<float>(nq);
        P.match = dev ? feature_match_out : c.take<int>(total_rows);
        P.nmatches = (dev && nmatches_out) ? nmatches_out : c.take<int>(nf);
        P.seqFlag = c.take<int>(nf);
    };
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    ORB_CUDA(cudaMemsetAsync(P.match, 0xff, sizeof(int) * (size_t)total_rows, h->stream));
    ORB_CUDA(cudaMemsetAsync(P.seqFlag, 0, sizeof(int) * nf, h->stream));
    if ((s = launch_proj(h, P, nf, maxq)) != ORB_OK) return s;
    if (!dev) {
        ORB_CUDA(cudaMemcpyAsync(feature_match_out, P.match, sizeof(int) * (size_t)total_rows, cudaMemcpyDeviceToHost, h->stream));
        if (nmatches_out) ORB_CUDA(cudaMemcpyAsync(nmatches_out, P.nmatches, sizeof(int) * nf, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    }
    return ORB_OK;
}

extern "C" orb_status orbm_search_bow(orbx_handle* h, const orbm_bow_queries* Q, float nnratio, int32_t check_orientation,
                                      int32_t* feature_match_out, int32_t* nmatches_out) {
    if (!h || !Q || !feature_match_out || Q->n_frames < 1 || !Q->frame_image || !Q->query_offset || !Q->feature_node)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const bool dev = Q->on_device != 0;
    const int nf = Q->n_frames;
    int nq, maxq, total_rows;
    orb_status s = frame_table(h, nf, Q->frame_image, Q->query_offset, dev, false, nq, maxq, total_rows);
    if (s != ORB_OK) return s;
    ProjParams P{};
    orbm_camera cam{1, 1, 0, 0, 0, 1, 0, (float)h->cur_w, 0, (float)h->cur_h};   // the grid is not used by this search
    fill_frame_side(h, &cam, P);
    P.uright = nullptr;
    P.mode = 2;
    P.nnratio = nnratio; P.checkOri = check_orientation;
    auto layout = [&](Carve& c) {
        P.frame_image = stage_in(c, Q->frame_image, nf, dev); P.qoff = stage_in(c, Q->query_offset, nf + 1, dev);
        P.level = stage_in(c, Q->query_node, nq, dev); P.f0 = stage_in(c, Q->query_angle, nq, dev);
        P.qdesc = stage_in(c, Q->desc, (size_t)nq * 32, dev); P.feat_node = stage_in(c, Q->feature_node, total_rows, dev);
        P.topk = c.take<unsigned long long>((size_t)nq * PM_K);
        P.cnt = c.take<int>(nq);
        P.quv = c.take<float>(nq);
        P.match = dev ? feature_match_out : c.take<int>(total_rows);
        P.nmatches = (dev && nmatches_out) ? nmatches_out : c.take<int>(nf);
    };
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    ORB_CUDA(cudaMemsetAsync(P.match, 0xff, sizeof(int) * (size_t)total_rows, h->stream));
    if ((s = launch_proj(h, P, nf, maxq)) != ORB_OK) return s;
    if (!dev) {
        ORB_CUDA(cudaMemcpyAsync(feature_match_out, P.match, sizeof(int) * (size_t)total_rows, cudaMemcpyDeviceToHost, h->stream));
        if (nmatches_out) ORB_CUDA(cudaMemcpyAsync(nmatches_out, P.nmatches, sizeof(int) * nf, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    }
    return ORB_OK;
}

extern "C" orb_status orbm_search_keyframe(orbx_handle* h, const orbm_camera* cam, const orbm_kf_queries* Q, int32_t variant,
                                           float th, float hamming_max, int32_t check_orientation, int32_t* match_out,
                                           int32_t* nmatches_out) {
    if (!h || !cam || !Q || !match_out || Q->n_targets < 1 || !Q->query_offset || !Q->Tcw || !Q->Ow || variant < 0 || variant > 4 ||
        (variant == 4 && !Q->Sim3))
        return set_error(ORB_ERR_INVALID, "bad arguments");
    if (Q->kp ? (!Q->feat_offset || !Q->desc) : !Q->target_image) return set_error(ORB_ERR_INVALID, "bad target description");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const int nt = Q->n_targets;
    const int nq = Q->query_offset[nt];
    if (nq > 0 && (!Q->world_pos || !Q->max_dist || !Q->min_dist || !Q->desc_q || (variant < 3 && !Q->normal) ||
                   (variant == 3 && check_orientation && !Q->angle)))
        return set_error(ORB_ERR_INVALID, "missing query arrays");
    int maxq = 0;
    for (int t = 0; t < nt; ++t) {
        if (Q->query_offset[t + 1] < Q->query_offset[t]) return set_error(ORB_ERR_INVALID, "bad query table");
        maxq = std::max(maxq, Q->query_offset[t + 1] - Q->query_offset[t]);
    }
    ProjParams P{};
    int rows = 0;
    int maxFeat = 1;
    std::vector<int> img(nt), nkp(nt);
    orb_status s;
    if (Q->kp) {
        for (int t = 0; t < nt; ++t) {
            const int n = Q->feat_offset[t + 1] - Q->feat_offset[t];
            if (n < 0 || n > 5400) return set_error(ORB_ERR_UNSUPPORTED, "keyframe with more than 5400 features");
            img[t] = t;
            nkp[t] = n;
            maxFeat = std::max(maxFeat, n);
        }
        rows = Q->feat_offset[nt];
    } else {
        if ((s = batch_rows(h, &rows)) != ORB_OK) return s;
        for (int t = 0; t < nt; ++t) {
            img[t] = Q->target_image[t];
            if (img[t] < 0 || img[t] >= h->last_batch) return set_error(ORB_ERR_INVALID, "bad target image");
        }
        maxFeat = h->geom.kpTotal;
    }
    fill_frame_side(h, cam, P);
    P.mode = 3;
    P.variant = variant;
    if (Q->kp) P.maxFeat = maxFeat;
    P.th = th; P.thr = hamming_max; P.checkOri = (variant == 3) ? check_orientation : 0;
    P.nLevels = h->cfg.n_levels;
    P.logScale = logf((float)h->cfg.scale_factor);                       // Frame.cc:121 mfLogScaleFactor = log(mfScaleFactor)
    for (int l = 0; l < ORB_MAX_LEVELS; ++l) P.invSigma2[l] = l < h->cfg.n_levels ? h->inv_sigma2[l] : 1.f;
    auto layout = [&](Carve& c) {
        P.frame_image = stage_in(c, img.data(), nt, false); P.qoff = stage_in(c, Q->query_offset, nt + 1, false);
        if (Q->kp) {
            P.kps = stage_in(c, Q->kp, rows, false); P.desc = stage_in(c, Q->desc, (size_t)rows * 32, false);
            P.uright = stage_in(c, Q->uright, rows, false); P.offsets = stage_in(c, Q->feat_offset, nt, false);
            P.nkp = stage_in(c, nkp.data(), nt, false);
        }
        P.flag = stage_in(c, Q->feat_claimed, rows, false);
        P.S = stage_in(c, Q->Sim3, (size_t)nt * 8, false);
        P.Tcw = stage_in(c, Q->Tcw, (size_t)nt * 7, false); P.Ow = stage_in(c, Q->Ow, (size_t)nt * 3, false);
        P.a0 = stage_in(c, Q->world_pos, (size_t)nq * 3, false); P.normal = stage_in(c, Q->normal, (size_t)nq * 3, false);
        P.maxD = stage_in(c, Q->max_dist, nq, false); P.minD = stage_in(c, Q->min_dist, nq, false);
        P.f0 = stage_in(c, Q->angle, nq, false); P.qdesc = stage_in(c, Q->desc_q, (size_t)nq * 32, false);
        P.gridOrder = c.take<uint16_t>((size_t)nt * P.maxFeat);
        P.gridStart = c.take<uint16_t>((size_t)nt * (GRID_COLS * GRID_ROWS + 1));
        P.topk = c.take<unsigned long long>((size_t)nq * PM_K);
        P.cnt = c.take<int>(nq);
        P.quv = c.take<float>(nq);
        P.match = c.take<int>(nq);
        P.nmatches = c.take<int>(nt);
    };
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    if (nq > 0) {
        if ((s = launch_proj(h, P, nt, maxq)) != ORB_OK) return s;
        ORB_CUDA(cudaMemcpyAsync(match_out, P.match, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToHost, h->stream));
        if (nmatches_out) ORB_CUDA(cudaMemcpyAsync(nmatches_out, P.nmatches, sizeof(int) * nt, cudaMemcpyDeviceToHost, h->stream));
    }
    ORB_CUDA(cudaStreamSynchronize(h->stream));   // also keeps the host vectors alive until the uploads are done
    if (nmatches_out && nq == 0) std::fill(nmatches_out, nmatches_out + nt, 0);
    return ORB_OK;
}

extern "C" orb_status orbm_search_bow_keyframes(orbx_handle* h, const orbm_bow_kf_queries* Q, float nnratio, int32_t check_orientation,
                                                int32_t* match12_out, int32_t* nmatches_out) {
    if (!h || !Q || !match12_out || Q->n_pairs < 1 || !Q->feat_offset || !Q->query_offset || !Q->kp2 || !Q->desc2 || !Q->node2)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const int nt = Q->n_pairs;
    const int nq = Q->query_offset[nt];
    const size_t rows = (size_t)Q->feat_offset[nt];
    if (nq > 0 && (!Q->query_node || !Q->query_angle || !Q->desc1)) return set_error(ORB_ERR_INVALID, "missing query arrays");
    int maxq = 0, maxFeat = 1;
    std::vector<int> img(nt), nkp(nt);
    for (int t = 0; t < nt; ++t) {
        const int n = Q->feat_offset[t + 1] - Q->feat_offset[t];
        if (n < 0 || n > 5400) return set_error(ORB_ERR_UNSUPPORTED, "keyframe with more than 5400 features");
        if (Q->query_offset[t + 1] < Q->query_offset[t]) return set_error(ORB_ERR_INVALID, "bad query table");
        img[t] = t;
        nkp[t] = n;
        maxFeat = std::max(maxFeat, n);
        maxq = std::max(maxq, Q->query_offset[t + 1] - Q->query_offset[t]);
    }
    std::vector<uint8_t> invalid(std::max<size_t>(rows, 1), 0);   // vbMatched2 starts false; features without a good map point never match
    if (Q->valid2)
        for (size_t i = 0; i < rows; ++i) invalid[i] = Q->valid2[i] ? 0 : 1;
    ProjParams P{};
    orbm_camera cam{1, 1, 0, 0, 0, 1, 0, 1, 0, 1};   // the grid is not used by this search
    fill_frame_side(h, &cam, P);
    P.mode = 2;
    P.variant = 1;
    P.uright = nullptr; P.maxFeat = maxFeat;
    P.nnratio = nnratio; P.checkOri = check_orientation;
    auto layout = [&](Carve& c) {
        P.frame_image = stage_in(c, img.data(), nt, false); P.qoff = stage_in(c, Q->query_offset, nt + 1, false);
        P.kps = stage_in(c, Q->kp2, rows, false); P.desc = stage_in(c, Q->desc2, rows * 32, false);
        P.offsets = stage_in(c, Q->feat_offset, nt, false); P.nkp = stage_in(c, nkp.data(), nt, false);
        P.feat_node = stage_in(c, Q->node2, rows, false); P.flag = stage_in(c, invalid.data(), rows, false);
        P.level = stage_in(c, Q->query_node, nq, false); P.f0 = stage_in(c, Q->query_angle, nq, false);
        P.qdesc = stage_in(c, Q->desc1, (size_t)nq * 32, false);
        P.topk = c.take<unsigned long long>((size_t)nq * PM_K);
        P.cnt = c.take<int>(nq);
        P.quv = c.take<float>(nq);
        P.match = c.take<int>(nq);
        P.nmatches = c.take<int>(nt);
    };
    orb_status s;
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    if (nq > 0) {
        if ((s = launch_proj(h, P, nt, maxq)) != ORB_OK) return s;
        ORB_CUDA(cudaMemcpyAsync(match12_out, P.match, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToHost, h->stream));
        if (nmatches_out) ORB_CUDA(cudaMemcpyAsync(nmatches_out, P.nmatches, sizeof(int) * nt, cudaMemcpyDeviceToHost, h->stream));
    }
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    if (nmatches_out && nq == 0) std::fill(nmatches_out, nmatches_out + nt, 0);
    return ORB_OK;
}

extern "C" orb_status orbm_search_initialization(orbx_handle* h, const orbm_camera* cam, const orbm_init_queries* Q, int32_t window_size,
                                                 float nnratio, int32_t check_orientation, int32_t* matches12_out, int32_t* nmatches_out) {
    if (!h || !cam || !Q || !matches12_out || Q->n1 < 0 || (Q->kp2 ? (!Q->desc2 || Q->n2 < 0) : Q->target_image < 0))
        return set_error(ORB_ERR_INVALID, "bad arguments");
    if (Q->n1 > 0 && (!Q->kp1 || !Q->desc1 || !Q->prev_matched)) return set_error(ORB_ERR_INVALID, "missing query arrays");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const int nq = Q->n1;
    orb_status s;
    size_t rows = 0;
    int img = 0, nkp_h = 0, off_h = 0;
    if (Q->kp2) {
        if (Q->n2 > 4700) return set_error(ORB_ERR_UNSUPPORTED, "frame with more than 4700 features");
        rows = (size_t)Q->n2;
        nkp_h = Q->n2;
    } else {
        if ((s = orbx_counts(h, nullptr, nullptr, nullptr)) != ORB_OK) return s;
        if (Q->target_image >= h->last_batch) return set_error(ORB_ERR_INVALID, "bad target image");
        img = Q->target_image;
    }
    std::vector<float> px(std::max(nq, 1)), py(std::max(nq, 1)), ang(std::max(nq, 1));
    std::vector<int> lvl(std::max(nq, 1));
    for (int i = 0; i < nq; ++i) {
        px[i] = Q->prev_matched[2 * i];
        py[i] = Q->prev_matched[2 * i + 1];
        ang[i] = Q->kp1[i].angle;
        lvl[i] = Q->kp1[i].octave;
    }
    const int qoff_h[2] = {0, nq};
    ProjParams P{};
    fill_frame_side(h, cam, P);
    P.uright = nullptr;
    P.mode = 4;
    if (Q->kp2) P.maxFeat = std::max(Q->n2, 1);
    P.th = (float)window_size;     // GetFeaturesInArea(x, y, windowSize, ...): int -> const float& r
    P.nnratio = nnratio; P.checkOri = check_orientation;
    auto layout = [&](Carve& c) {
        P.frame_image = stage_in(c, &img, 1, false); P.qoff = stage_in(c, qoff_h, 2, false);
        if (Q->kp2) {
            P.kps = stage_in(c, Q->kp2, rows, false); P.desc = stage_in(c, Q->desc2, rows * 32, false);
            P.offsets = stage_in(c, &off_h, 1, false); P.nkp = stage_in(c, &nkp_h, 1, false);
        }
        P.a0 = stage_in(c, px.data(), nq, false); P.a1 = stage_in(c, py.data(), nq, false);
        P.f0 = stage_in(c, ang.data(), nq, false); P.level = stage_in(c, lvl.data(), nq, false);
        P.qdesc = stage_in(c, Q->desc1, (size_t)nq * 32, false);
        P.gridOrder = c.take<uint16_t>((size_t)P.maxFeat);
        P.gridStart = c.take<uint16_t>((size_t)(GRID_COLS * GRID_ROWS + 1));
        P.topk = c.take<unsigned long long>((size_t)nq * PM_K);
        P.cnt = c.take<int>(nq);
        P.quv = c.take<float>(nq);
        P.match = c.take<int>(nq);
        P.nmatches = c.take<int>(1);
    };
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    if (nq > 0) {
        if ((s = launch_proj(h, P, 1, nq)) != ORB_OK) return s;
        ORB_CUDA(cudaMemcpyAsync(matches12_out, P.match, sizeof(int) * (size_t)nq, cudaMemcpyDeviceToHost, h->stream));
        if (nmatches_out) ORB_CUDA(cudaMemcpyAsync(nmatches_out, P.nmatches, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    }
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    if (nmatches_out && nq == 0) *nmatches_out = 0;
    return ORB_OK;
}

extern "C" orb_status orbf_is_in_frustum(orbx_handle* h, const orbm_camera* cam, const orbf_frustum_points* in, float viewing_cos_limit,
                                         uint8_t* in_view_out, float* proj_x_out, float* proj_y_out, float* proj_xr_out, int32_t* level_out,
                                         float* view_cos_out, float* track_depth_out) {
    if (!h || !cam || !in || in->n_frames < 1 || !in->point_offset || !in->Rcw || !in->tcw || !in->Ow || !in_view_out || !proj_x_out ||
        !proj_y_out || !proj_xr_out || !level_out || !view_cos_out || !track_depth_out)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const bool dev = in->on_device != 0;
    const int nf = in->n_frames;
    if (dev && in->n_points_max < 0) return set_error(ORB_ERR_INVALID, "n_points_max is required for device callers");
    const int np = dev ? in->n_points_max : in->point_offset[nf];
    int maxp = np;                                   // grid.x covers the largest frame; device callers: the total bound
    if (!dev) {
        maxp = 0;
        for (int f = 0; f < nf; ++f) {
            if (in->point_offset[f + 1] < in->point_offset[f]) return set_error(ORB_ERR_INVALID, "bad point table");
            maxp = std::max(maxp, in->point_offset[f + 1] - in->point_offset[f]);
        }
    }
    if (np > 0 && (!in->world_pos || !in->normal || !in->max_dist || !in->min_dist)) return set_error(ORB_ERR_INVALID, "missing point arrays");
    FrustumParams P{};
    P.fx = cam->fx; P.fy = cam->fy; P.cx = cam->cx; P.cy = cam->cy; P.bf = cam->bf;
    P.minX = cam->min_x; P.maxX = cam->max_x; P.minY = cam->min_y; P.maxY = cam->max_y;
    P.logScale = logf((float)h->cfg.scale_factor);
    P.cosLimit = viewing_cos_limit;
    P.nLevels = h->cfg.n_levels;
    auto layout = [&](Carve& c) {
        P.poff = stage_in(c, in->point_offset, nf + 1, dev); P.Rcw = stage_in(c, in->Rcw, (size_t)nf * 9, dev);
        P.tcw = stage_in(c, in->tcw, (size_t)nf * 3, dev); P.Ow = stage_in(c, in->Ow, (size_t)nf * 3, dev);
        P.xw = stage_in(c, in->world_pos, (size_t)np * 3, dev); P.normal = stage_in(c, in->normal, (size_t)np * 3, dev);
        P.maxD = stage_in(c, in->max_dist, np, dev); P.minD = stage_in(c, in->min_dist, np, dev);
        P.in_view = dev ? in_view_out : c.take<uint8_t>(np);
        P.px = dev ? proj_x_out : c.take<float>(np);
        P.py = dev ? proj_y_out : c.take<float>(np);
        P.pxr = dev ? proj_xr_out : c.take<float>(np);
        P.vc = dev ? view_cos_out : c.take<float>(np);
        P.depth = dev ? track_depth_out : c.take<float>(np);
        P.level = dev ? level_out : c.take<int>(np);
    };
    orb_status s;
    if ((s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout)) != ORB_OK) return s;
    if (maxp > 0) {
        k_in_frustum<<<dim3((maxp + 255) / 256, nf), 256, 0, h->stream>>>(P);
        ORB_LAUNCHED();
        ORB_CUDA(cudaGetLastError());
    }
    if (!dev) {
        if (np > 0) {
            ORB_CUDA(cudaMemcpyAsync(in_view_out, P.in_view, (size_t)np, cudaMemcpyDeviceToHost, h->stream));
            ORB_CUDA(cudaMemcpyAsync(proj_x_out, P.px, sizeof(float) * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
            ORB_CUDA(cudaMemcpyAsync(proj_y_out, P.py, sizeof(float) * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
            ORB_CUDA(cudaMemcpyAsync(proj_xr_out, P.pxr, sizeof(float) * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
            ORB_CUDA(cudaMemcpyAsync(level_out, P.level, sizeof(int) * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
            ORB_CUDA(cudaMemcpyAsync(view_cos_out, P.vc, sizeof(float) * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
            ORB_CUDA(cudaMemcpyAsync(track_depth_out, P.depth, sizeof(float) * (size_t)np, cudaMemcpyDeviceToHost, h->stream));
        }
        ORB_CUDA(cudaStreamSynchronize(h->stream));
    }
    return ORB_OK;
}
