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
//
// The kernel bodies live in matcher_core.cuh.  This file builds them in two forms: the shared-memory form, which stages the searched
// frame in each CTA, and the global-memory form (*_xl) for frames too large for that (launch_proj picks one per call).
#include <algorithm>
#include <vector>

#include "extractor.h"
#include "matcher_core.cuh"

using namespace orb;
using namespace orbdev;

namespace orb {

// ---- Frame::AssignFeaturesToGrid (Frame.cc:469-504) as a CSR table: feature ids sorted by (cell, id) -------------
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

// ---- the search kernels, shared-memory form (bodies: matcher_core.cuh) -------------------------------------------------
template <int G>
__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates_grp(const __grid_constant__ ProjParams P) {
    proj_candidates_grp_body<G>(P, SmemFrame{});
}

__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates(const __grid_constant__ ProjParams P) {
    proj_candidates_body(P, SmemFrame{});
}

__global__ void __launch_bounds__(256) k_proj_resolve(const __grid_constant__ ProjParams P) {
    const SmemFrame S{};
#include "matcher_resolve.inc"
}

__global__ void __launch_bounds__(PR_THREADS) k_proj_resolve_par(const __grid_constant__ ProjParams P) {
    const SmemFrame S{};
#include "matcher_resolve_par.inc"
}

// ---- the same kernels, global-memory form ---------------------------------------------------------------------------------
// One CTA per frame writes the FrameFeat block (and for the grid searches the GridFeat block, after k_frame_grid) that the
// shared-memory form stages in every CTA.
__global__ void __launch_bounds__(1024) k_stage_frames_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
    const int frame = blockIdx.x;
    FrameFeat F;
    int N, row0;
    stage_frame(P, P.frame_image[frame], S.featBlocks + (size_t)frame * S.featStride, F, N, row0);
    if (S.gridBlocks) {
        GridFeat GF;
        stage_grid(P, frame, S.gridBlocks + (size_t)frame * S.gridStride, GF, N, row0);
    }
}

template <int G>
__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates_grp_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
    proj_candidates_grp_body<G>(P, S);
}

__global__ void __launch_bounds__(PM_WARPS * 32) k_proj_candidates_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
    proj_candidates_body(P, S);
}

__global__ void __launch_bounds__(256) k_proj_resolve_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
#include "matcher_resolve.inc"
}

__global__ void __launch_bounds__(PR_THREADS) k_proj_resolve_par_xl(const __grid_constant__ ProjParams P, const GlobalFrame S) {
#include "matcher_resolve_par.inc"
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
// Runs one search.  The call's shared-memory need (the largest block its kernels ask for) decides the form, once per call: the
// shared-memory form whenever the device can give it, else the global-memory form (*_xl), whose frame blocks live in
// h->d_xl and whose kernels keep only the per-feature resolve state in shared memory.  Both compute the same matches.  A search
// without queries launches nothing and zeroes its counts, so no caller sees an earlier call's.
static orb_status launch_proj(orbx_handle* h, ProjParams& P, int n_frames, int n_queries, int max_q_per_frame) {
    cudaStream_t st = h->stream;
    if (n_queries == 0) {
        ORB_CUDA(cudaMemsetAsync(P.nmatches, 0, sizeof(int) * n_frames, st));
        return ORB_OK;
    }
    const size_t fsm = ((size_t)P.maxFeat * 23 + 16 + 15) / 16 * 16;                       // the staged frame
    const size_t gsm = ((size_t)P.maxFeat * 17 + (PM_NCELL + 1) * 2 + 32 + 15) / 16 * 16;  // the staged grid
    const size_t csm = std::max(fsm, gsm);
    // the resolve kernels' own arrays, after the staged frame
    const size_t pown = (size_t)P.maxFeat * 9 + (size_t)(PR_QCAP + PR_LIST) * 4 + 64;
    const size_t rown = (size_t)PM_CHUNK * PM_K * 8 + (size_t)PM_CHUNK * 4 + (size_t)P.maxFeat * (P.mode == 4 ? 9 : 5) + (size_t)PM_CHUNK * 5 + 256;
    // static __shared__ arrays count against the same limit; the *_xl kernels share the resolve bodies and so their static arrays
    static const size_t candStatic = std::max({static_smem(k_proj_candidates), static_smem(k_proj_candidates_grp<4>),
                                               static_smem(k_proj_candidates_grp<8>), static_smem(k_proj_candidates_grp<16>)});
    static const size_t parStatic = static_smem(k_proj_resolve_par), resStatic = static_smem(k_proj_resolve);
    const size_t optin = (size_t)smem_optin(h);
    const bool global = csm + candStatic > optin || (P.seqFlag && fsm + pown + parStatic > optin) || fsm + rown + resStatic > optin;
    GlobalFrame S{};
    orb_status s;
    if (global) {   // the same kernels without the staged frame in shared memory
        if ((P.seqFlag && (s = check_smem(h, pown, parStatic, "k_proj_resolve_par_xl")) != ORB_OK) ||
            (s = check_smem(h, rown, resStatic, "k_proj_resolve_xl")) != ORB_OK)
            return s;
        S.featStride = (fsm + 255) / 256 * 256;
        S.gridStride = (gsm + 255) / 256 * 256;
        auto layout = [&](Carve& c) {
            S.featBlocks = c.take<unsigned char>((size_t)n_frames * S.featStride);
            S.gridBlocks = P.mode != 2 ? c.take<unsigned char>((size_t)n_frames * S.gridStride) : nullptr;
        };
        if ((s = carve_scratch(h->xl_bytes, h->d_xl, h->capturing, st, layout).status) != ORB_OK) return s;
    }
    // One kernel role: the shared-memory kernel with `staged` bytes of frame or grid ahead of its `own` bytes, or its *_xl twin with
    // only its own bytes and the frame blocks S.  An empty grid launches nothing.
    auto run = [&](auto kern, auto kern_xl, dim3 grid, int threads, size_t staged, size_t own) -> orb_status {
        const size_t smem = global ? own : staged + own;
        if (smem) ORB_CUDA(global ? cudaFuncSetAttribute(kern_xl, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                                  : cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (grid.x == 0) return ORB_OK;
        if (global) launch_p(kern_xl, grid, dim3(threads), smem, st, P, S);
        else launch_p(kern, grid, dim3(threads), smem, st, P);
        ORB_LAUNCHED();
        return ORB_OK;
    };
    if (P.mode != 2) {   // modes 0, 1, 3 search a window of the feature grid
        const size_t gridSm = (size_t)(PM_NCELL + 2) * 4 + (size_t)P.maxFeat * 4 + 16;
        static const size_t gridStatic = static_smem(k_frame_grid);
        if ((s = check_smem(h, gridSm, gridStatic, "k_frame_grid")) != ORB_OK) return s;
        ORB_CUDA(cudaFuncSetAttribute(k_frame_grid, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(gridSm, (size_t)1024)));
        launch_p(k_frame_grid, dim3(n_frames), dim3(256), gridSm, st, P);
        ORB_LAUNCHED();
    }
    if (global) {
        launch_p(k_stage_frames_xl, dim3(n_frames), dim3(1024), 0, st, P, S);
        ORB_LAUNCHED();
    }
    // modes 0 / 1 (the two per-frame searches): G lanes per query (ORB_PROJ_LANES = 4 | 8 | 16; 32 = the warp-per-query kernel)
    const char* vLanes = getenv("ORB_PROJ_LANES");
    const char* vQpb = getenv("ORB_PROJ_QPB");
    const int envLanes = vLanes ? atoi(vLanes) : 0, envQpb = vQpb ? atoi(vQpb) : 0;
    const int lanes = P.mode > 1 ? 32 : (envLanes ? envLanes : (P.mode == 0 ? 4 : 8));
    auto cand = k_proj_candidates;
    auto cand_xl = k_proj_candidates_xl;
    int qpb = PM_QPB;
    if (lanes == 4 || lanes == 8 || lanes == 16) {
        qpb = P.qpb = envQpb > 0 ? envQpb : (P.mode == 0 ? 128 : 64);
        cand = lanes == 4 ? k_proj_candidates_grp<4> : (lanes == 8 ? k_proj_candidates_grp<8> : k_proj_candidates_grp<16>);
        cand_xl = lanes == 4 ? k_proj_candidates_grp_xl<4> : (lanes == 8 ? k_proj_candidates_grp_xl<8> : k_proj_candidates_grp_xl<16>);
    }
    if ((s = run(cand, cand_xl, dim3((max_q_per_frame + qpb - 1) / qpb, n_frames), PM_WARPS * 32, csm, 0)) != ORB_OK) return s;
    // modes 0 / 1: parallel fixed-point resolve; frames it cannot finish are flagged for the sequential kernel
    if (P.seqFlag && (s = run(k_proj_resolve_par, k_proj_resolve_par_xl, dim3(n_frames), PR_THREADS, fsm, pown)) != ORB_OK) return s;
    if ((s = run(k_proj_resolve, k_proj_resolve_xl, dim3(n_frames), 256, fsm, rown)) != ORB_OK) return s;
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
    if (nq > 0 && (!Q->proj_x || !Q->proj_y || !Q->proj_xr || !Q->level || !Q->view_cos || !Q->desc))
        return set_error(ORB_ERR_INVALID, "missing query arrays");
    ProjParams P{};
    fill_frame_side(h, cam, P);
    if ((s = check_frame_rows(P.maxFeat, "frame")) != ORB_OK) return s;
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
        P.match = stage_out(c, match_out, nq, dev);
        P.nmatches = stage_out(c, nmatches_out, nf, dev);
        P.seqFlag = c.take<int>(nf);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    ORB_CUDA(cudaMemsetAsync(P.seqFlag, 0, sizeof(int) * nf, h->stream));
    if ((s = launch_proj(h, P, nf, nq, maxq)) != ORB_OK) return s;
    return dev ? ORB_OK : copy_out(c);
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
    if (nq > 0 && (!Q->world_pos || !Q->last_octave || !Q->last_angle || !Q->desc)) return set_error(ORB_ERR_INVALID, "missing query arrays");
    ProjParams P{};
    fill_frame_side(h, cam, P);
    if ((s = check_frame_rows(P.maxFeat, "frame")) != ORB_OK) return s;
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
        P.match = stage_out(c, feature_match_out, total_rows, dev);
        P.nmatches = stage_out(c, nmatches_out, nf, dev);
        P.seqFlag = c.take<int>(nf);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    ORB_CUDA(cudaMemsetAsync(P.match, 0xff, sizeof(int) * (size_t)total_rows, h->stream));
    ORB_CUDA(cudaMemsetAsync(P.seqFlag, 0, sizeof(int) * nf, h->stream));
    if ((s = launch_proj(h, P, nf, nq, maxq)) != ORB_OK) return s;
    return dev ? ORB_OK : copy_out(c);
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
    if (nq > 0 && (!Q->query_node || !Q->query_angle || !Q->desc)) return set_error(ORB_ERR_INVALID, "missing query arrays");
    ProjParams P{};
    orbm_camera cam{1, 1, 0, 0, 0, 1, 0, (float)h->cur_w, 0, (float)h->cur_h};   // the grid is not used by this search
    fill_frame_side(h, &cam, P);
    if ((s = check_frame_rows(P.maxFeat, "frame")) != ORB_OK) return s;
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
        P.match = stage_out(c, feature_match_out, total_rows, dev);
        P.nmatches = stage_out(c, nmatches_out, nf, dev);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    ORB_CUDA(cudaMemsetAsync(P.match, 0xff, sizeof(int) * (size_t)total_rows, h->stream));
    if ((s = launch_proj(h, P, nf, nq, maxq)) != ORB_OK) return s;
    return dev ? ORB_OK : copy_out(c);
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
            if (n < 0) return set_error(ORB_ERR_UNSUPPORTED, "keyframe with a negative feature count");
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
    if ((s = check_frame_rows(P.maxFeat, Q->kp ? "keyframe" : "frame")) != ORB_OK) return s;
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
        P.match = stage_out(c, match_out, nq, false);
        P.nmatches = stage_out(c, nmatches_out, nt, false);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    if ((s = launch_proj(h, P, nt, nq, maxq)) != ORB_OK) return s;
    return copy_out(c);   // also keeps the host vectors alive until the uploads are done
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
    orb_status s;
    for (int t = 0; t < nt; ++t) {
        const int n = Q->feat_offset[t + 1] - Q->feat_offset[t];
        if (n < 0) return set_error(ORB_ERR_UNSUPPORTED, "keyframe with a negative feature count");
        if ((s = check_frame_rows(n, "keyframe")) != ORB_OK) return s;
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
        P.match = stage_out(c, match12_out, nq, false);
        P.nmatches = stage_out(c, nmatches_out, nt, false);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    if ((s = launch_proj(h, P, nt, nq, maxq)) != ORB_OK) return s;
    return copy_out(c);
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
    if ((s = check_frame_rows(P.maxFeat, "frame")) != ORB_OK) return s;
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
        P.match = stage_out(c, matches12_out, nq, false);
        P.nmatches = stage_out(c, nmatches_out, 1, false);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    if ((s = launch_proj(h, P, 1, nq, nq)) != ORB_OK) return s;
    return copy_out(c);
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
        P.in_view = stage_out(c, in_view_out, np, dev);
        P.px = stage_out(c, proj_x_out, np, dev);
        P.py = stage_out(c, proj_y_out, np, dev);
        P.pxr = stage_out(c, proj_xr_out, np, dev);
        P.vc = stage_out(c, view_cos_out, np, dev);
        P.depth = stage_out(c, track_depth_out, np, dev);
        P.level = stage_out(c, level_out, np, dev);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    if (maxp > 0) {
        k_in_frustum<<<dim3((maxp + 255) / 256, nf), 256, 0, h->stream>>>(P);
        ORB_LAUNCHED();
        ORB_CUDA(cudaGetLastError());
    }
    return dev ? ORB_OK : copy_out(c);
}
