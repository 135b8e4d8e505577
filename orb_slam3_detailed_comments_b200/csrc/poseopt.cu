// poseopt.cu -- Optimizer::PoseOptimization(Frame*) on the device, Nleft == -1
//   /root/reference/src/Optimizer.cc:55-412 (called twice per frame by the tracking thread: Tracking.cc:3222, 3443, 3522)
// One VertexSE3Expmap and unary edges EdgeSE3ProjectXYZOnlyPose (src/OptimizableTypes.cpp) /
// EdgeStereoSE3ProjectXYZOnlyPose (Thirdparty/g2o/g2o/types/types_six_dof_expmap.cpp:339-404); g2o Levenberg over a dense
// 6 x 6 system; 4 rounds of 10 iterations that restart from the frame's pose; chi2 classification after every round
// (5.991 / 7.815 as floats); the robust kernel is dropped after round 2.
//
// One CTA per frame, a batch of frames per launch.  The edges are spread over the threads; every thread carries the pose,
// lambda and the LM control state replicated in registers (the robust chi2 comes out of a butterfly + fixed-order warp sum
// that gives every thread bit-identical values, so accept / reject needs no broadcast), while the 6 x 6 system is summed,
// factorised (LDL^T) and applied (exponential map) by thread 0 only and the new pose is handed over through shared memory.
#include <algorithm>
#include <vector>

#include "extractor.h"
#include "ba_math.cuh"

using namespace orb;

namespace orb {

#define PO_THREADS 256
#define PO_WARPS (PO_THREADS / 32)

struct PoseOptParams {
    const int* eoff;          // [n_frames + 1]
    const float* pose;        // [n_frames][7]
    const float* xw;          // [ne][3]
    const float* obs;         // [ne][3]
    const float* invs2;       // [ne]
    double fx, fy, cx, cy, bf;
    double* err;              // [ne] scratch: e->chi2() as left by the last computeActiveErrors
    uint8_t* outlier;         // [ne] out (doubles as the edge level)
    double* pose_out;         // [n_frames][7]
    int* inliers;             // [n_frames]
    int* stats;               // [n_frames][4] rounds, LM iterations, LM trials, -
};

__device__ __forceinline__ double po_block_sum(double v, double* s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                               // s_red free again
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = s_red[0];
#pragma unroll
    for (int w = 1; w < PO_WARPS; ++w) s += s_red[w];
    return s;
}

// residual of one edge at pose T; returns the dimension (2 mono, 3 stereo)
__device__ __forceinline__ int po_edge_error(const PoseOptParams& P, const double* T, int e, double r[3], double Xc[3]) {
    const double X[3] = {(double)P.xw[3 * (size_t)e], (double)P.xw[3 * (size_t)e + 1], (double)P.xw[3 * (size_t)e + 2]};
    se3_map(T, X, Xc);
    const double z0 = (double)P.obs[3 * (size_t)e], z1 = (double)P.obs[3 * (size_t)e + 1], z2 = (double)P.obs[3 * (size_t)e + 2];
    if (z2 < 0) {   // EdgeSE3ProjectXYZOnlyPose::computeError + Pinhole::project(Vector3d)
        r[0] = z0 - (P.fx * Xc[0] / Xc[2] + P.cx);
        r[1] = z1 - (P.fy * Xc[1] / Xc[2] + P.cy);
        r[2] = 0;
        return 2;
    }
    const double invz = (double)__fdiv_rn(1.0f, (float)Xc[2]);   // cam_project: const float invz = 1.0f/trans_xyz[2]
    const double u = Xc[0] * invz * P.fx + P.cx;
    r[0] = z0 - u;
    r[1] = z1 - (Xc[1] * invz * P.fy + P.cy);
    r[2] = z2 - (u - P.bf * invz);
    return 3;
}

__global__ void __launch_bounds__(PO_THREADS) k_pose_opt(const __grid_constant__ PoseOptParams P) {
    __shared__ double s_red[PO_WARPS];
    __shared__ double s_part[PO_WARPS][27];
    __shared__ double s_T[7], s_scale, s_md;
    __shared__ int s_ok2;
    const int frame = blockIdx.x, tid = threadIdx.x;
    const int e0 = P.eoff[frame], n = P.eoff[frame + 1] - e0;
    double pose0[7], T[7];
#pragma unroll
    for (int i = 0; i < 7; ++i) pose0[i] = T[i] = (double)P.pose[7 * frame + i];
    if (n < 3) {   // Optimizer.cc:292-293: return 0, the frame keeps its pose
        if (tid == 0) {
            for (int i = 0; i < 7; ++i) P.pose_out[7 * frame + i] = pose0[i];
            P.inliers[frame] = 0;
            P.stats[4 * frame] = P.stats[4 * frame + 1] = P.stats[4 * frame + 2] = 0;
        }
        for (int e = tid; e < n; e += PO_THREADS) P.outlier[e0 + e] = 0;
        return;
    }
    const double dM = (double)(float)sqrt(5.991), dS = (double)(float)sqrt(7.815);       // const float deltaMono / deltaStereo
    const double sqM = (double)(float)(dM * dM), sqS = (double)(float)(dS * dS);           // RobustKernelHuber::dsqr
    for (int e = tid; e < n; e += PO_THREADS) P.outlier[e0 + e] = 0;
    bool robust = true;
    int nBadEdges = 0, rounds = 0, totalIters = 0, totalTrials = 0;

    auto compute_errors = [&](const double* pose) -> double {   // computeActiveErrors + activeRobustChi2 (level-0 edges)
        double chi = 0;
        for (int e = tid; e < n; e += PO_THREADS) {
            if (P.outlier[e0 + e]) continue;
            double r[3], Xc[3];
            const int D = po_edge_error(P, pose, e0 + e, r, Xc);
            const double c = (double)P.invs2[e0 + e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
            P.err[e0 + e] = c;
            double w;
            chi += robust ? huber_rho(c, D == 2 ? dM : dS, D == 2 ? sqM : sqS, &w) : c;
        }
        return po_block_sum(chi, s_red);
    };

    for (int it = 0; it < 4; ++it) {
#pragma unroll
        for (int i = 0; i < 7; ++i) T[i] = pose0[i];             // vSE3->setEstimate(pFrame->GetPose())
        int nActive = 0;
        for (int e = tid; e < n; e += PO_THREADS) nActive += P.outlier[e0 + e] == 0;
        nActive = (int)po_block_sum((double)nActive, s_red);
        if (nActive > 0) {
            double lambda = 0, ni = 2, currentChi = 0;
            int nBadIt = 0;
            for (int iter = 0; iter < 10; ++iter) {
                currentChi = compute_errors(T);
                double tempChi = currentChi;
                const double iniChi = currentChi;
                // ---- buildSystem: H (upper triangle, 21) and b (6) ------------------------------------------------
                double acc[27];
#pragma unroll
                for (int i = 0; i < 27; ++i) acc[i] = 0;
                for (int e = tid; e < n; e += PO_THREADS) {
                    if (P.outlier[e0 + e]) continue;
                    double r[3], Xc[3], B[18];
                    const int D = po_edge_error(P, T, e0 + e, r, Xc);
                    pose_jacobian(D, P.fx, P.fy, P.bf, Xc, B);
                    const double c2 = (double)P.invs2[e0 + e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
                    double w = 1.0;
                    if (robust) huber_rho(c2, D == 2 ? dM : dS, D == 2 ? sqM : sqS, &w);
                    const double om = w * (double)P.invs2[e0 + e];
                    int k = 0;
#pragma unroll
                    for (int i = 0; i < 6; ++i) {
#pragma unroll
                        for (int j = i; j < 6; ++j) {
                            double s = B[i] * B[j] + B[6 + i] * B[6 + j];
                            if (D == 3) s += B[12 + i] * B[12 + j];
                            acc[k++] += om * s;
                        }
                        double s = B[i] * r[0] + B[6 + i] * r[1];
                        if (D == 3) s += B[12 + i] * r[2];
                        acc[21 + i] += -om * s;
                    }
                }
#pragma unroll
                for (int i = 0; i < 27; ++i) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], o);
                }
                __syncthreads();
                if ((tid & 31) == 0)
                    for (int i = 0; i < 27; ++i) s_part[tid >> 5][i] = acc[i];
                __syncthreads();
                double H[36], b[6];          // live in thread 0 only
                if (tid == 0) {
                    int k = 0;
                    for (int i = 0; i < 6; ++i)
                        for (int j = i; j < 6; ++j) {
                            double s = s_part[0][k];
                            for (int w = 1; w < PO_WARPS; ++w) s += s_part[w][k];
                            H[6 * i + j] = H[6 * j + i] = s;
                            ++k;
                        }
                    for (int i = 0; i < 6; ++i) {
                        double s = s_part[0][21 + i];
                        for (int w = 1; w < PO_WARPS; ++w) s += s_part[w][21 + i];
                        b[i] = s;
                    }
                    double md = 0;
                    for (int j = 0; j < 6; ++j) md = fmax(fabs(H[7 * j]), md);
                    s_md = md;
                }
                if (iter == 0) {   // computeLambdaInit: tau * max diagonal
                    __syncthreads();
                    lambda = 1e-5 * s_md;
                    ni = 2;
                    nBadIt = 0;
                }
                double rho = 0;
                int qmax = 0;
                do {
                    double saved[7];
#pragma unroll
                    for (int i = 0; i < 7; ++i) saved[i] = T[i];                 // push
                    if (tid == 0) {
                        double x[6], Tn[7];
                        s_ok2 = ldlt6_solve(H, lambda, b, x) ? 1 : 0;
#pragma unroll
                        for (int i = 0; i < 7; ++i) Tn[i] = T[i];
                        pose_oplus(Tn, x);
#pragma unroll
                        for (int i = 0; i < 7; ++i) s_T[i] = Tn[i];
                        double sc = 0;
                        for (int j = 0; j < 6; ++j) sc += x[j] * (lambda * x[j] + b[j]);
                        s_scale = sc;
                    }
                    __syncthreads();
#pragma unroll
                    for (int i = 0; i < 7; ++i) T[i] = s_T[i];
                    const bool ok2 = s_ok2 != 0;
                    const double scale = s_scale + 1e-3;
                    tempChi = compute_errors(T);     // its barriers also fence s_T / s_scale against the next trial
                    if (!ok2) tempChi = 1.7976931348623157e308;
                    rho = currentChi - tempChi;
                    rho /= scale;
                    if (rho > 0 && isfinite(tempChi)) {
                        double alpha = 2 * rho - 1;
                        alpha = 1. - alpha * alpha * alpha;
                        alpha = fmin(alpha, 2. / 3.);
                        lambda *= fmax(1. / 3., alpha);
                        ni = 2;
                        currentChi = tempChi;
                    } else {
                        lambda *= ni;
                        ni *= 2;
#pragma unroll
                        for (int i = 0; i < 7; ++i) T[i] = saved[i];             // pop
                    }
                    ++qmax;
                    ++totalTrials;
                } while (rho < 0 && qmax < 10);
                ++totalIters;
                if (qmax == 10 || rho == 0) break;
                if ((iniChi - currentChi) * 1e3 < iniChi) ++nBadIt; else nBadIt = 0;
                if (nBadIt >= 3) break;
            }
        }
        // ---- classification (Optimizer.cc:312-390) ------------------------------------------------------------------
        int bad = 0;
        for (int e = tid; e < n; e += PO_THREADS) {
            double c = P.err[e0 + e];
            if (P.outlier[e0 + e]) {           // e->computeError() for the edges the optimiser did not touch
                double r[3], Xc[3];
                po_edge_error(P, T, e0 + e, r, Xc);
                c = (double)P.invs2[e0 + e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
                P.err[e0 + e] = c;
            }
            const float chi2 = (float)c;
            const float th = P.obs[3 * (size_t)(e0 + e) + 2] < 0 ? 5.991f : 7.815f;
            const bool out = chi2 > th;
            P.outlier[e0 + e] = out ? 1 : 0;
            bad += out;
        }
        nBadEdges = (int)po_block_sum((double)bad, s_red);
        if (it == 2) robust = false;
        ++rounds;
        if (n < 10) break;                     // optimizer.edges().size() < 10
    }
    if (tid == 0) {
        for (int i = 0; i < 7; ++i) P.pose_out[7 * frame + i] = T[i];
        P.inliers[frame] = n - nBadEdges;
        P.stats[4 * frame] = rounds; P.stats[4 * frame + 1] = totalIters; P.stats[4 * frame + 2] = totalTrials; P.stats[4 * frame + 3] = 0;
    }
}


// ---- edge list of PoseOptimization from the searches' device-resident outputs ----------------------------------------
// The reference walks pFrame->mvpMapPoints in feature order (Optimizer.cc:104-290): one edge per feature that holds a map
// point.  feature_match (per compact keypoint row: query index or -1) is what orbm_search_last_frame / orbm_search_bow
// write; query_match (per query: feature index or -1) is what orbm_search_local_points writes and is scattered to the
// features first.  Two launches: counts per frame, then (offset = sum of the counts before) the ordered fill.
struct EdgeParams {
    const orbx_keypoint* kps;
    const float* uright;          // null => monocular
    const int* offsets;
    const int* nkp;
    int maxFeat;
    const int* frame_image;
    const int* feature_match;     // or null
    const int* qoff;              // with query_match
    const int* query_match;       // or null
    const float* xw;              // [nq][3]
    const float* xw2;             // with BOTH sources: world positions of the query_match entries (xw then belongs to feature_match)
    float invSigma2[ORB_MAX_LEVELS];
    int* cnt;                     // [n_frames]
    int* eoff;                    // [n_frames + 1]
    int* efeat;                   // [ne] feature index inside the frame
    float* exw;                   // [ne][3]
    float* eobs;                  // [ne][3]
    float* ew;                    // [ne]
};

#define PE_THREADS 256

template <bool FILL>
__global__ void __launch_bounds__(PE_THREADS) k_pose_edges(const __grid_constant__ EdgeParams P, int n_frames) {
    extern __shared__ int pe_holder[];   // maxFeat
    __shared__ int s_warp[PE_THREADS / 32 + 1];
    __shared__ int s_base, s_run;
    const int frame = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int img = P.frame_image[frame];
    const int N = min(P.nkp[img], P.maxFeat), row0 = P.offsets[img];
    for (int i = tid; i < N; i += PE_THREADS) pe_holder[i] = P.feature_match ? P.feature_match[row0 + i] : -1;
    __syncthreads();
    if (P.query_match) {
        const int q0 = P.qoff[frame], q1 = P.qoff[frame + 1];
        const int tag = P.xw2 ? 0x40000000 : 0;      // both sources: entries of the second one carry a tag (their positions come from xw2)
        for (int q = q0 + tid; q < q1; q += PE_THREADS) {
            const int f = P.query_match[q];
            if (f >= 0 && f < N) pe_holder[f] = q | tag;   // a feature is claimed by at most one query of a search
        }
        __syncthreads();
    }
    if (!FILL) {
        int c = 0;
        for (int i = tid; i < N; i += PE_THREADS) c += pe_holder[i] >= 0;
        c = __reduce_add_sync(0xffffffffu, c);
        if (lane == 0) s_warp[wid] = c;
        __syncthreads();
        if (tid == 0) {
            int t = 0;
            for (int w = 0; w < PE_THREADS / 32; ++w) t += s_warp[w];
            P.cnt[frame] = t;
        }
        return;
    }
    if (tid == 0) {
        int b = 0;
        for (int f = 0; f < frame; ++f) b += P.cnt[f];
        s_base = b;
        s_run = 0;
        P.eoff[frame] = b;
        if (frame == n_frames - 1) P.eoff[n_frames] = b + P.cnt[frame];
    }
    __syncthreads();
    for (int base = 0; base < N; base += PE_THREADS) {          // ordered compaction, PE_THREADS features at a time
        const int i = base + tid;
        const int q = i < N ? pe_holder[i] : -1;
        const unsigned m = __ballot_sync(0xffffffffu, q >= 0);
        if (lane == 0) s_warp[wid] = __popc(m);
        __syncthreads();
        int before = s_run;
        for (int w = 0; w < wid; ++w) before += s_warp[w];
        if (q >= 0) {
            const int e = s_base + before + __popc(m & ((1u << lane) - 1u));
            const orbx_keypoint k = P.kps[row0 + i];
            P.efeat[e] = i;
            const float* wp = (q & 0x40000000) ? P.xw2 + 3 * (size_t)(q & 0x3fffffff) : P.xw + 3 * (size_t)q;
            P.exw[3 * (size_t)e] = wp[0]; P.exw[3 * (size_t)e + 1] = wp[1]; P.exw[3 * (size_t)e + 2] = wp[2];
            P.eobs[3 * (size_t)e] = k.x; P.eobs[3 * (size_t)e + 1] = k.y; P.eobs[3 * (size_t)e + 2] = P.uright ? P.uright[row0 + i] : -1.0f;
            P.ew[e] = P.invSigma2[k.octave];
        }
        __syncthreads();
        if (tid == 0) {
            int t = 0;
            for (int w = 0; w < PE_THREADS / 32; ++w) t += s_warp[w];
            s_run += t;
        }
        __syncthreads();
    }
}

}  // namespace orb

extern "C" orb_status orbo_pose_optimization(orbx_handle* h, const orbo_pose_problems* in, double* pose_out, uint8_t* outlier_out,
                                             int32_t* inliers_out, int32_t* stats_out) {
    if (!h || !in || in->n_frames < 1 || !in->edge_offset || !in->pose || !pose_out || !inliers_out)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const bool dev = in->on_device != 0;
    const int nf = in->n_frames;
    // device callers give an upper bound of the edge count (it sizes the scratch): no read-back, no synchronisation
    const int ne = dev ? in->n_edges_max : in->edge_offset[nf];
    if (ne < 0 || (ne > 0 && (!in->world_pos || !in->obs || !in->inv_sigma2 || !outlier_out))) return set_error(ORB_ERR_INVALID, "missing edge arrays");
    // scratch (and, for host callers, staging) comes from the handle's matcher stage buffer
    PoseOptParams P{};
    P.fx = in->fx; P.fy = in->fy; P.cx = in->cx; P.cy = in->cy; P.bf = in->bf;   // float members promoted (Optimizer.cc:146-150)
    auto layout = [&](Carve& c) {
        P.err = c.take<double>(ne);
        P.eoff = stage_in(c, in->edge_offset, nf + 1, dev); P.pose = stage_in(c, in->pose, (size_t)nf * 7, dev);
        P.xw = stage_in(c, in->world_pos, (size_t)ne * 3, dev); P.obs = stage_in(c, in->obs, (size_t)ne * 3, dev);
        P.invs2 = stage_in(c, in->inv_sigma2, ne, dev);
        P.outlier = stage_out(c, outlier_out, ne, dev);
        P.pose_out = stage_out(c, pose_out, (size_t)nf * 7, dev);
        P.inliers = stage_out(c, inliers_out, nf, dev);
        P.stats = stage_out(c, stats_out, (size_t)nf * 4, dev);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    k_pose_opt<<<nf, PO_THREADS, 0, h->stream>>>(P);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return dev ? ORB_OK : copy_out(c);
}

extern "C" orb_status orbo_pose_edges(orbx_handle* h, const orbo_edge_source* src, int32_t* edge_offset_out, int32_t* edge_feature_out,
                                      float* world_pos_out, float* obs_out, float* inv_sigma2_out) {
    const bool both = src && src->feature_match && src->query_match;
    if (!h || !src || src->n_frames < 1 || !src->frame_image || !src->world_pos || (!src->feature_match && !src->query_match) ||
        (both && !src->query_world_pos) || (!both && src->query_world_pos) || (src->query_match && !src->query_offset) || !edge_offset_out || !edge_feature_out || !world_pos_out || !obs_out || !inv_sigma2_out)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    if (h->last_batch < 1) return set_error(ORB_ERR_INVALID, "no batch has been extracted");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const int nf = src->n_frames;
    EdgeParams P{};
    P.kps = h->d_kps; P.uright = h->stereo_valid ? h->d_uright : nullptr; P.offsets = h->d_offsets; P.nkp = h->d_nkp;
    P.maxFeat = h->geom.kpTotal;
    P.frame_image = src->frame_image; P.feature_match = src->feature_match; P.qoff = src->query_offset; P.query_match = src->query_match;
    P.xw = src->world_pos;
    P.xw2 = src->query_world_pos;
    for (int l = 0; l < ORB_MAX_LEVELS; ++l) P.invSigma2[l] = l < h->cfg.n_levels ? h->inv_sigma2[l] : 1.f;
    const orb_status s = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, [&](Carve& c) { P.cnt = c.take<int>(nf); }).status;
    if (s != ORB_OK) return s;
    P.eoff = edge_offset_out; P.efeat = edge_feature_out; P.exw = world_pos_out; P.eobs = obs_out; P.ew = inv_sigma2_out;
    // one int per row of the handle: past 12 276 rows (48 KB less the 48 B of static arrays) the launch needs more than the default
    // window.  It always fits the opt-in limit: a handle has extracted a batch (checked above), and extraction refuses any row capacity
    // whose k_order block ((rows + 64) x 4 B plus its static arrays, extractor.cu) does not fit, which is the larger of the two
    const size_t sm = (size_t)P.maxFeat * 4;
    ORB_CUDA(cudaFuncSetAttribute(k_pose_edges<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    ORB_CUDA(cudaFuncSetAttribute(k_pose_edges<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    k_pose_edges<false><<<nf, PE_THREADS, sm, h->stream>>>(P, nf);
    ORB_LAUNCHED();
    k_pose_edges<true><<<nf, PE_THREADS, sm, h->stream>>>(P, nf);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return ORB_OK;
}

extern "C" orb_status orbo_pose_optimization_frames(orbx_handle* h, const orbo_frame_matches* in, double* pose_out,
                                                    uint8_t* feature_outlier_out, int32_t* inliers_out) {
    if (!h || !in || in->n_frames < 1 || !in->frame_image || !in->pose || !in->world_pos || in->n_queries < 0 ||
        ((in->feature_match != nullptr) == (in->query_match != nullptr)) || (in->query_match && !in->query_offset) || !pose_out || !inliers_out)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    int total_rows = 0;
    orb_status s = batch_rows(h, &total_rows);
    if (s != ORB_OK) return s;
    const int nf = in->n_frames;
    size_t cap = 0;                               // edges <= features of the listed frames
    for (int f = 0; f < nf; ++f) {
        const int img = in->frame_image[f];
        if (img < 0 || img >= h->last_batch) return set_error(ORB_ERR_INVALID, "bad frame image");
        cap += (size_t)image_features(h, img);
    }
    cap = std::max<size_t>(cap, 1);
    const int nq = in->n_queries;
    const int nqm = in->query_match ? in->query_offset[nf] : 0;
    cudaStream_t st = h->stream;
    orbo_edge_source src{nf};
    int *d_eoff, *d_efeat, *d_inl; float *d_pose, *d_exw, *d_eobs, *d_ew; double* d_pout; uint8_t* d_out;
    std::vector<int> eoff(nf + 1), efeat(cap);    // the edge walk, read back only to scatter the outlier flags
    std::vector<uint8_t> outl(cap);
    const bool scatter = feature_outlier_out != nullptr;
    auto layout = [&](Carve& c) {
        src.frame_image = stage_in(c, in->frame_image, nf, false); d_pose = stage_in(c, in->pose, (size_t)nf * 7, false);
        src.world_pos = stage_in(c, in->world_pos, (size_t)nq * 3, false);
        src.feature_match = stage_in(c, in->feature_match, total_rows, false);
        if (in->query_match) { src.query_offset = stage_in(c, in->query_offset, nf + 1, false); src.query_match = stage_in(c, in->query_match, nqm, false); }
        d_eoff = stage_out(c, scatter ? eoff.data() : nullptr, nf + 1, false);
        d_efeat = stage_out(c, scatter ? efeat.data() : nullptr, cap, false);
        d_exw = c.take<float>(cap * 3); d_eobs = c.take<float>(cap * 3); d_ew = c.take<float>(cap);
        d_pout = stage_out(c, pose_out, (size_t)nf * 7, false);
        d_out = stage_out(c, scatter ? outl.data() : nullptr, cap, false);
        d_inl = stage_out(c, inliers_out, nf, false);
    };
    const Carve c = carve_scratch(h->po_bytes, h->d_po, h->capturing, st, layout);
    if (c.status != ORB_OK) return c.status;
    if ((s = orbo_pose_edges(h, &src, d_eoff, d_efeat, d_exw, d_eobs, d_ew)) != ORB_OK) return s;
    orbo_pose_problems pp{nf, 1, d_eoff, d_pose, d_exw, d_eobs, d_ew, in->fx, in->fy, in->cx, in->cy, in->bf, (int32_t)cap};
    if ((s = orbo_pose_optimization(h, &pp, d_pout, d_out, d_inl, nullptr)) != ORB_OK) return s;
    if ((s = copy_out(c)) != ORB_OK) return s;
    if (scatter) {                     // pFrame->mvbOutlier[i] of every feature of the listed frames
        for (int f = 0; f < nf; ++f) {
            const int img = in->frame_image[f], row0 = image_row0(h, img);
            std::fill(feature_outlier_out + row0, feature_outlier_out + row0 + image_features(h, img), (uint8_t)0);
            for (int e = eoff[f]; e < eoff[f + 1]; ++e) feature_outlier_out[row0 + efeat[e]] = outl[e];
        }
    }
    return ORB_OK;
}
