// lba.cu -- Optimizer::LocalBundleAdjustment's numeric core on the device
// (/root/reference/src/Optimizer.cc:1859-2150: g2o OptimizationAlgorithmLevenberg over BlockSolver_6_3,
// Huber kernels, 10 iterations; math spec: SURVEY.md Appendix C).
//
// One CTA per problem runs the WHOLE Levenberg-Marquardt loop on the device (no host round trips):
//   E  per-edge reprojection residuals + robust chi2            (sparse_optimizer.cpp:61-113)
//   B  point-parallel linearisation: every thread owns map points, walks their edges, keeps H_ll / b_l in
//      registers, writes H_pl per edge and the per-edge pose terms; pose blocks are then reduced per pose in
//      a fixed order (deterministic -- LM accept/reject decisions must not depend on atomics ordering)
//      (base_binary_edge.hpp:55-120, types_six_dof_expmap.cpp:228-275, OptimizableTypes.cpp:175-197)
//   S  Schur complement: D^-1 per landmark, then one warp per upper pose-block pair sums B_i D^-1 B_j^T over
//      the landmarks the two poses share (block_solver.hpp:367-439)
//   L  dense LDL^T of the reduced pose system in shared memory (linear_solver_eigen.h:94-122: SimplicialLDLT;
//      at <= 24 poses the sparse ordering is irrelevant)
//   X  back-substitution of the landmarks, exp-map pose update (se3quat.h:223-255), gain ratio, lambda schedule
//      (optimization_algorithm_levenberg.cpp:61-169).
// All arithmetic is fp64 (the stereo edge keeps g2o's float32 reciprocal depth).
#include <stdlib.h>

#include <algorithm>
#include <chrono>
#include <thread>
#include <vector>

#include <cooperative_groups.h>

#include "common.cuh"
#include "ba_math.cuh"
#include "lba_pack.h"
#include "scratch.h"

using namespace orb;

namespace orb {

#define LBA_THREADS 256
#define LBA_CS_MAX 16    // CTAs (SMs) per problem: 16 (the non-portable cluster size sm_90 allows) for one or two problems, 8 while they fit the SMs

__device__ __forceinline__ int edge_error(const LbaDev& P, int e, double r[3], double Xc[3]) {
    se3_map(P.pose + 7 * P.ekf[e], P.point + 3 * P.emp[e], Xc);
    const double* z = P.obs + 3 * e;
    if (z[2] < 0) {   // EdgeSE3ProjectXYZ::computeError + Pinhole::project(Vector3d)
        r[0] = z[0] - (P.fx * Xc[0] / Xc[2] + P.cx);
        r[1] = z[1] - (P.fy * Xc[1] / Xc[2] + P.cy);
        r[2] = 0;
        return 2;
    }
    const double invz = (double)__fdiv_rn(1.0f, (float)Xc[2]);   // const float invz = 1.0f/trans_xyz[2]
    const double u = Xc[0] * invz * P.fx + P.cx;
    r[0] = z[0] - u;
    r[1] = z[1] - (Xc[1] * invz * P.fy + P.cy);
    r[2] = z[2] - (u - P.bf * invz);
    return 3;
}

struct Huber {
    double dM, dS, sqM, sqS;
};

// ---- cluster-wide helpers.  One thread-block CLUSTER (LBA_CS CTAs on LBA_CS SMs) works on one problem; all
// cross-CTA traffic goes through global memory (L2) and is ordered by the hardware cluster barrier.
namespace cg = cooperative_groups;

struct Team {
    int rank, cs, tid, gtid, gstride, gwarp, nwarps;
    __device__ void sync() const {
        if (cs > 1) cg::this_cluster().sync(); else __syncthreads();
    }
};

// deterministic sum over the whole team: fixed tree inside the CTA, then the CTA partials in rank order
__device__ double team_sum(const Team& T, double v, double* red, double* partials /* global, LBA_CS_MAX */) {
    red[T.tid] = v;
    __syncthreads();
    for (int s = LBA_THREADS / 2; s > 0; s >>= 1) {
        if (T.tid < s) red[T.tid] += red[T.tid + s];
        __syncthreads();
    }
    if (T.cs == 1) {
        const double out = red[0];
        __syncthreads();
        return out;
    }
    if (T.tid == 0) partials[T.rank] = red[0];
    T.sync();
    double out = 0;
    for (int r = 0; r < T.cs; ++r) out += partials[r];
    T.sync();   // partials may be rewritten by the next reduction
    return out;
}

__device__ double team_max(const Team& T, double v, double* red, double* partials) {
    red[T.tid] = v;
    __syncthreads();
    for (int s = LBA_THREADS / 2; s > 0; s >>= 1) {
        if (T.tid < s) red[T.tid] = fmax(red[T.tid], red[T.tid + s]);
        __syncthreads();
    }
    if (T.tid == 0) partials[T.rank] = red[0];
    T.sync();
    double out = 0;
    for (int r = 0; r < T.cs; ++r) out = fmax(out, partials[r]);
    T.sync();
    return out;
}

__device__ double compute_errors(const LbaDev& P, const Huber& H, const Team& T, double* red) {
    double chi = 0;
    for (int e = T.gtid; e < P.nE; e += T.gstride) {
        double r[3], Xc[3];
        const int D = edge_error(P, e, r, Xc);
        const double c = P.invs2[e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
        P.err[e] = c;
        double w;
        chi += huber_rho(c, D == 2 ? H.dM : H.dS, D == 2 ? H.sqM : H.sqS, &w);
    }
    return team_sum(T, chi, red, P.partials);
}

// B phase, part 1: an 8-lane group per map point, lane = edge: every lane linearises one edge, writes its H_pl block and
// pose terms; a landmark with more than 8 observations loops over them 8 at a time, each lane accumulating its own edges in
// order.  The H_ll / b_l contributions are then summed across the group with a fixed shuffle tree (deterministic).
__device__ void build_points(const LbaDev& P, const Huber& H, int gtid, int gstride) {
    const int sub = gtid & 7, ngroups = gstride >> 3;
    const int warpFirstGroup = (gtid & ~31) >> 3;
    for (int l0 = warpFirstGroup; l0 < P.nMP; l0 += ngroups) {   // warp-uniform trip count
        const int l = l0 + ((gtid & 31) >> 3);
        const bool active = l < P.nMP;
        const int k0 = active ? P.mpStart[l] : 0, ne = active ? P.mpStart[l + 1] - k0 : 0;
        double hl[6] = {0, 0, 0, 0, 0, 0};
        double b0 = 0, b1 = 0, b2 = 0;
        for (int base = 0; __any_sync(0xffffffffu, base < ne); base += 8) {
            const int k = k0 + base + sub;
            if (base + sub < ne) {
    const int e = P.mpEdge[k];
                double r[3], Xc[3];
                const int D = edge_error(P, e, r, Xc);
                const double xx = Xc[0], yy = Xc[1], zz = Xc[2], iz = 1.0 / zz, iz2 = iz * iz;
                double R[9];
                quat_to_R(P.pose + 7 * P.ekf[e], R);
                double A[9], B[18];
                if (D == 3) {   // EdgeStereoSE3ProjectXYZ::linearizeOplus
                    for (int c = 0; c < 3; ++c) {
                        A[c] = -P.fx * R[c] * iz + P.fx * xx * R[6 + c] * iz2;
                        A[3 + c] = -P.fy * R[3 + c] * iz + P.fy * yy * R[6 + c] * iz2;
                        A[6 + c] = A[c] - P.bf * R[6 + c] * iz2;
                    }
                    B[0] = xx * yy * iz2 * P.fx; B[1] = -(1 + (xx * xx * iz2)) * P.fx; B[2] = yy * iz * P.fx;
                    B[3] = -iz * P.fx; B[4] = 0; B[5] = xx * iz2 * P.fx;
                    B[6] = (1 + yy * yy * iz2) * P.fy; B[7] = -xx * yy * iz2 * P.fy; B[8] = -xx * iz * P.fy;
                    B[9] = 0; B[10] = -iz * P.fy; B[11] = yy * iz2 * P.fy;
                    B[12] = B[0] - P.bf * yy * iz2; B[13] = B[1] + P.bf * xx * iz2; B[14] = B[2];
                    B[15] = B[3]; B[16] = 0; B[17] = B[5] - P.bf * iz2;
                } else {        // ORB_SLAM3::EdgeSE3ProjectXYZ::linearizeOplus with Pinhole::projectJac
                    const double j0 = -(P.fx * iz), j2 = P.fx * xx * iz2, j4 = -(P.fy * iz), j5 = P.fy * yy * iz2;
                    for (int c = 0; c < 3; ++c) {
                        A[c] = j0 * R[c] + j2 * R[6 + c];
                        A[3 + c] = j4 * R[3 + c] + j5 * R[6 + c];
                        A[6 + c] = 0;
                    }
                    B[0] = j2 * yy;  B[1] = j0 * zz - j2 * xx; B[2] = -j0 * yy; B[3] = j0; B[4] = 0;  B[5] = j2;
                    B[6] = -j4 * zz + j5 * yy; B[7] = -j5 * xx; B[8] = j4 * xx; B[9] = 0;  B[10] = j4; B[11] = j5;
                    for (int c = 12; c < 18; ++c) B[c] = 0;
                }
                const double c2 = P.invs2[e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
                double w;
                huber_rho(c2, D == 2 ? H.dM : H.dS, D == 2 ? H.sqM : H.sqS, &w);
                const double om = w * P.invs2[e];
                // H_ll += A^T om A ; b_l += -A^T om r
                hl[0] += om * (A[0] * A[0] + A[3] * A[3] + A[6] * A[6]);
                hl[1] += om * (A[0] * A[1] + A[3] * A[4] + A[6] * A[7]);
                hl[2] += om * (A[0] * A[2] + A[3] * A[5] + A[6] * A[8]);
                hl[3] += om * (A[1] * A[1] + A[4] * A[4] + A[7] * A[7]);
                hl[4] += om * (A[1] * A[2] + A[4] * A[5] + A[7] * A[8]);
                hl[5] += om * (A[2] * A[2] + A[5] * A[5] + A[8] * A[8]);
                b0 += -om * (A[0] * r[0] + A[3] * r[1] + A[6] * r[2]);
                b1 += -om * (A[1] * r[0] + A[4] * r[1] + A[7] * r[2]);
                b2 += -om * (A[2] * r[0] + A[5] * r[1] + A[8] * r[2]);
                if (P.pidx[P.ekf[e]] >= 0) {
                    double* hx = P.Hpl + 18 * (size_t)e;
                    double* wv = P.W + 27 * (size_t)P.poseSlot[e];
                    int u = 0;
                    for (int i = 0; i < 6; ++i) {
                        for (int j = 0; j < 3; ++j) hx[3 * i + j] = om * (B[i] * A[j] + B[6 + i] * A[3 + j] + B[12 + i] * A[6 + j]);
                        for (int j = i; j < 6; ++j) wv[u++] = om * (B[i] * B[j] + B[6 + i] * B[6 + j] + B[12 + i] * B[12 + j]);
                        wv[21 + i] = -om * (B[i] * r[0] + B[6 + i] * r[1] + B[12 + i] * r[2]);
                    }
                }
            }
        }
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) {
#pragma unroll
            for (int q = 0; q < 6; ++q) hl[q] += __shfl_xor_sync(0xffffffffu, hl[q], o);
            b0 += __shfl_xor_sync(0xffffffffu, b0, o);
            b1 += __shfl_xor_sync(0xffffffffu, b1, o);
            b2 += __shfl_xor_sync(0xffffffffu, b2, o);
        }
        if (active && sub == 0) {
            double* o = P.Hll + 9 * (size_t)l;
            o[0] = hl[0]; o[1] = hl[1]; o[2] = hl[2]; o[3] = hl[1]; o[4] = hl[3]; o[5] = hl[4]; o[6] = hl[2]; o[7] = hl[4]; o[8] = hl[5];
            P.bl[3 * l] = b0; P.bl[3 * l + 1] = b1; P.bl[3 * l + 2] = b2;
        }
    }
}

// B phase, part 2: H_pp / b_p = per-pose sums of the per-edge terms.  The terms are stored in pose-sorted order,
// so a warp streams a contiguous [slots][27] slab (lane = term).  Each pose is cut into LBA_PCH chunks handled by
// different warps of the team; partial sums are combined in a fixed order (deterministic).
__device__ void build_poses(const LbaDev& P, const Team& T) {
    const int lane = T.tid & 31;
    for (int task = T.gwarp; task < P.nP * LBA_PCH; task += T.nwarps) {
        const int p = task / LBA_PCH, c = task - p * LBA_PCH;
        const int s0 = P.poseStart[p], s1 = P.poseStart[p + 1];
        const int len = (s1 - s0 + LBA_PCH - 1) / LBA_PCH;
        const int b = s0 + c * len, e = min(b + len, s1);
        double s = 0;
        if (lane < 27)
            for (int k = b; k < e; ++k) s += P.W[27 * (size_t)k + lane];
        if (lane < 27) P.posePart[(size_t)task * 27 + lane] = s;
    }
    T.sync();
    for (int i = T.gtid; i < P.nP * 27; i += T.gstride) {
        const int p = i / 27, c = i - p * 27;
        double s = 0;
        for (int k = 0; k < LBA_PCH; ++k) s += P.posePart[(size_t)(p * LBA_PCH + k) * 27 + c];
        if (c < 21) {
            int r = 0, rem = c;
            while (rem >= 6 - r) { rem -= 6 - r; ++r; }
            const int j = r + rem;
            P.Hpp[36 * (size_t)p + 6 * r + j] = s;
            P.Hpp[36 * (size_t)p + 6 * j + r] = s;
        } else {
            P.bp[6 * p + (c - 21)] = s;
        }
    }
}

// dense LDL^T of the upper-stored n x n matrix Hs (row-major), in place, by ONE CTA: after the call row j holds
// D_j on the diagonal and L(i,j) at (j,i), i > j.  Warps own rows of the trailing block, lanes walk a row
// (conflict-free, no integer division).  Returns false on a zero / non-finite pivot.
__device__ bool ldlt_factor(double* Hs, int n, double* col /* >= n doubles, shared */, int* s_ok) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = LBA_THREADS / 32;
    if (tid == 0) *s_ok = 1;
    __syncthreads();
    for (int j = 0; j < n; ++j) {
        const double dj = Hs[(size_t)j * n + j];
        if (!(fabs(dj) > 0) || !isfinite(dj)) {
            if (tid == 0) *s_ok = 0;
            break;   // uniform: every thread reads the same dj
        }
        const int m = n - j - 1;
        const double inv = 1.0 / dj;
        for (int i = tid; i < m; i += LBA_THREADS) col[i] = Hs[(size_t)j * n + j + 1 + i] * inv;   // L(j+1+i, j)
        __syncthreads();
        for (int a = warp; a < m; a += nw) {
            const double la = col[a] * dj;
            double* row = Hs + (size_t)(j + 1 + a) * n + (j + 1);
            for (int b = a + lane; b < m; b += 32) row[b] -= la * col[b];
        }
        for (int i = tid; i < m; i += LBA_THREADS) Hs[(size_t)j * n + j + 1 + i] = col[i];
        __syncthreads();
    }
    __syncthreads();
    return *s_ok != 0;
}

// Blocked variant for systems that live in shared memory (n <= LBA_SMEM_N, n a multiple of 6): 6x6 pose blocks are
// the pivots, so a factorisation costs 3 barriers per pose instead of 2 per scalar column.  Produces the same
// storage as ldlt_factor (D on the diagonal, L(i,j) at (j,i)).  W = 6 x n panel (D L^T rows), Lp = n x 6 panel.
__device__ bool ldlt_factor_blocked(double* Hs, int n, double* Wp, double* Lp, int* s_ok) {
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = LBA_THREADS / 32;
    if (tid == 0) *s_ok = 1;
    __syncthreads();
    for (int j0 = 0; j0 < n; j0 += 6) {
        // 1. scalar LDL^T of the 6x6 diagonal block by warp 0 (6 mini steps)
        if (warp == 0) {
            for (int c = 0; c < 6; ++c) {
                const double dj = Hs[(size_t)(j0 + c) * n + j0 + c];
                if (!(fabs(dj) > 0) || !isfinite(dj)) {
                    if (lane == 0) *s_ok = 0;
                    break;
                }
                // trailing update inside the block: rows a > c, cols b >= a
                if (lane < 21) {   // the 21 upper-triangular elements (a <= b) of the 6x6 block, one per lane
                    int a = 0, rem = lane;
                    while (rem >= 6 - a) { rem -= 6 - a; ++a; }
                    const int b = a + rem;
                    if (a > c) {
                        const double la = Hs[(size_t)(j0 + c) * n + j0 + a] / dj, lb = Hs[(size_t)(j0 + c) * n + j0 + b];
                        Hs[(size_t)(j0 + a) * n + j0 + b] -= la * lb;
                    }
                }
                __syncwarp();
                if (lane > c && lane < 6) Hs[(size_t)(j0 + c) * n + j0 + lane] /= dj;   // L(lane, c) stored at (c, lane)
                if (lane == 0) Lp[6 * LBA_SMEM_N + c] = 1.0 / dj;
                __syncwarp();
            }
        }
        __syncthreads();
        if (*s_ok == 0) break;
        const int m = n - j0 - 6;
        if (m <= 0) break;
        // 2. panel: W = L_JJ^-1 A(J, right) (6 x m), Lp(i, c) = W(c, i) / D_c
        for (int i = tid; i < m; i += LBA_THREADS) {
            double w[6];
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                double v = Hs[(size_t)(j0 + c) * n + j0 + 6 + i];
#pragma unroll
                for (int c2 = 0; c2 < 6; ++c2)
                    if (c2 < c) v -= Hs[(size_t)(j0 + c2) * n + j0 + c] * w[c2];   // L_JJ(c, c2) stored at (c2, c)
                w[c] = v;
            }
#pragma unroll
            for (int c = 0; c < 6; ++c) {
                Wp[c * LBA_SMEM_N + i] = w[c];
                Lp[i * 6 + c] = w[c] * Lp[6 * LBA_SMEM_N + c];   // 1 / D_c, published by warp 0
            }
        }
        __syncthreads();
        // 3. trailing update A(i, k) -= sum_c Lp(i, c) W(c, k), k >= i; four rows per warp pass share the W loads
        for (int a0 = 4 * warp; a0 < m; a0 += 4 * nw) {
            double l[4][6];
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 6; ++c) l[r][c] = (a0 + r < m) ? Lp[(a0 + r) * 6 + c] : 0.0;
            for (int b = a0 + lane; b < m; b += 32) {
                double w[6];
#pragma unroll
                for (int c = 0; c < 6; ++c) w[c] = Wp[c * LBA_SMEM_N + b];
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (a0 + r < m && b >= a0 + r) {
                        double* e = Hs + (size_t)(j0 + 6 + a0 + r) * n + (j0 + 6) + b;
                        *e -= l[r][0] * w[0] + l[r][1] * w[1] + l[r][2] * w[2] + l[r][3] * w[3] + l[r][4] * w[4] + l[r][5] * w[5];
                    }
                }
            }
        }
        for (int i = tid; i < m * 6; i += LBA_THREADS) {
            const int c = i / m, k = i - c * m;
            Hs[(size_t)(j0 + c) * n + j0 + 6 + k] = Lp[k * 6 + c];
        }
        __syncthreads();
    }
    __syncthreads();
    return *s_ok != 0;
}

// x = (L D L^T)^-1 b by warp 0; y lives in shared memory, lanes update the rows below / above the pivot
__device__ void ldlt_solve_warp(const double* Hs, int n, const double* b, double* x, double* y /* shared, n */) {
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < n; i += 32) y[i] = b[i];
    __syncwarp();
    for (int i = 0; i < n; ++i) {   // forward: y_k -= L(k,i) y_i for k > i   (L(k,i) stored at (i,k): contiguous)
        const double yi = y[i];
        for (int k = i + 1 + lane; k < n; k += 32) y[k] -= Hs[(size_t)i * n + k] * yi;
        __syncwarp();
    }
    for (int i = lane; i < n; i += 32) y[i] /= Hs[(size_t)i * n + i];
    __syncwarp();
    for (int i = n - 1; i >= 0; --i) {   // backward: x_i = y_i - sum_{k>i} L(k,i) x_k  (row i of the stored U)
        double sdot = 0;
        for (int k = i + 1 + lane; k < n; k += 32) sdot += Hs[(size_t)i * n + k] * y[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sdot += __shfl_xor_sync(0xffffffffu, sdot, o);
        if (lane == 0) y[i] -= sdot;
        __syncwarp();
    }
    for (int i = lane; i < n; i += 32) x[i] = y[i];
}

// The same solve, blocked by pose (n = 6 nP): per 6-row block, six in-block substitution steps over shuffles and ONE lane-parallel
// update of all remaining rows with the block's six values (forward), or six lane-parallel dot products with everything already
// solved (backward) -- 2 x nP dependent steps instead of 2 x n (tools/lba_phases.py clocks both forms; the scalar one
// is the longer dependent chain at 18 free poses).
__device__ void ldlt_solve_warp_blocked(const double* Hs, int n, const double* b, double* x, double* y /* shared, n */) {
    const int lane = threadIdx.x & 31;
    for (int i = lane; i < n; i += 32) y[i] = b[i];
    __syncwarp();
    for (int j0 = 0; j0 < n; j0 += 6) {   // forward: L y' = b
        double yl = lane < 6 ? y[j0 + lane] : 0.0;
#pragma unroll
        for (int c = 0; c < 5; ++c) {
            const double yc = __shfl_sync(0xffffffffu, yl, c);
            if (lane > c && lane < 6) yl -= Hs[(size_t)(j0 + c) * n + j0 + lane] * yc;   // L(j0 + lane, j0 + c) stored at (j0 + c, j0 + lane)
        }
        if (lane < 6) y[j0 + lane] = yl;
        double yb[6];
#pragma unroll
        for (int c = 0; c < 6; ++c) yb[c] = __shfl_sync(0xffffffffu, yl, c);
        for (int k = j0 + 6 + lane; k < n; k += 32) {
            double v = y[k];
#pragma unroll
            for (int c = 0; c < 6; ++c) v -= Hs[(size_t)(j0 + c) * n + k] * yb[c];
            y[k] = v;
        }
        __syncwarp();
    }
    for (int i = lane; i < n; i += 32) y[i] /= Hs[(size_t)i * n + i];
    __syncwarp();
    for (int j0 = n - 6; j0 >= 0; j0 -= 6) {   // backward: L^T x = y''
        double s[6] = {0, 0, 0, 0, 0, 0};
        for (int k = j0 + 6 + lane; k < n; k += 32) {
            const double xk = y[k];
#pragma unroll
            for (int c = 0; c < 6; ++c) s[c] += Hs[(size_t)(j0 + c) * n + k] * xk;
        }
#pragma unroll
        for (int c = 0; c < 6; ++c)
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
        double xl = 0.0;
        if (lane < 6) {
            double sc = s[0];
#pragma unroll
            for (int c = 1; c < 6; ++c) sc = (lane == c) ? s[c] : sc;
            xl = y[j0 + lane] - sc;
        }
#pragma unroll
        for (int c = 5; c > 0; --c) {      // x_c final; rows above it inside the block subtract L(j0 + c, j0 + r) x_c, stored at (j0 + r, j0 + c)
            const double xc = __shfl_sync(0xffffffffu, xl, c);
            if (lane < c) xl -= Hs[(size_t)(j0 + lane) * n + j0 + c] * xc;
        }
        if (lane < 6) y[j0 + lane] = xl;
        __syncwarp();
    }
    for (int i = lane; i < n; i += 32) x[i] = y[i];
}

__global__ void __launch_bounds__(LBA_THREADS, 1) k_lba(const LbaDev* __restrict__ problems, int cs) {
    extern __shared__ __align__(16) unsigned char lba_smem[];
    __shared__ LbaDev Ps;
    __shared__ int s_ok;
    Team T;
    T.cs = cs;
    T.rank = blockIdx.x % cs;
    T.tid = threadIdx.x;
    T.gtid = T.rank * LBA_THREADS + T.tid;
    T.gstride = cs * LBA_THREADS;
    T.gwarp = T.gtid >> 5;
    T.nwarps = T.gstride >> 5;
    if (threadIdx.x == 0) Ps = problems[blockIdx.x / cs];
    __syncthreads();
    const LbaDev& P = Ps;
    double* red = reinterpret_cast<double*>(lba_smem);   // LBA_THREADS doubles (reductions) / >= n doubles (LDLT column)
    double* colbuf = red + LBA_THREADS;                  // 960 (column / rhs) + 6 x 144 + 144 x 6 + 8 (block panels, 1/D)
    double* Hs = (P.n <= LBA_SMEM_N) ? (colbuf + 960 + 12 * LBA_SMEM_N + 8) : P.HsGlobal;   // only rank 0 touches it
    const int tid = T.tid, n = P.n;
    Huber H;
    H.dM = (double)(float)sqrt(5.991);     // Optimizer.cc:1957-1958: const float thHuberMono / thHuberStereo
    H.dS = (double)(float)sqrt(7.815);
    H.sqM = (double)(float)(H.dM * H.dM);  // RobustKernelHuber::dsqr is a float member
    H.sqS = (double)(float)(H.dS * H.dS);
    long long tph[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    long long tlast = clock64();
#define LBA_TICK(k) { const long long _t = clock64(); tph[k] += _t - tlast; tlast = _t; }

    for (int i = T.gtid; i < 7 * P.nKF; i += T.gstride) P.pose[i] = P.pose0[i];
    for (int i = T.gtid; i < 3 * P.nMP; i += T.gstride) P.point[i] = P.point0[i];
    T.sync();

    double lambda = -1, ni = 2, currentChi = 0, iniChi0 = 0;
    int nBad = 0, iters = 0, trials = 0, fslot = 0;   // the stop flag is published through two alternating slots so
    bool ok = true;                                    // that a slow CTA never reads a slot that is being rewritten
    for (int it = 0; it < P.maxIters && ok; ++it) {
        fslot ^= 2;
        if (T.gtid == 0) P.flags[fslot] = (P.stop && *P.stop) ? 1 : 0;   // one reader: the decision must be uniform
        T.sync();
        if (P.flags[fslot]) break;
        LBA_TICK(11)
        currentChi = compute_errors(P, H, T, red);
        LBA_TICK(0)
        if (it == 0) iniChi0 = currentChi;
        const double iniChi = currentChi;
        double tempChi = currentChi;
        build_points(P, H, T.gtid, T.gstride);
        T.sync();
        LBA_TICK(1)
        build_poses(P, T);
        T.sync();
        LBA_TICK(2)
        if (it == 0) {
            if (P.lambdaInit > 0) lambda = P.lambdaInit;
            else {   // computeLambdaInit: tau * max |H_jj|
                double md = 0;
                for (int i = T.gtid; i < 6 * P.nP; i += T.gstride) md = fmax(md, fabs(P.Hpp[36 * (size_t)(i / 6) + 7 * (i % 6)]));
                for (int i = T.gtid; i < 3 * P.nMP; i += T.gstride) md = fmax(md, fabs(P.Hll[9 * (size_t)(i / 3) + 4 * (i % 3)]));
                lambda = 1e-5 * team_max(T, md, red, P.partials);
            }
            ni = 2;
            nBad = 0;
        }
        double rho = 0;
        int qmax = 0;
        bool stopped = false;
        do {
            // push
            for (int i = T.gtid; i < 7 * P.nKF; i += T.gstride) P.poseSave[i] = P.pose[i];
            for (int i = T.gtid; i < 3 * P.nMP; i += T.gstride) P.pointSave[i] = P.point[i];
            // ---- S: Schur complement -------------------------------------------------------------
            // the thread that owns landmark l inverts D_l and writes B_e1 D_l^-1 B_e2^T for every pair of its edges
            // with free poses p(e1) <= p(e2) into that pair's slot of its pose-block (no atomics)
            for (int l = T.gtid; l < P.nMP; l += T.gstride) {
                const double* M = P.Hll + 9 * (size_t)l;
                const double a = M[0] + lambda, b = M[1], c = M[2], d = M[3], e = M[4] + lambda, f = M[5], g = M[6], h = M[7], i = M[8] + lambda;
                const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
                const double id = 1.0 / det;
                const double d0 = (e * i - f * h) * id, d1 = (c * h - b * i) * id, d2 = (b * f - c * e) * id;
                const double d3 = (f * g - d * i) * id, d4 = (a * i - c * g) * id, d5 = (c * d - a * f) * id;
                const double d6 = (d * h - e * g) * id, d7 = (b * g - a * h) * id, d8 = (a * e - b * d) * id;
                double* Di = P.Dinv + 9 * (size_t)l;
                Di[0] = d0; Di[1] = d1; Di[2] = d2; Di[3] = d3; Di[4] = d4; Di[5] = d5; Di[6] = d6; Di[7] = d7; Di[8] = d8;
                const double* bl = P.bl + 3 * l;
                P.db[3 * l] = d0 * bl[0] + d1 * bl[1] + d2 * bl[2];
                P.db[3 * l + 1] = d3 * bl[0] + d4 * bl[1] + d5 * bl[2];
                P.db[3 * l + 2] = d6 * bl[0] + d7 * bl[1] + d8 * bl[2];
            }
            T.sync();
            for (int k = T.gtid; k < P.nFreeEdges; k += T.gstride) {   // BD_e = B_e D_l^-1, one thread per edge of a free pose
                const int e2 = P.poseEdge[k];
                const double* __restrict__ Di = P.Dinv + 9 * (size_t)P.emp[e2];
                const double d0 = Di[0], d1 = Di[1], d2 = Di[2], d3 = Di[3], d4 = Di[4], d5 = Di[5], d6 = Di[6], d7 = Di[7], d8 = Di[8];
                const double* __restrict__ Bm = P.Hpl + 18 * (size_t)e2;
                double* __restrict__ o = P.BD + 18 * (size_t)e2;
#pragma unroll
                for (int r = 0; r < 6; ++r) {
                    const double a0 = Bm[3 * r], a1 = Bm[3 * r + 1], a2 = Bm[3 * r + 2];
                    o[3 * r] = a0 * d0 + a1 * d3 + a2 * d6;
                    o[3 * r + 1] = a0 * d1 + a1 * d4 + a2 * d7;
                    o[3 * r + 2] = a0 * d2 + a1 * d5 + a2 * d8;
                }
            }
            T.sync();
            LBA_TICK(3)
            {
                const int lane = tid & 31;
                // Schur sums: one warp per pose-block pair; every lane owns a slice of the pair's co-observation items
                // and keeps a private 6x6 accumulator (no atomics, no intermediate array); lanes are combined with a
                // fixed shuffle tree => one deterministic summation order.
                for (int task = T.gwarp; task < P.nTasks; task += T.nwarps) {
                    const int kb = P.taskStart[task], ke = P.taskStart[task + 1];
                    double acc[36];
#pragma unroll
                    for (int q = 0; q < 36; ++q) acc[q] = 0.0;
                    int4 nxt = (kb + lane < ke) ? P.ptItem[kb + lane] : make_int4(0, 0, 0, 0);
                    for (int k = kb + lane; k < ke; k += 32) {
                        const int4 it4 = nxt;
                        if (k + 32 < ke) nxt = P.ptItem[k + 32];   // software prefetch: one L2 round trip per round
                        const double2* __restrict__ B1 = reinterpret_cast<const double2*>(P.BD + 18 * (size_t)it4.x);   // B_e1 D^-1
                        const double2* __restrict__ B2 = reinterpret_cast<const double2*>(P.Hpl + 18 * (size_t)it4.y);
                        double b1[18], b2[18];
#pragma unroll
                        for (int q = 0; q < 9; ++q) {
                            const double2 u = B1[q], v = B2[q];
                            b1[2 * q] = u.x; b1[2 * q + 1] = u.y; b2[2 * q] = v.x; b2[2 * q + 1] = v.y;
                        }
#pragma unroll
                        for (int r = 0; r < 6; ++r)
#pragma unroll
                            for (int j = 0; j < 6; ++j)
                                acc[6 * r + j] += b1[3 * r] * b2[3 * j] + b1[3 * r + 1] * b2[3 * j + 1] + b1[3 * r + 2] * b2[3 * j + 2];
                    }
#pragma unroll
                    for (int q = 0; q < 36; ++q) {
                        double v = acc[q];
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                        acc[q] = v;
                    }
                    if (lane == 0) {
#pragma unroll
                        for (int q = 0; q < 36; ++q) P.taskSum[36 * (size_t)task + q] = acc[q];
                    }
                }
                for (int p = T.gwarp; p < P.nP; p += T.nwarps) {   // b_schur = b_p - sum_e B_e (D^-1 b_l)
                    double s[6] = {0, 0, 0, 0, 0, 0};
                    for (int k = P.poseStart[p] + lane; k < P.poseStart[p + 1]; k += 32) {
                        const int e = P.poseEdge[k];
                        const double* Bm = P.Hpl + 18 * (size_t)e;
                        const double* d = P.db + 3 * P.emp[e];
                        for (int i = 0; i < 6; ++i) s[i] += Bm[3 * i] * d[0] + Bm[3 * i + 1] * d[1] + Bm[3 * i + 2] * d[2];
                    }
                    for (int i = 0; i < 6; ++i)
                        for (int o = 16; o > 0; o >>= 1) s[i] += __shfl_xor_sync(0xffffffffu, s[i], o);
                    if (lane == 0)
                        for (int i = 0; i < 6; ++i) P.bs[6 * p + i] = P.bp[6 * p + i] - s[i];
                }
            }
            T.sync();
            LBA_TICK(5)
            // ---- L: the reduced system is assembled, factorised and solved by rank 0 -----------------
            if (T.rank == 0) {
                for (int i = tid; i < n * n; i += LBA_THREADS) Hs[i] = 0.0;
                __syncthreads();
                for (int i = tid; i < P.nPairBlocks * 36; i += LBA_THREADS) {
                    const int blk = i / 36, e = i - blk * 36, r = e / 6, c = e - r * 6;
                    const int p1 = P.blockP1[blk], p2 = P.blockP2[blk];
                    double sum = 0;
                    for (int t = P.blockTask[blk]; t < P.blockTask[blk + 1]; ++t) sum += P.taskSum[36 * (size_t)t + e];
                    const double base = (p1 == p2) ? P.Hpp[36 * (size_t)p1 + e] + (r == c ? lambda : 0.0) : 0.0;
                    Hs[(size_t)(6 * p1 + r) * n + 6 * p2 + c] = base - sum;
                }
                __syncthreads();
                const bool okf = (n <= LBA_SMEM_N) ? ldlt_factor_blocked(Hs, n, colbuf + 960, colbuf + 960 + 6 * LBA_SMEM_N, &s_ok)
                                                   : ldlt_factor(Hs, n, colbuf, &s_ok);
                LBA_TICK(6)
                if (tid < 32) {
                    if (okf) ldlt_solve_warp_blocked(Hs, n, P.bs, P.xp, colbuf);
                    else for (int i = tid; i < n; i += 32) P.xp[i] = 0.0;
                }
                if (tid == 0) P.flags[1] = okf ? 1 : 0;
            }
            T.sync();
            LBA_TICK(7)
            const bool ok2 = P.flags[1] != 0;
            // ---- X: landmarks x_l = D^-1 (b_l - B^T x_p) -------------------------------------------
            for (int l = T.gtid; l < P.nMP; l += T.gstride) {
                double c0 = P.bl[3 * l], c1 = P.bl[3 * l + 1], c2 = P.bl[3 * l + 2];
                for (int k = P.mpStart[l]; k < P.mpStart[l + 1]; ++k) {
                    const int e = P.mpEdge[k];
                    const int p = P.pidx[P.ekf[e]];
                    if (p < 0) continue;
                    const double* Bm = P.Hpl + 18 * (size_t)e;
                    const double* x = P.xp + 6 * p;
                    for (int i = 0; i < 6; ++i) {
                        c0 -= Bm[3 * i] * x[i];
                        c1 -= Bm[3 * i + 1] * x[i];
                        c2 -= Bm[3 * i + 2] * x[i];
                    }
                }
                const double* Di = P.Dinv + 9 * (size_t)l;
                double x0 = Di[0] * c0 + Di[1] * c1 + Di[2] * c2, x1 = Di[3] * c0 + Di[4] * c1 + Di[5] * c2, x2 = Di[6] * c0 + Di[7] * c1 + Di[8] * c2;
                if (!ok2) { x0 = x1 = x2 = 0.0; }
                P.xl[3 * l] = x0; P.xl[3 * l + 1] = x1; P.xl[3 * l + 2] = x2;
                // SparseOptimizer::update for the landmark
                P.point[3 * l] += x0; P.point[3 * l + 1] += x1; P.point[3 * l + 2] += x2;
            }
            for (int k = T.gtid; k < P.nKF; k += T.gstride)
                if (P.pidx[k] >= 0) pose_oplus(P.pose + 7 * k, P.xp + 6 * P.pidx[k]);
            T.sync();
            LBA_TICK(8)
            tempChi = compute_errors(P, H, T, red);
            LBA_TICK(9)
            if (!ok2) tempChi = 1.7976931348623157e308;
            // computeScale: sum_j x_j (lambda x_j + b_j)
            double sc = 0;
            for (int i = T.gtid; i < n; i += T.gstride) sc += P.xp[i] * (lambda * P.xp[i] + P.bp[i]);
            for (int i = T.gtid; i < 3 * P.nMP; i += T.gstride) sc += P.xl[i] * (lambda * P.xl[i] + P.bl[i]);
            const double scale = team_sum(T, sc, red, P.partials) + 1e-3;
            rho = (currentChi - tempChi) / scale;
            if (rho > 0 && isfinite(tempChi)) {
                double alpha = 1. - pow((2 * rho - 1), 3);
                alpha = fmin(alpha, 2. / 3.);
                lambda *= fmax(1. / 3., alpha);
                ni = 2;
                currentChi = tempChi;
            } else {
                lambda *= ni;
                ni *= 2;
                for (int i = T.gtid; i < 7 * P.nKF; i += T.gstride) P.pose[i] = P.poseSave[i];   // pop
                for (int i = T.gtid; i < 3 * P.nMP; i += T.gstride) P.point[i] = P.pointSave[i];
            }
            fslot ^= 2;
            if (T.gtid == 0) P.flags[fslot] = (P.stop && *P.stop) ? 1 : 0;
            T.sync();
            ++qmax;
            ++trials;
            stopped = P.flags[fslot] != 0;
            LBA_TICK(10)
        } while (rho < 0 && qmax < 10 && !stopped);
        ++iters;
        if (qmax == 10 || rho == 0) { ok = false; break; }
        if ((iniChi - currentChi) * 1e3 < iniChi) ++nBad; else nBad = 0;
        if (nBad >= 3) { ok = false; break; }
    }
    T.sync();
    for (int e = T.gtid; e < P.nE; e += T.gstride) {
        double Xc[3];
        se3_map(P.pose + 7 * P.ekf[e], P.point + 3 * P.emp[e], Xc);
        P.depthPos[e] = Xc[2] > 0.0 ? 1 : 0;
    }
    if (T.gtid == 0) {
        P.stats[0] = iters; P.stats[1] = lambda; P.stats[2] = currentChi; P.stats[3] = trials; P.stats[4] = iniChi0;
        for (int k = 0; k < 12; ++k) P.stats[8 + k] = (double)tph[k];
    }
}

}  // namespace orb

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
struct lba_handle : SolverHandle {
    int* h_stop = nullptr;         // mapped pinned flag the kernel polls
    int* d_stop = nullptr;
};

// k_lba's dynamic shared memory with a reduced system of n x n in it
static size_t lba_smem_bytes(int n) { return (LBA_THREADS + 960 + 12 * LBA_SMEM_N + 8 + (size_t)n * n) * sizeof(double); }

extern "C" void lba_destroy(lba_handle* h) {
    if (!h) return;
    solver_release(h);
    if (h->h_stop) cudaFreeHost(h->h_stop);
    delete h;
}

extern "C" orb_status lba_create(int32_t device, lba_handle** out) {
    const orb_status s = solver_create(device, k_lba, lba_smem_bytes(LBA_SMEM_N), out);
    if (s != ORB_OK) return s;
    lba_handle* h = *out;
    if (cudaHostAlloc((void**)&h->h_stop, sizeof(int), cudaHostAllocMapped) != cudaSuccess ||
        cudaHostGetDevicePointer((void**)&h->d_stop, h->h_stop, 0) != cudaSuccess) {
        lba_destroy(h);
        *out = nullptr;
        return set_error(ORB_ERR_CUDA, "mapped stop flag allocation failed");
    }
    *h->h_stop = 0;
    return ORB_OK;
}

// *pbStopFlag of the reference is a C++ bool written by another thread (LocalMapping::InterruptBA); the C ABI also takes an
// int32 flag.  flag_bytes selects how the relay reads it.
static inline bool read_stop_flag(const volatile void* p, int bytes) {
    return bytes == 1 ? *static_cast<const volatile uint8_t*>(p) != 0 : *static_cast<const volatile int32_t*>(p) != 0;
}

static orb_status lba_solve_impl(lba_handle* h, int32_t n_problems, const lba_problem* in, lba_result* out, const volatile void* stop_flag,
                                 int flag_bytes) {
    if (!h || !in || !out || n_problems < 1) return set_error(ORB_ERR_INVALID, "bad arguments");
    ORB_CUDA(cudaSetDevice(h->device));
    std::vector<LbaPrep> prep(n_problems);
    for (int i = 0; i < n_problems; ++i) {
        const lba_problem& p = in[i];
        if (p.n_kf < 1 || p.n_mp < 1 || p.n_edges < 1 || !p.pose || !p.fixed || !p.point || !p.edge_kf || !p.edge_mp || !p.obs ||
            !p.inv_sigma2 || !out[i].pose || !out[i].point)
            return set_error(ORB_ERR_INVALID, "incomplete lba_problem / lba_result");
        const char* why = nullptr;
        const orb_status s = lba_prepare(p, prep[i], &why);
        if (s != ORB_OK) return set_error(s, why);
    }
    const volatile int* stop = stop_flag ? h->d_stop : nullptr;
    const LbaLayout lay = lba_pack(n_problems, in, prep.data(), stop, nullptr, nullptr);
    const size_t mirror = lay.in_bytes + lay.desc_bytes;
    orb_status s = grow_device(h->d_bytes, h->d_buf, mirror + lay.work_bytes, false);
    if (s != ORB_OK || (s = grow_pinned(h->h_bytes, h->h_buf, mirror)) != ORB_OK) return s;
    uint8_t* hb = h->h_buf;
    lba_pack(n_problems, in, prep.data(), stop, hb, h->d_buf);
    const LbaDev* dev = reinterpret_cast<const LbaDev*>(hb + lay.in_bytes);
    *h->h_stop = (stop_flag && read_stop_flag(stop_flag, flag_bytes)) ? 1 : 0;
    ORB_CUDA(cudaMemcpyAsync(h->d_buf, hb, mirror, cudaMemcpyHostToDevice, h->stream));
    // k_lba keeps a problem's reduced system in shared memory iff ITS n <= LBA_SMEM_N, so the launch must carry the largest such
    // n -- not the batch-wide maximum: a batch mixing a > 24-keyframe problem with smaller ones still needs the smaller ones' slots
    int maxn = 0;
    for (int i = 0; i < n_problems; ++i)
        if (dev[i].n <= LBA_SMEM_N) maxn = std::max(maxn, dev[i].n);
    const size_t smem = lba_smem_bytes(maxn);
    int cs = cluster_size_for(n_problems, h->n_sms);
    if (const char* v = getenv("ORB_LBA_CLUSTER")) cs = std::max(1, std::min(atoi(v), cs));   // experiments: cap the cluster size
    ORB_CUDA(fit_cluster_size(k_lba, &cs, LBA_THREADS, smem));
    ORB_CUDA(launch_cluster(k_lba, n_problems, cs, LBA_THREADS, smem, h->stream, reinterpret_cast<const LbaDev*>(h->d_buf + lay.in_bytes), cs));
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    // relay *pbStopFlag to the mapped flag while the kernel runs (LocalMapping::InterruptBA writes it asynchronously)
    if (stop_flag) {
        while (cudaStreamQuery(h->stream) == cudaErrorNotReady) {
            if (read_stop_flag(stop_flag, flag_bytes)) *h->h_stop = 1;
            std::this_thread::sleep_for(std::chrono::microseconds(20));
        }
    }
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n_problems; ++i) {
        const lba_problem& p = in[i];
        const LbaDev& d = dev[i];
        ORB_CUDA(cudaMemcpyAsync(out[i].pose, d.pose, (size_t)p.n_kf * 56, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaMemcpyAsync(out[i].point, d.point, (size_t)p.n_mp * 24, cudaMemcpyDeviceToHost, h->stream));
        if (out[i].edge_chi2) ORB_CUDA(cudaMemcpyAsync(out[i].edge_chi2, d.err, (size_t)p.n_edges * 8, cudaMemcpyDeviceToHost, h->stream));
        if (out[i].edge_depth_positive)
            ORB_CUDA(cudaMemcpyAsync(out[i].edge_depth_positive, d.depthPos, (size_t)p.n_edges, cudaMemcpyDeviceToHost, h->stream));
        ORB_CUDA(cudaMemcpyAsync(hb + 256 * i, d.stats, 160, cudaMemcpyDeviceToHost, h->stream));
    }
    ORB_CUDA(cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n_problems; ++i) {
        const double* st = (const double*)(hb + 256 * i);
        if (getenv("ORB_LBA_PHASES")) {
            static const char* nm[12] = {"errors0", "build_points", "build_poses", "dinv+zero", "pair_products", "block_reduce+bs", "ldlt", "tri_solve", "landmarks+update", "errors1", "gain", "other"};
            fprintf(stderr, "[lba %d] phase kcycles:", i);
            for (int k = 0; k < 12; ++k) fprintf(stderr, " %s=%.0f", nm[k], st[8 + k] / 1e3);
            fprintf(stderr, "\n");
        }
        out[i].iterations = (int32_t)st[0];
        out[i].lambda = st[1];
        out[i].chi2 = st[2];
        out[i].trials = (int32_t)st[3];
        out[i].chi2_initial = st[4];
    }
    return ORB_OK;
}

extern "C" orb_status lba_solve_batch(lba_handle* h, int32_t n_problems, const lba_problem* in, lba_result* out,
                                      const volatile int32_t* stop_flag) {
    return lba_solve_impl(h, n_problems, in, out, stop_flag, 4);
}

extern "C" orb_status lba_solve_bool(lba_handle* h, const lba_problem* in, lba_result* out, const volatile uint8_t* stop_flag) {
    return lba_solve_impl(h, 1, in, out, stop_flag, 1);
}

extern "C" orb_status lba_solve(lba_handle* h, const lba_problem* in, lba_result* out, const volatile int32_t* stop_flag) {
    return lba_solve_impl(h, 1, in, out, stop_flag, 4);
}
