// liba_core.cuh -- Optimizer::LocalInertialBA's numeric core (/root/reference/src/Optimizer.cc:2203-2812) as
// barrier-separated SPMD phases run by a TEAM of threads (a thread-block cluster on the device; see "Execution model" below).
// Like quadtree_core.cuh, the identical source compiles for the device and for the host, so tests/host_emul can run this very
// algorithm against the CPU oracle -- by one thread, and by several threads with real barriers under ThreadSanitizer -- without a
// GPU.  There are no atomics: every sum is a gather in a fixed order, so Levenberg's accept / reject decisions do not depend on
// scheduling.
//
// g2o graph being solved (single camera, Nleft == -1):
//   vertices  VertexPose (ImuCamPose: twb += Rwb ut, Rwb = Rwb Exp(ur); G2oTypes.cc:221-244), VertexVelocity,
//             VertexGyroBias, VertexAccBias per keyframe (15 parameters, fixed or free as a whole), VertexSBAPointXYZ
//             per map point (marginalised)
//   edges     EdgeMono / EdgeStereo (G2oTypes.cc:390-490), Huber sqrt(5.991) / sqrt(7.815)
//             EdgeInertial (G2oTypes.cc:563-687), optional Huber sqrt(16.92); EdgeGyroRW / EdgeAccRW (G2oTypes.h:736-800)
//   solver    OptimizationAlgorithmLevenberg with a user lambda, BlockSolverX: landmarks eliminated by the Schur complement,
//             the reduced (15 nFree)^2 system factorised densely (LDL^T), gain ratio / lambda schedule / stop rules as g2o.
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define LIBA_HD __host__ __device__ inline
#else
#define LIBA_HD inline
#endif

// Execution model.  A TEAM works on one window: on the device a thread-block cluster of `cs` CTAs (cs = 1: one CTA); in
// tests/host_emul/liba_mt.cpp `cs` groups of host threads; in tests/host_emul/emul.cpp a single thread.  Every thread holds its own
// copy of the descriptor `P` with its place in the team (t_id / t_stride over the whole team, l_id / l_stride inside its CTA, rank).
//   LIBA_PAR_FOR / LIBA_SYNC      team-wide strided loop / team-wide barrier (cluster barrier: orders global memory across the CTAs)
//   LIBA_LOCAL_FOR / LIBA_LOCAL_SYNC   the same inside one CTA; used by the dense factorisation, which runs on rank 0 only because
//                                      it needs two barriers per column and a CTA barrier is an order of magnitude cheaper
#define LIBA_PAR_FOR(i, n) for (int i = P.t_id; i < (n); i += P.t_stride)
#define LIBA_LOCAL_FOR(i, n) for (int i = P.l_id; i < (n); i += P.l_stride)
#define LIBA_LEADER() (P.t_id == 0)
#define LIBA_RANK0() (P.rank == 0)
#if defined(__CUDA_ARCH__)
#include <cooperative_groups.h>
#define LIBA_SYNC() do { if (P.cs > 1) cooperative_groups::this_cluster().sync(); else __syncthreads(); } while (0)
#define LIBA_LOCAL_SYNC() __syncthreads()
#define LIBA_FLAG_SET(p) (*(p) = 1)
#elif defined(LIBA_EMUL_THREADS)
// tests/host_emul/liba_mt.cpp: host threads play the team with REAL barriers, so ThreadSanitizer reports a missing LIBA_SYNC, a
// LIBA_LOCAL_SYNC where a team barrier is needed, or two threads accumulating into one location, as a data race.
namespace orb {
void liba_barrier_team();
void liba_barrier_cta(int rank);
}
#define LIBA_SYNC() orb::liba_barrier_team()
#define LIBA_LOCAL_SYNC() orb::liba_barrier_cta(P.rank)
#define LIBA_FLAG_SET(p) __atomic_store_n((p), 1, __ATOMIC_RELAXED)
#else
#define LIBA_SYNC() ((void)0)
#define LIBA_LOCAL_SYNC() ((void)0)
#define LIBA_FLAG_SET(p) (*(p) = 1)
#endif

namespace orb {

#define LIBA_CHUNKS 8     // the long gathers (edges of a keyframe, co-observations of a keyframe pair) are summed in this many
                          // contiguous chunks by different threads, then the chunk sums in order: still a fixed order

struct LibaLink {   // == liba_link of include/orbslam3_b200.h
    int k1, k2, robust, pad;
    double dt;
    float dR[9], dV[3], dP[3], JRg[9], JVg[9], JVa[9], JPg[9], JPa[9], bias[6];
    double info[81], infoG[9], infoA[9];
};

struct LibaDev {
    int nKF, nMP, nE, nL, nFree, sp;   // sp = 15 nFree
    double* state;        // [nKF][21] Rwb(9) twb v bg ba
    double* state_saved;
    double* point;        // [nMP][3]
    double* point_saved;
    const int* pidx;      // [nKF] free index or -1
    const int* ekf;       // [nE]
    const int* emp;
    const double* obs;    // [nE][3]
    const double* invs2;  // [nE]
    const int* pt_off;    // [nMP + 1] edges by point (CSR, ascending edge index inside a point)
    const int* pt_edge;   // [nE]
    const int* kf_off;    // [nKF + 1] edges by keyframe (CSR, ascending edge index)
    const int* kf_edge;   // [nE]
    const int* kl_off;    // [nKF + 1] links by keyframe; entry = 2 * link + role (0: the keyframe is k1, 1: it is k2)
    const int* kl_ent;    // [2 nL]
    int nPairs;           // upper block pairs (p1 <= p2) of optimisable keyframes that share at least one map point
    const int* pair_p;    // [nPairs] p1 << 16 | p2
    const int* pair_off;  // [nPairs + 1] into co_e1 / co_e2, entries ordered by map point
    const int* co_e1;     // edge of p1 observing the shared point
    const int* co_e2;     // edge of p2
    const LibaLink* links;
    double Rcb[9], tcb[3], Rbc[9], tbc[3];
    double fx, fy, cx, cy, bf;
    double lambda_init;
    int max_iters;
    // work
    double* err;          // [nE]
    double* lerr;         // [nL][3]
    double* Hpp;          // [sp][sp]
    double* Hs;           // [sp][sp]
    double* b;            // [sp + 3 nMP]
    double* bs;           // [sp]
    double* x;            // [sp + 3 nMP]
    double* y;            // [sp]
    double* Hll;          // [nMP][9]
    double* Dinv;         // [nMP][9]
    double* W;            // [nE][18]  pose(6) x point(3)
    double* WD;           // [nE][18]  W D^-1 (per trial)
    double* Wdb;          // [nE][6]   W D^-1 b_l
    double* Epp;          // [nE][27]  upper triangle (21) of the edge's 6 x 6 pose block, then its 6 b terms
    double* Lblk;         // [nL][930] 30 x 30 block over [k1 15 | k2 15] of the inertial + random-walk edges, then 30 b terms
    double* part;         // [LIBA_CHUNKS * max(27 nKF, 36 nPairs)] chunk sums of the two long gathers
    double* part_b;       // [LIBA_CHUNKS * 6 nKF] chunk sums of the reduced right-hand side
    double* Ypan;         // [15][sp] panel D1 L21^T of the blocked factorisation
    int* flag;            // [4] solver failure flag
    double* red;          // reduction scratch of this CTA (device: shared memory, one double per warp; emulation: per thread)
    double* partials;     // [16] per-CTA partial results of a team reduction (global memory)
    int t_id, t_stride;   // this thread's place in the team ...
    int l_id, l_stride;   // ... and inside its CTA
    int rank, cs;         // CTA rank in the team, CTAs per team
    // results
    double* out_scalars;  // iterations, trials, lambda, chi2, chi2_initial, chi2 of the last trial
    unsigned char* dpos;  // [nE] isDepthPositive at the final estimate
};

// ---- small fixed-size linear algebra -------------------------------------------------------------------------------
LIBA_HD void m3_mul(const double* a, const double* b, double* c) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) c[3 * i + j] = a[3 * i] * b[j] + a[3 * i + 1] * b[3 + j] + a[3 * i + 2] * b[6 + j];
}
LIBA_HD void m3_T(const double* a, double* t) {
    t[0] = a[0]; t[1] = a[3]; t[2] = a[6]; t[3] = a[1]; t[4] = a[4]; t[5] = a[7]; t[6] = a[2]; t[7] = a[5]; t[8] = a[8];
}
LIBA_HD void m3_vec(const double* a, const double* v, double* o) {
    for (int i = 0; i < 3; ++i) o[i] = a[3 * i] * v[0] + a[3 * i + 1] * v[1] + a[3 * i + 2] * v[2];
}
LIBA_HD void m3_skew(const double* w, double* W) {
    W[0] = 0; W[1] = -w[2]; W[2] = w[1]; W[3] = w[2]; W[4] = 0; W[5] = -w[0]; W[6] = -w[1]; W[7] = w[0]; W[8] = 0;
}
LIBA_HD void so3_exp(const double* w, double* R) {   // G2oTypes.cc:908-929 (NormalizeRotation omitted: ~1e-16)
    const double d2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2], d = sqrt(d2);
    double W[9], W2[9];
    m3_skew(w, W);
    m3_mul(W, W, W2);
    const double a = d < 1e-5 ? 1.0 : sin(d) / d, c = d < 1e-5 ? 0.5 : (1.0 - cos(d)) / d2;
    for (int i = 0; i < 9; ++i) R[i] = ((i & 3) == 0 ? 1.0 : 0.0) + a * W[i] + c * W2[i];
}
LIBA_HD void so3_log(const double* R, double* w) {   // G2oTypes.cc:931-945
    const double tr = R[0] + R[4] + R[8];
    w[0] = (R[7] - R[5]) / 2; w[1] = (R[2] - R[6]) / 2; w[2] = (R[3] - R[1]) / 2;
    const double costheta = (tr - 1.0) * 0.5;
    if (costheta > 1 || costheta < -1) return;
    const double theta = acos(costheta), s = sin(theta);
    if (fabs(s) < 1e-5) return;
    for (int i = 0; i < 3; ++i) w[i] = theta * w[i] / s;
}
LIBA_HD void so3_jr(const double* v, bool inverse, double* J) {   // G2oTypes.cc:947-985
    const double d2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2], d = sqrt(d2);
    for (int i = 0; i < 9; ++i) J[i] = (i & 3) == 0 ? 1.0 : 0.0;
    if (d < 1e-5) return;
    double W[9], W2[9];
    m3_skew(v, W);
    m3_mul(W, W, W2);
    if (inverse) { const double c = 1.0 / d2 - (1.0 + cos(d)) / (2.0 * d * sin(d)); for (int i = 0; i < 9; ++i) J[i] += W[i] / 2 + W2[i] * c; }
    else { const double a = (1.0 - cos(d)) / d2, c = (d - sin(d)) / (d2 * d); for (int i = 0; i < 9; ++i) J[i] += -W[i] * a + W2[i] * c; }
}
LIBA_HD bool m3_inv(const double* M, double* Mi) {
    const double c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
    const double det = M[0] * c00 + M[1] * c01 + M[2] * c02;
    const double id = 1.0 / det;
    if (!isfinite(id)) return false;          // det == 0, subnormal, or not finite: the block solver reports failure
    Mi[0] = c00 * id; Mi[1] = (M[2] * M[7] - M[1] * M[8]) * id; Mi[2] = (M[1] * M[5] - M[2] * M[4]) * id;
    Mi[3] = c01 * id; Mi[4] = (M[0] * M[8] - M[2] * M[6]) * id; Mi[5] = (M[2] * M[3] - M[0] * M[5]) * id;
    Mi[6] = c02 * id; Mi[7] = (M[1] * M[6] - M[0] * M[7]) * id; Mi[8] = (M[0] * M[4] - M[1] * M[3]) * id;
    return true;
}
LIBA_HD double liba_huber(double e, double delta, double dsqr, double* w) {
    if (e <= dsqr) { *w = 1.0; return e; }
    const double s = sqrt(e);
    *w = delta / s;
    return 2 * s * delta - dsqr;
}

// float32 a . b with every product and sum rounded on its own, as the reference's Eigen float arithmetic and the oracle round them
// (DESIGN.md §2: float32 without FMA contraction).  Written with plain operators, nvcc fuses them into FFMA, which rounds once: the
// bias-corrected preintegrated deltas then differ by a float ulp from the reference's, and so do the inertial residuals built on them.
LIBA_HD float liba_fdot3(const float* a, const float* b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
#else
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];      // host builds of this file use -ffp-contract=off
#endif
}

// team-wide sum / max in a fixed order (warp tree, warps in order, CTAs in rank order): every thread receives the same value
LIBA_HD double liba_sum(const LibaDev& P, double v) {
#if defined(__CUDA_ARCH__)
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) P.red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += P.red[w];
    if (P.cs > 1) {
        if (threadIdx.x == 0) P.partials[P.rank] = s;
        cooperative_groups::this_cluster().sync();
        s = 0;
        for (int r = 0; r < P.cs; ++r) s += P.partials[r];
        cooperative_groups::this_cluster().sync();      // partials are rewritten by the next reduction
    }
    return s;
#elif defined(LIBA_EMUL_THREADS)
    liba_barrier_team();
    P.red[P.t_id] = v;
    liba_barrier_team();
    double s = 0;
    for (int w = 0; w < P.t_stride; ++w) s += P.red[w];
    return s;
#else
    (void)P;
    return v;
#endif
}
LIBA_HD double liba_max(const LibaDev& P, double v) {
#if defined(__CUDA_ARCH__)
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) P.red[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = P.red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) s = fmax(s, P.red[w]);
    if (P.cs > 1) {
        if (threadIdx.x == 0) P.partials[P.rank] = s;
        cooperative_groups::this_cluster().sync();
        s = P.partials[0];
        for (int r = 1; r < P.cs; ++r) s = fmax(s, P.partials[r]);
        cooperative_groups::this_cluster().sync();
    }
    return s;
#elif defined(LIBA_EMUL_THREADS)
    liba_barrier_team();
    P.red[P.t_id] = v;
    liba_barrier_team();
    double s = P.red[0];
    for (int w = 1; w < P.t_stride; ++w) s = fmax(s, P.red[w]);
    return s;
#else
    (void)P;
    return v;
#endif
}

// ---- edges -----------------------------------------------------------------------------------------------------------
LIBA_HD void liba_cam_pose(const LibaDev& P, const double* s, double* Rcw, double* tcw) {   // ImuCamPose::Update tail
    double Rbw[9], tbw[3];
    m3_T(s, Rbw);
    m3_vec(Rbw, s + 9, tbw);
    for (int i = 0; i < 3; ++i) tbw[i] = -tbw[i];
    m3_mul(P.Rcb, Rbw, Rcw);
    m3_vec(P.Rcb, tbw, tcw);
    for (int i = 0; i < 3; ++i) tcw[i] += P.tcb[i];
}

// EdgeMono / EdgeStereo: residual r (3), optionally Jp (D x 3, point) and Jx (D x 6, pose).  Returns D.
LIBA_HD int liba_reproj(const LibaDev& P, int e, double* r, double* Jp, double* Jx) {
    double Rcw[9], tcw[3], Xc[3];
    liba_cam_pose(P, P.state + 21 * (size_t)P.ekf[e], Rcw, tcw);
    m3_vec(Rcw, P.point + 3 * (size_t)P.emp[e], Xc);
    for (int i = 0; i < 3; ++i) Xc[i] += tcw[i];
    const double* z = P.obs + 3 * (size_t)e;
    const int D = z[2] < 0 ? 2 : 3;
    const double u = P.fx * Xc[0] / Xc[2] + P.cx, v = P.fy * Xc[1] / Xc[2] + P.cy;
    r[0] = z[0] - u;
    r[1] = z[1] - v;
    r[2] = D == 3 ? z[2] - (u - P.bf * (1 / Xc[2])) : 0.0;
    if (Jp) {
        double pj[9] = {P.fx / Xc[2], 0, -P.fx * Xc[0] / (Xc[2] * Xc[2]), 0, P.fy / Xc[2], -P.fy * Xc[1] / (Xc[2] * Xc[2]), 0, 0, 0};
        if (D == 3) { pj[6] = pj[0]; pj[7] = pj[1]; pj[8] = pj[2] + P.bf * (1.0 / (Xc[2] * Xc[2])); }
        double Xb[3];
        m3_vec(P.Rbc, Xc, Xb);
        for (int i = 0; i < 3; ++i) Xb[i] += P.tbc[i];
        const double S[18] = {0, Xb[2], -Xb[1], 1, 0, 0, -Xb[2], 0, Xb[0], 0, 1, 0, Xb[1], -Xb[0], 0, 0, 0, 1};
        for (int d = 0; d < D; ++d) {
            double pr[3];
            for (int c = 0; c < 3; ++c) {
                Jp[3 * d + c] = -(pj[3 * d] * Rcw[c] + pj[3 * d + 1] * Rcw[3 + c] + pj[3 * d + 2] * Rcw[6 + c]);
                pr[c] = pj[3 * d] * P.Rcb[c] + pj[3 * d + 1] * P.Rcb[3 + c] + pj[3 * d + 2] * P.Rcb[6 + c];
            }
            for (int c = 0; c < 6; ++c) Jx[6 * d + c] = pr[0] * S[c] + pr[1] * S[6 + c] + pr[2] * S[12 + c];
        }
    }
    return D;
}

// EdgeInertial: e9 and (optionally) J, 9 x 24 over [pose1 6 | v1 3 | bg1 3 | ba1 3 | pose2 6 | v2 3]
LIBA_HD void liba_inertial(const LibaDev& P, const LibaLink& L, double* e9, double* J) {
    const double* s1 = P.state + 21 * (size_t)L.k1;
    const double* s2 = P.state + 21 * (size_t)L.k2;
    const double g[3] = {0, 0, -(double)9.81f};
    float dbg[3], dba[3], wv[3];
    for (int i = 0; i < 3; ++i) { dba[i] = (float)s1[18 + i] - L.bias[i]; dbg[i] = (float)s1[15 + i] - L.bias[3 + i]; }
    for (int i = 0; i < 3; ++i) wv[i] = liba_fdot3(L.JRg + 3 * i, dbg);
    const double wd[3] = {wv[0], wv[1], wv[2]};
    double E[9], dR[9], dV[3], dP[3];
    so3_exp(wd, E);
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            dR[3 * i + j] = (double)(float)((double)L.dR[3 * i] * E[j] + (double)L.dR[3 * i + 1] * E[3 + j] + (double)L.dR[3 * i + 2] * E[6 + j]);
    for (int i = 0; i < 3; ++i) {
        dV[i] = (double)(L.dV[i] + liba_fdot3(L.JVg + 3 * i, dbg) + liba_fdot3(L.JVa + 3 * i, dba));
        dP[i] = (double)(L.dP[i] + liba_fdot3(L.JPg + 3 * i, dbg) + liba_fdot3(L.JPa + 3 * i, dba));
    }
    double Rbw1[9], dRt[9], t1[9], eR[9], er[3];
    m3_T(s1, Rbw1);
    m3_T(dR, dRt);
    m3_mul(dRt, Rbw1, t1);
    m3_mul(t1, s2, eR);
    so3_log(eR, er);
    const double dt = L.dt;
    double a[3], bb[3], ra[3], rb[3];
    for (int i = 0; i < 3; ++i) {
        a[i] = s2[12 + i] - s1[12 + i] - g[i] * dt;
        bb[i] = s2[9 + i] - s1[9 + i] - s1[12 + i] * dt - g[i] * dt * dt / 2;
    }
    m3_vec(Rbw1, a, ra);
    m3_vec(Rbw1, bb, rb);
    for (int i = 0; i < 3; ++i) { e9[i] = er[i]; e9[3 + i] = ra[i] - dV[i]; e9[6 + i] = rb[i] - dP[i]; }
    if (!J) return;
    for (int i = 0; i < 9 * 24; ++i) J[i] = 0.0;
#define LIBA_PUT(row0, col0, M, sgn) for (int i_ = 0; i_ < 3; ++i_) for (int j_ = 0; j_ < 3; ++j_) J[((row0) + i_) * 24 + (col0) + j_] = (sgn) * (M)[3 * i_ + j_];
    double invJr[9], R2t[9], m1[9], m2[9], sk[9], I3[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
    so3_jr(er, true, invJr);
    m3_T(s2, R2t);
    m3_mul(invJr, R2t, m1);
    m3_mul(m1, s1, m2);
    LIBA_PUT(0, 0, m2, -1.0)
    m3_skew(ra, sk);
    LIBA_PUT(3, 0, sk, 1.0)
    m3_skew(rb, sk);
    LIBA_PUT(6, 0, sk, 1.0)
    LIBA_PUT(6, 3, I3, -1.0)
    LIBA_PUT(3, 6, Rbw1, -1.0)
    for (int i = 0; i < 9; ++i) m1[i] = Rbw1[i] * dt;
    LIBA_PUT(6, 6, m1, -1.0)
    double JRg[9], JVg[9], JPg[9], JVa[9], JPa[9], jw[3], eRt[9], Jr[9];
    for (int i = 0; i < 9; ++i) { JRg[i] = L.JRg[i]; JVg[i] = L.JVg[i]; JPg[i] = L.JPg[i]; JVa[i] = L.JVa[i]; JPa[i] = L.JPa[i]; }
    const double dbgd[3] = {dbg[0], dbg[1], dbg[2]};
    m3_vec(JRg, dbgd, jw);
    so3_jr(jw, false, Jr);
    m3_T(eR, eRt);
    m3_mul(invJr, eRt, m1);
    m3_mul(m1, Jr, m2);
    m3_mul(m2, JRg, m1);
    LIBA_PUT(0, 9, m1, -1.0)
    LIBA_PUT(3, 9, JVg, -1.0)
    LIBA_PUT(6, 9, JPg, -1.0)
    LIBA_PUT(3, 12, JVa, -1.0)
    LIBA_PUT(6, 12, JPa, -1.0)
    LIBA_PUT(0, 15, invJr, 1.0)
    m3_mul(Rbw1, s2, m1);
    LIBA_PUT(6, 18, m1, 1.0)
    LIBA_PUT(3, 21, Rbw1, 1.0)
#undef LIBA_PUT
}

LIBA_HD void liba_kf_oplus(double* s, const double* d15) {
    double dt[3], E[9], R[9];
    m3_vec(s, d15 + 3, dt);
    for (int i = 0; i < 3; ++i) s[9 + i] += dt[i];
    so3_exp(d15, E);
    m3_mul(s, E, R);
    for (int i = 0; i < 9; ++i) s[i] = R[i];
    for (int i = 0; i < 3; ++i) { s[12 + i] += d15[6 + i]; s[15 + i] += d15[9 + i]; s[18 + i] += d15[12 + i]; }
}

// ---- phases -----------------------------------------------------------------------------------------------------------
struct LibaHuber { double dM, dS, dI, sqM, sqS, sqI; };

LIBA_HD LibaHuber liba_huber_constants() {
    LibaHuber h;
    h.dM = (double)(float)sqrt(5.991); h.dS = (double)(float)sqrt(7.815); h.dI = sqrt(16.92);
    h.sqM = (double)(float)(h.dM * h.dM); h.sqS = (double)(float)(h.dS * h.dS); h.sqI = (double)(float)(h.dI * h.dI);
    return h;
}

LIBA_HD void liba_link_chi2(const LibaDev& P, const LibaLink& L, double* c3) {
    double e9[9];
    liba_inertial(P, L, e9, nullptr);
    double c = 0;
    for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) c += e9[i] * L.info[9 * i + j] * e9[j];
    c3[0] = c;
    const double* s1 = P.state + 21 * (size_t)L.k1;
    const double* s2 = P.state + 21 * (size_t)L.k2;
    double cg = 0, ca = 0;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            cg += (s2[15 + i] - s1[15 + i]) * L.infoG[3 * i + j] * (s2[15 + j] - s1[15 + j]);
            ca += (s2[18 + i] - s1[18 + i]) * L.infoA[3 * i + j] * (s2[18 + j] - s1[18 + j]);
        }
    c3[1] = cg; c3[2] = ca;
}

LIBA_HD double liba_compute_errors(const LibaDev& P, const LibaHuber& H) {   // computeActiveErrors + activeRobustChi2
    double chi = 0;
    LIBA_PAR_FOR(e, P.nE) {
        double r[3];
        const int D = liba_reproj(P, e, r, nullptr, nullptr);
        const double c = P.invs2[e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
        P.err[e] = c;
        double w;
        chi += liba_huber(c, D == 2 ? H.dM : H.dS, D == 2 ? H.sqM : H.sqS, &w);
    }
    LIBA_PAR_FOR(l, P.nL) {
        double c3[3], w;
        liba_link_chi2(P, P.links[l], c3);
        for (int i = 0; i < 3; ++i) P.lerr[3 * l + i] = c3[i];
        chi += (P.links[l].robust ? liba_huber(c3[0], H.dI, H.sqI, &w) : c3[0]) + c3[1] + c3[2];
    }
    return liba_sum(P, chi);
}

LIBA_HD int liba_tri(int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); }   // (i <= j) of a 6 x 6 upper triangle -> [0, 21)

// linearizeOplus + constructQuadraticForm of every edge.  Phase 1 computes per-edge / per-link blocks, phase 2 gathers them into
// H_pp and b in a fixed order (edges of a keyframe ascending, then its links ascending).
LIBA_HD void liba_build(const LibaDev& P, const LibaHuber& H) {
    const int sp = P.sp;
    LIBA_PAR_FOR(i, sp * sp) P.Hpp[i] = 0.0;
    LIBA_PAR_FOR(l, P.nMP) {     // a thread owns a map point: H_ll and b_l stay in registers
        double hl[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, bl[3] = {0, 0, 0};
        for (int k = P.pt_off[l]; k < P.pt_off[l + 1]; ++k) {
            const int e = P.pt_edge[k];
            double r[3], Jp[9], Jx[18];
            const int D = liba_reproj(P, e, r, Jp, Jx);
            const double c2 = P.invs2[e] * (r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
            double w;
            liba_huber(c2, D == 2 ? H.dM : H.dS, D == 2 ? H.sqM : H.sqS, &w);
            const double om = w * P.invs2[e];
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) { double s = 0; for (int d = 0; d < D; ++d) s += Jp[3 * d + i] * Jp[3 * d + j]; hl[3 * i + j] += om * s; }
                double s = 0; for (int d = 0; d < D; ++d) s += Jp[3 * d + i] * r[d];
                bl[i] += -om * s;
            }
            const bool freeKf = P.pidx[P.ekf[e]] >= 0;
            double* We = P.W + 18 * (size_t)e;
            double* Ee = P.Epp + 27 * (size_t)e;
            for (int i = 0; i < 6; ++i) {
                for (int j = 0; j < 3; ++j) { double s = 0; for (int d = 0; d < D; ++d) s += Jx[6 * d + i] * Jp[3 * d + j]; We[3 * i + j] = freeKf ? om * s : 0.0; }
                for (int j = i; j < 6; ++j) { double s = 0; for (int d = 0; d < D; ++d) s += Jx[6 * d + i] * Jx[6 * d + j]; Ee[liba_tri(i, j)] = om * s; }
                double s = 0; for (int d = 0; d < D; ++d) s += Jx[6 * d + i] * r[d];
                Ee[21 + i] = -om * s;
            }
        }
        for (int i = 0; i < 9; ++i) P.Hll[9 * (size_t)l + i] = hl[i];
        for (int i = 0; i < 3; ++i) P.b[sp + 3 * l + i] = bl[i];
    }
    LIBA_PAR_FOR(t, P.nL * 25) {   // inertial links -> one 30 x 30 block over [k1 15 | k2 15] each; a thread owns one column (24: the tail)
        const int l = t / 25, cb = t % 25;
        const LibaLink& L = P.links[l];
        double* B = P.Lblk + 930 * (size_t)l;
        double e9[9], J[9 * 24];
        liba_inertial(P, L, e9, J);
        double c = 0;
        for (int i = 0; i < 9; ++i) for (int j = 0; j < 9; ++j) c += e9[i] * L.info[9 * i + j] * e9[j];
        double w = 1.0;
        if (L.robust) liba_huber(c, H.dI, H.sqI, &w);
        if (cb < 24) {        // column cb of w Info J, then J^T times it (inertial columns 0..23 sit at block columns 0..23)
            double oj[9];
            for (int i = 0; i < 9; ++i) { double s2 = 0; for (int k = 0; k < 9; ++k) s2 += L.info[9 * i + k] * J[k * 24 + cb]; oj[i] = w * s2; }
            for (int ca = 0; ca < 24; ++ca) { double s2 = 0; for (int k = 0; k < 9; ++k) s2 += J[k * 24 + ca] * oj[k]; B[ca * 30 + cb] = s2; }
            for (int ca = 24; ca < 30; ++ca) B[ca * 30 + cb] = 0.0;
        } else {              // columns 24..29 (bias of k2: random walks only, added below) and the right-hand side
            double Oe[9];
            for (int i = 0; i < 9; ++i) { double s2 = 0; for (int k = 0; k < 9; ++k) s2 += L.info[9 * i + k] * e9[k]; Oe[i] = w * s2; }
            for (int ca = 0; ca < 30; ++ca) for (int cc = 24; cc < 30; ++cc) B[ca * 30 + cc] = 0.0;
            for (int ca = 0; ca < 24; ++ca) { double s2 = 0; for (int k = 0; k < 9; ++k) s2 += J[k * 24 + ca] * Oe[k]; B[900 + ca] = -s2; }
            for (int ca = 24; ca < 30; ++ca) B[900 + ca] = 0.0;
        }
    }
    LIBA_SYNC();
    LIBA_PAR_FOR(t, P.nKF * 27 * LIBA_CHUNKS) {     // chunk sums of the 21 + 6 per-edge pose terms over a keyframe's edges
        const int k = t / (27 * LIBA_CHUNKS), slot = (t / LIBA_CHUNKS) % 27, ch = t % LIBA_CHUNKS;
        if (P.pidx[k] < 0) continue;
        const int n0 = P.kf_off[k], len = P.kf_off[k + 1] - n0;
        const int a = n0 + (int)((long long)len * ch / LIBA_CHUNKS), b = n0 + (int)((long long)len * (ch + 1) / LIBA_CHUNKS);
        double acc = 0.0;
        for (int n = a; n < b; ++n) acc += P.Epp[27 * (size_t)P.kf_edge[n] + slot];
        P.part[t] = acc;
    }
    LIBA_PAR_FOR(l, P.nL) {      // the two bias random walks of a link (e = b2 - b1, J1 = -I, J2 = I) go into the same block
        const LibaLink& L = P.links[l];
        double* B = P.Lblk + 930 * (size_t)l;
        const double* s1 = P.state + 21 * (size_t)L.k1;
        const double* s2 = P.state + 21 * (size_t)L.k2;
        for (int which = 0; which < 2; ++which) {
            const double* info = which == 0 ? L.infoG : L.infoA;
            const int off = which == 0 ? 9 : 12, so = which == 0 ? 15 : 18;
            double e3[3], Oe3[3];
            for (int i = 0; i < 3; ++i) e3[i] = s2[so + i] - s1[so + i];
            for (int i = 0; i < 3; ++i) Oe3[i] = info[3 * i] * e3[0] + info[3 * i + 1] * e3[1] + info[3 * i + 2] * e3[2];
            for (int i = 0; i < 3; ++i) {
                B[900 + off + i] += Oe3[i];
                B[900 + 15 + off + i] += -Oe3[i];
                for (int j = 0; j < 3; ++j) {
                    B[(off + i) * 30 + off + j] += info[3 * i + j];
                    B[(15 + off + i) * 30 + 15 + off + j] += info[3 * i + j];
                    B[(off + i) * 30 + 15 + off + j] -= info[3 * i + j];
                    B[(15 + off + i) * 30 + off + j] -= info[3 * i + j];
                }
            }
        }
    }
    LIBA_SYNC();
    LIBA_PAR_FOR(t, P.nKF * 240) {      // a thread owns one entry of a keyframe's 15 x 15 diagonal block (t % 240 < 225) or of its b
        const int k = t / 240, q = t % 240, pi = P.pidx[k];
        if (pi < 0) continue;
        const bool isB = q >= 225;
        const int r = isB ? q - 225 : q / 15, c = isB ? 0 : q % 15;
        double acc = 0.0;
        if (r < 6 && (isB || c < 6)) {
            const int slot = isB ? 21 + r : (r <= c ? liba_tri(r, c) : liba_tri(c, r));
            const double* pp = P.part + ((size_t)k * 27 + slot) * LIBA_CHUNKS;
            for (int ch = 0; ch < LIBA_CHUNKS; ++ch) acc += pp[ch];
        }
        for (int n = P.kl_off[k]; n < P.kl_off[k + 1]; ++n) {
            const int l = P.kl_ent[n] >> 1, o = 15 * (P.kl_ent[n] & 1);
            acc += isB ? P.Lblk[930 * (size_t)l + 900 + o + r] : P.Lblk[930 * (size_t)l + (o + r) * 30 + o + c];
        }
        if (isB) P.b[15 * pi + r] = acc; else P.Hpp[(size_t)(15 * pi + r) * sp + 15 * pi + c] = acc;
    }
    LIBA_PAR_FOR(t, P.nL * 225) {       // the k1-k2 coupling of a link (at most one link per keyframe pair: liba_pack checks)
        const int l = t / 225, r = (t % 225) / 15, c = t % 15;
        const int p1 = P.pidx[P.links[l].k1], p2 = P.pidx[P.links[l].k2];
        if (p1 < 0 || p2 < 0) continue;
        const double* B = P.Lblk + 930 * (size_t)l;
        P.Hpp[(size_t)(15 * p1 + r) * sp + 15 * p2 + c] = B[r * 30 + 15 + c];
        P.Hpp[(size_t)(15 * p2 + c) * sp + 15 * p1 + r] = B[(15 + c) * 30 + r];
    }
    LIBA_SYNC();
}

// (H + lambda I) x = b through the Schur complement on the landmarks; false on a singular block / pivot
LIBA_HD bool liba_solve_system(const LibaDev& P, double lambda) {
    const int sp = P.sp;
    LIBA_PAR_FOR(i, sp * sp) P.Hs[i] = P.Hpp[i] + ((i / sp) == (i % sp) ? lambda : 0.0);
    if (LIBA_LEADER()) { P.flag[0] = 0; P.flag[1] = 0; }
    LIBA_SYNC();
    LIBA_PAR_FOR(l, P.nMP) {     // D^-1 per landmark, W D^-1 and W D^-1 b_l per edge
        double D[9], Di[9];
        for (int i = 0; i < 9; ++i) D[i] = P.Hll[9 * (size_t)l + i];
        D[0] += lambda; D[4] += lambda; D[8] += lambda;
        if (!m3_inv(D, Di)) { LIBA_FLAG_SET(&P.flag[0]); continue; }
        for (int i = 0; i < 9; ++i) P.Dinv[9 * (size_t)l + i] = Di[i];
        const double* bl = P.b + sp + 3 * l;
        double Dib[3];
        for (int i = 0; i < 3; ++i) Dib[i] = Di[3 * i] * bl[0] + Di[3 * i + 1] * bl[1] + Di[3 * i + 2] * bl[2];
        for (int k = P.pt_off[l]; k < P.pt_off[l + 1]; ++k) {
            const int e = P.pt_edge[k];
            const double* W1 = P.W + 18 * (size_t)e;
            double* WD = P.WD + 18 * (size_t)e;
            for (int i = 0; i < 6; ++i) {
                for (int j = 0; j < 3; ++j) WD[3 * i + j] = W1[3 * i] * Di[j] + W1[3 * i + 1] * Di[3 + j] + W1[3 * i + 2] * Di[6 + j];
                P.Wdb[6 * (size_t)e + i] = W1[3 * i] * Dib[0] + W1[3 * i + 1] * Dib[1] + W1[3 * i + 2] * Dib[2];
            }
        }
    }
    LIBA_SYNC();
    LIBA_PAR_FOR(t, P.nKF * 6 * LIBA_CHUNKS) {      // reduced right-hand side, chunk sums of W D^-1 b_l over a keyframe's edges
        const int k = t / (6 * LIBA_CHUNKS), r = (t / LIBA_CHUNKS) % 6, ch = t % LIBA_CHUNKS;
        if (P.pidx[k] < 0) continue;
        const int n0 = P.kf_off[k], len = P.kf_off[k + 1] - n0;
        const int a = n0 + (int)((long long)len * ch / LIBA_CHUNKS), b = n0 + (int)((long long)len * (ch + 1) / LIBA_CHUNKS);
        double acc = 0.0;
        for (int n = a; n < b; ++n) acc += P.Wdb[6 * (size_t)P.kf_edge[n] + r];
        P.part_b[t] = acc;
    }
    LIBA_PAR_FOR(t, P.nPairs * 36 * LIBA_CHUNKS) {   // Schur complement, chunk sums: one entry of one 6 x 6 block, one chunk of the pair's list
        const int q = t / (36 * LIBA_CHUNKS), ij = (t / LIBA_CHUNKS) % 36, ch = t % LIBA_CHUNKS, i = ij / 6, j = ij % 6;
        const int n0 = P.pair_off[q], len = P.pair_off[q + 1] - n0;
        const int a = n0 + (int)((long long)len * ch / LIBA_CHUNKS), b = n0 + (int)((long long)len * (ch + 1) / LIBA_CHUNKS);
        double acc = 0.0;
        for (int n = a; n < b; ++n) {
            const double* WD = P.WD + 18 * (size_t)P.co_e1[n] + 3 * i;
            const double* W2 = P.W + 18 * (size_t)P.co_e2[n] + 3 * j;
            acc += WD[0] * W2[0] + WD[1] * W2[1] + WD[2] * W2[2];
        }
        P.part[t] = acc;
    }
    LIBA_SYNC();
    LIBA_PAR_FOR(t, P.nKF * 15) {      // reduced right-hand side: chunk sums in order
        const int k = t / 15, r = t % 15, pi = P.pidx[k];
        if (pi < 0) continue;
        double acc = 0.0;
        if (r < 6) for (int ch = 0; ch < LIBA_CHUNKS; ++ch) acc += P.part_b[((size_t)k * 6 + r) * LIBA_CHUNKS + ch];
        P.bs[15 * pi + r] = P.b[15 * pi + r] - acc;
    }
    LIBA_PAR_FOR(t, P.nPairs * 36) {   // a thread owns one entry of one 6 x 6 block (upper block triangle only): chunk sums in order
        const int q = t / 36, i = (t % 36) / 6, j = t % 6;
        const int p1 = P.pair_p[q] >> 16, p2 = P.pair_p[q] & 0xffff;
        double* dst = P.Hs + (size_t)(15 * p1 + i) * sp + 15 * p2 + j;
        const double* pp = P.part + (size_t)t * LIBA_CHUNKS;
        double acc = 0.0;
        for (int ch = 0; ch < LIBA_CHUNKS; ++ch) acc += pp[ch];
        *dst -= acc;
    }
    LIBA_SYNC();
    // Dense LDL^T of Hs (upper triangle) and the triangular solves, on the team's first CTA only, BLOCKED by keyframe (15 x 15 pivots):
    // per block column (a) one thread factorises the diagonal block, (b) a thread per remaining column solves the 15 x 15 unit
    // lower system for the panel (Y = L11^-1 A12 = D1 L21^T, kept in Ypan; L21^T = D1^-1 Y stored in place), (c) the trailing
    // update A22 -= Y^T (D1^-1 Y).  Afterwards row j holds D_j at (j,j) and L(i,j) at (j,i), i > j.  Seven CTA barriers per block
    // column over the whole solve instead of six per scalar column.
    if (LIBA_RANK0()) {
        bool bad = P.flag[0] != 0;            // a singular landmark block (set before the team barrier above)
        const int nb = sp / 15;
        for (int J = 0; J < nb && !bad; ++J) {
            const int j0 = 15 * J, j1 = j0 + 15, m = sp - j1;
            if (P.l_id == 0) {
                bool ok = true;
                for (int jj = j0; jj < j1 && ok; ++jj) {
                    const double dj = P.Hs[(size_t)jj * sp + jj];
                    if (!(fabs(dj) > 0) || !isfinite(dj)) { ok = false; break; }
                    for (int ii = jj + 1; ii < j1; ++ii) {
                        const double f = P.Hs[(size_t)jj * sp + ii] / dj;
                        for (int kk = ii; kk < j1; ++kk) P.Hs[(size_t)ii * sp + kk] -= f * P.Hs[(size_t)jj * sp + kk];
                    }
                    for (int ii = jj + 1; ii < j1; ++ii) P.Hs[(size_t)jj * sp + ii] /= dj;
                }
                if (!ok) LIBA_FLAG_SET(&P.flag[1]);
            }
            LIBA_LOCAL_SYNC();
            bad = P.flag[1] != 0;             // uniform: written before the barrier, by one thread
            if (bad) break;
            LIBA_LOCAL_FOR(t, m) {
                const int c = j1 + t;
                double yv[15];
                for (int a = 0; a < 15; ++a) {
                    double sacc = P.Hs[(size_t)(j0 + a) * sp + c];
                    for (int b2 = 0; b2 < a; ++b2) sacc -= P.Hs[(size_t)(j0 + b2) * sp + j0 + a] * yv[b2];
                    yv[a] = sacc;
                }
                for (int a = 0; a < 15; ++a) {
                    P.Ypan[(size_t)a * sp + c] = yv[a];
                    P.Hs[(size_t)(j0 + a) * sp + c] = yv[a] / P.Hs[(size_t)(j0 + a) * sp + j0 + a];
                }
            }
            LIBA_LOCAL_SYNC();
            LIBA_LOCAL_FOR(t, m * m) {
                const int ii = j1 + t / m, kk = j1 + t % m;
                if (kk >= ii) {
                    double sacc = 0.0;
                    for (int a = 0; a < 15; ++a) sacc += P.Ypan[(size_t)a * sp + ii] * P.Hs[(size_t)(j0 + a) * sp + kk];
                    P.Hs[(size_t)ii * sp + kk] -= sacc;
                }
            }
            LIBA_LOCAL_SYNC();
        }
        if (bad) {
            LIBA_LOCAL_SYNC();                // every thread has read the flags before flag[0] is (re)written
            if (P.l_id == 0) LIBA_FLAG_SET(&P.flag[0]);
        } else {
            // forward L y = bs, diagonal, backward L^T x = y, block by block
            LIBA_LOCAL_FOR(i2, sp) P.y[i2] = P.bs[i2];
            LIBA_LOCAL_SYNC();
            for (int J = 0; J < nb; ++J) {
                const int j0 = 15 * J, j1 = j0 + 15, m = sp - j1;
                if (P.l_id == 0)
                    for (int a = 1; a < 15; ++a) {
                        double sacc = P.y[j0 + a];
                        for (int b2 = 0; b2 < a; ++b2) sacc -= P.Hs[(size_t)(j0 + b2) * sp + j0 + a] * P.y[j0 + b2];
                        P.y[j0 + a] = sacc;
                    }
                LIBA_LOCAL_SYNC();
                LIBA_LOCAL_FOR(t, m) {
                    const int c = j1 + t;
                    double sacc = 0.0;
                    for (int a = 0; a < 15; ++a) sacc += P.Hs[(size_t)(j0 + a) * sp + c] * P.y[j0 + a];
                    P.y[c] -= sacc;
                }
                LIBA_LOCAL_SYNC();
            }
            LIBA_LOCAL_FOR(i2, sp) P.y[i2] /= P.Hs[(size_t)i2 * sp + i2];
            LIBA_LOCAL_SYNC();
            for (int J = nb - 1; J >= 0; --J) {
                const int j0 = 15 * J, j1 = j0 + 15;
                LIBA_LOCAL_FOR(a, 15) {
                    double sacc = 0.0;
                    for (int c = j1; c < sp; ++c) sacc += P.Hs[(size_t)(j0 + a) * sp + c] * P.y[c];
                    P.y[j0 + a] -= sacc;
                }
                LIBA_LOCAL_SYNC();
                if (P.l_id == 0)
                    for (int a = 13; a >= 0; --a) {
                        double sacc = P.y[j0 + a];
                        for (int b2 = a + 1; b2 < 15; ++b2) sacc -= P.Hs[(size_t)(j0 + a) * sp + j0 + b2] * P.y[j0 + b2];
                        P.y[j0 + a] = sacc;
                    }
                LIBA_LOCAL_SYNC();
            }
            LIBA_LOCAL_FOR(i2, sp) P.x[i2] = P.y[i2];
        }
    }
    LIBA_SYNC();      // x (keyframe part) and the failure flag reach the whole team
    const bool failed = P.flag[0] != 0;
    if (!failed) {
        LIBA_PAR_FOR(l, P.nMP) {
            double c[3] = {P.b[sp + 3 * l], P.b[sp + 3 * l + 1], P.b[sp + 3 * l + 2]};
            for (int k = P.pt_off[l]; k < P.pt_off[l + 1]; ++k) {
                const int e = P.pt_edge[k], p = P.pidx[P.ekf[e]];
                if (p < 0) continue;
                const double* Wm = P.W + 18 * (size_t)e;
                for (int j = 0; j < 3; ++j) for (int i = 0; i < 6; ++i) c[j] -= Wm[3 * i + j] * P.x[15 * p + i];
            }
            const double* Di = P.Dinv + 9 * (size_t)l;
            for (int i = 0; i < 3; ++i) P.x[sp + 3 * l + i] = Di[3 * i] * c[0] + Di[3 * i + 1] * c[1] + Di[3 * i + 2] * c[2];
        }
        LIBA_SYNC();
    }
    return !failed;
}

// the whole optimisation: g2o SparseOptimizer::optimize(max_iters) over OptimizationAlgorithmLevenberg
LIBA_HD void liba_optimize(const LibaDev& P) {
    const LibaHuber H = liba_huber_constants();
    const int sp = P.sp, sl = 3 * P.nMP;
    double lambda = P.lambda_init, ni = 2, currentChi = 0, iniChi0 = 0, lastChi = 0;
    int nBad = 0, iters = 0, trials = 0;
    for (int it = 0; it < P.max_iters; ++it) {
        currentChi = liba_compute_errors(P, H);
        lastChi = currentChi;
        if (it == 0) iniChi0 = currentChi;
        double tempChi = currentChi;
        const double iniChi = currentChi;
        liba_build(P, H);
        if (it == 0) {
            if (!(P.lambda_init > 0)) {      // computeLambdaInit: tau * max diagonal over all vertices
                double md = 0;
                LIBA_PAR_FOR(j, sp) md = fmax(md, fabs(P.Hpp[(size_t)j * sp + j]));
                LIBA_PAR_FOR(l, P.nMP) for (int j = 0; j < 3; ++j) md = fmax(md, fabs(P.Hll[9 * (size_t)l + 4 * j]));
                lambda = 1e-5 * liba_max(P, md);
            }
            ni = 2;
            nBad = 0;
        }
        double rho = 0;
        int qmax = 0;
        do {
            LIBA_PAR_FOR(i, 21 * P.nKF) P.state_saved[i] = P.state[i];      // push
            LIBA_PAR_FOR(i, sl) P.point_saved[i] = P.point[i];
            LIBA_SYNC();
            const bool ok2 = liba_solve_system(P, lambda);
            LIBA_PAR_FOR(k, P.nKF) if (P.pidx[k] >= 0) liba_kf_oplus(P.state + 21 * (size_t)k, P.x + 15 * P.pidx[k]);
            LIBA_PAR_FOR(i, sl) P.point[i] += P.x[sp + i];
            LIBA_SYNC();
            tempChi = liba_compute_errors(P, H);
            lastChi = tempChi;
            if (!ok2) tempChi = 1.7976931348623157e308;
            double sc = 0;
            LIBA_PAR_FOR(j, sp + sl) sc += P.x[j] * (lambda * P.x[j] + P.b[j]);
            const double scale = liba_sum(P, sc) + 1e-3;
            rho = (currentChi - tempChi) / scale;
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
                LIBA_SYNC();
                LIBA_PAR_FOR(i, 21 * P.nKF) P.state[i] = P.state_saved[i];  // pop
                LIBA_PAR_FOR(i, sl) P.point[i] = P.point_saved[i];
                LIBA_SYNC();
            }
            ++qmax;
            ++trials;
        } while (rho < 0 && qmax < 10);
        ++iters;
        if (qmax == 10 || rho == 0) break;
        if ((iniChi - currentChi) * 1e3 < iniChi) ++nBad; else nBad = 0;
        if (nBad >= 3) break;
    }
    LIBA_PAR_FOR(e, P.nE) {      // EdgeMono / EdgeStereo::isDepthPositive at the final estimate (G2oTypes.cc:212-215)
        double Rcw[9], tcw[3];
        liba_cam_pose(P, P.state + 21 * (size_t)P.ekf[e], Rcw, tcw);
        const double* X = P.point + 3 * (size_t)P.emp[e];
        P.dpos[e] = (Rcw[6] * X[0] + Rcw[7] * X[1] + Rcw[8] * X[2] + tcw[2]) > 0.0 ? 1 : 0;
    }
    if (LIBA_LEADER()) {
        P.out_scalars[0] = iters; P.out_scalars[1] = trials; P.out_scalars[2] = lambda; P.out_scalars[3] = currentChi; P.out_scalars[4] = iniChi0;
        P.out_scalars[5] = lastChi;
    }
    LIBA_SYNC();
}

}  // namespace orb
