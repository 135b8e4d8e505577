// lba_pack.h -- host-side index structures and device layout of a batch of lba_problems for k_lba (lba.cu).  Pure host C++ so
// that the CPU emulation harness (tests/host_emul) checks them without a GPU.
//   [in]    per problem: inputs, index structures      mirrored on the host, one host -> device copy with the descriptors
//   [desc]  one LbaDev per problem
//   [work]  per problem: state, normal equations, Schur scratch, outputs
#pragma once
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "../../include/orbslam3_b200.h"
#include "pack.h"

struct int4;   // CUDA's vector type; only pointed to here

namespace orb {

#define LBA_ICH 128      // co-observation items per Schur task
#define LBA_SMEM_N 144   // reduced systems up to 144 x 144 (24 free keyframes) are factorised in shared memory
#define LBA_PCH 8        // chunks per pose of the per-pose reduction (build_poses)

struct LbaDev {
    int nKF, nMP, nE, nP, n;   // n = 6 * nP
    // inputs
    const double* pose0;   // [nKF][7] qx qy qz qw tx ty tz
    const double* point0;  // [nMP][3]
    const int* pidx;       // [nKF] pose index or -1 (fixed)
    const int* ekf;
    const int* emp;
    const double* obs;     // [nE][3], ur < 0 => monocular edge
    const double* invs2;
    const int* mpStart;    // [nMP + 1]
    const int* mpEdge;     // edges grouped by map point
    const int* poseStart;  // [nP + 1]
    const int* poseEdge;   // edges grouped by free pose
    const int* pairStart;  // [nPairBlocks + 1]: item slots of pose-block pair b are [pairStart[b], pairStart[b+1])
    const int* ptItemStart;  // null: k_lba does not read it
    const int4* ptItem;      // (e1, e2, 0, landmark): same landmark, pose(e1) <= pose(e2), grouped by pose-block pair
    int nItems, nTasks, nFreeEdges;   // nItems: 0, k_lba does not read it
    const int* taskStart;   // [nTasks + 1] item ranges (<= LBA_ICH items, never across a pose-block pair)
    const int* blockTask;   // [nPairBlocks + 1] tasks of every pose-block pair
    double* taskSum;        // [nTasks][36]
    double* BD;             // [nE][18] B_e D_l^-1
    const int* poseSlot;     // [nE] position of the edge in the pose-sorted order (-1: fixed pose)
    const int* blockP1;    // [nPairBlocks]
    const int* blockP2;
    int nPairBlocks;
    double fx, fy, cx, cy, bf, lambdaInit;
    int maxIters;
    const volatile int* stop;   // mapped host flag or null
    // state + scratch
    double* pose;     // current estimate
    double* point;
    double* poseSave;
    double* pointSave;
    double* Hpl;      // [nE][18]
    double* W;        // [pose-sorted slot][27] per-edge pose terms (21 upper H + 6 b)
    double* Prod;     // null: k_lba does not read it
    double* Hll;      // [nMP][9]
    double* bl;       // [nMP][3]
    double* Dinv;     // [nMP][9]
    double* db;       // [nMP][3]
    double* Hpp;      // [nP][36]
    double* bp;       // [nP][6]
    double* xl;       // [nMP][3]
    double* HsGlobal; // [n][n] when n > LBA_SMEM_N
    double* posePart; // [nP * LBA_PCH][27] partial pose sums
    double* HsBlocks; // [nPairBlocks][36] Schur sums per pose-block pair
    double* bs;       // [n] reduced right-hand side
    double* xp;       // [n] pose update
    double* partials; // [LBA_CS_MAX] cross-CTA reduction scratch
    int* flags;       // [0] / [2] stop requested (alternating), [1] factorisation ok
    double* err;      // [nE] chi2 per edge (last evaluation)
    // outputs
    uint8_t* depthPos;   // [nE]
    double* stats;       // iterations, lambda, chi2, trials, initial chi2
};

struct LbaItem { int32_t e1, e2, slot, l; };   // one co-observation; k_lba reads it as an int4

struct LbaPrep {   // host-side index structures of one problem
    int nP = 0, nBlocks = 0;
    std::vector<int> pidx, mpStart, mpEdge, poseStart, poseEdge, pairStart, blockP1, blockP2, poseSlot;
    std::vector<LbaItem> ptItem;
    std::vector<int> taskStart, blockTask;
};

// ORB_OK, or the status and *why of a problem k_lba does not take
inline orb_status lba_prepare(const lba_problem& in, LbaPrep& R, const char** why) {
    const int nKF = in.n_kf, nMP = in.n_mp, nE = in.n_edges;
    R.pidx.assign(nKF, -1);
    R.nP = 0;
    for (int k = 0; k < nKF; ++k)
        if (!in.fixed[k]) R.pidx[k] = R.nP++;
    if (R.nP > 160) {
        *why = "more than 160 free keyframes in one local BA";
        return ORB_ERR_UNSUPPORTED;
    }
    R.mpStart.assign(nMP + 1, 0);
    R.poseStart.assign(R.nP + 1, 0);
    for (int e = 0; e < nE; ++e) {
        if (in.edge_kf[e] < 0 || in.edge_kf[e] >= nKF || in.edge_mp[e] < 0 || in.edge_mp[e] >= nMP) {
            *why = "edge index out of range";
            return ORB_ERR_INVALID;
        }
        ++R.mpStart[in.edge_mp[e] + 1];
        const int p = R.pidx[in.edge_kf[e]];
        if (p >= 0) ++R.poseStart[p + 1];
    }
    for (int l = 0; l < nMP; ++l) R.mpStart[l + 1] += R.mpStart[l];
    for (int p = 0; p < R.nP; ++p) R.poseStart[p + 1] += R.poseStart[p];
    R.mpEdge.resize(nE);
    R.poseEdge.resize(R.poseStart[R.nP]);
    {
        std::vector<int> a(R.mpStart.begin(), R.mpStart.end() - 1), b(R.poseStart.begin(), R.poseStart.end() - 1);
        for (int e = 0; e < nE; ++e) {
            R.mpEdge[a[in.edge_mp[e]]++] = e;
            const int p = R.pidx[in.edge_kf[e]];
            if (p >= 0) R.poseEdge[b[p]++] = e;
        }
    }
    // upper pose-block pairs that share at least one landmark (the sparsity pattern of H_schur,
    // block_solver.hpp:199-238) + every diagonal block
    const int nP = R.nP;
    auto forEachCo = [&](auto fn) {   // co-observations (e1, e2) of landmark l, pose(e1) <= pose(e2), landmark by landmark
        for (int l = 0; l < nMP; ++l)
            for (int a = R.mpStart[l]; a < R.mpStart[l + 1]; ++a) {
                const int e1 = R.mpEdge[a], p1 = R.pidx[in.edge_kf[e1]];
                if (p1 < 0) continue;
                for (int b = R.mpStart[l]; b < R.mpStart[l + 1]; ++b) {
                    const int e2 = R.mpEdge[b], p2 = R.pidx[in.edge_kf[e2]];
                    if (p2 > p1 || (p2 == p1 && b == a)) fn(p1, p2, e1, e2, l);   // a landmark has one edge per keyframe; guard duplicates
                }
            }
    };
    std::vector<int> cnt((size_t)nP * nP, 0);
    forEachCo([&](int p1, int p2, int, int, int) { ++cnt[(size_t)p1 * nP + p2]; });
    std::vector<int> blockOf((size_t)nP * nP, -1);
    R.blockP1.clear(); R.blockP2.clear(); R.pairStart.assign(1, 0);
    for (int p1 = 0; p1 < nP; ++p1)
        for (int p2 = p1; p2 < nP; ++p2)
            if (cnt[(size_t)p1 * nP + p2] > 0 || p1 == p2) {
                blockOf[(size_t)p1 * nP + p2] = (int)R.blockP1.size();
                R.blockP1.push_back(p1);
                R.blockP2.push_back(p2);
                R.pairStart.push_back(R.pairStart.back() + cnt[(size_t)p1 * nP + p2]);
            }
    R.nBlocks = (int)R.blockP1.size();
    R.ptItem.assign(R.pairStart.back(), LbaItem{0, 0, 0, 0});   // items stored block by block
    std::vector<int> fill(R.pairStart.begin(), R.pairStart.end() - 1);
    forEachCo([&](int p1, int p2, int e1, int e2, int l) { R.ptItem[fill[blockOf[(size_t)p1 * nP + p2]]++] = LbaItem{e1, e2, 0, l}; });
    R.taskStart.assign(1, 0);
    R.blockTask.assign(1, 0);
    for (int b = 0; b < R.nBlocks; ++b) {
        for (int k = R.pairStart[b]; k < R.pairStart[b + 1]; k += LBA_ICH) R.taskStart.push_back(std::min(k + LBA_ICH, R.pairStart[b + 1]));
        R.blockTask.push_back((int)R.taskStart.size() - 1);
    }
    R.poseSlot.assign(nE, -1);
    for (int k = 0; k < (int)R.poseEdge.size(); ++k) R.poseSlot[R.poseEdge[k]] = k;
    return ORB_OK;
}

struct LbaLayout { size_t in_bytes = 0, desc_bytes = 0, work_bytes = 0; };

// Lays out n prepared problems: [in] and [desc] at host (the descriptors at host + in_bytes) and at dev, [work] after them at dev.
// Every array starts on 256 bytes; the inputs that may be empty keep one spare element.  dev == nullptr: sizes only.
// stop: the device address of the mapped stop flag, or null.
inline LbaLayout lba_pack(int n, const lba_problem* in, const LbaPrep* prep, const volatile int* stop, uint8_t* host, uint8_t* dev) {
    LbaLayout lay;
    std::vector<LbaDev> D(n);
    PackRegion inputs{dev, host, 256};
    for (int i = 0; i < n; ++i) {
        const lba_problem& p = in[i];
        const LbaPrep& R = prep[i];
        LbaDev& d = D[i];
        d.nKF = p.n_kf; d.nMP = p.n_mp; d.nE = p.n_edges; d.nP = R.nP; d.n = 6 * R.nP;
        d.nFreeEdges = (int)R.poseEdge.size(); d.nTasks = (int)R.taskStart.size() - 1; d.nPairBlocks = R.nBlocks;
        d.fx = p.fx; d.fy = p.fy; d.cx = p.cx; d.cy = p.cy; d.bf = p.bf; d.lambdaInit = p.lambda_init; d.maxIters = p.max_iters;
        d.stop = stop;
        d.pose0 = inputs.put(p.pose, 7 * (size_t)p.n_kf); d.point0 = inputs.put(p.point, 3 * (size_t)p.n_mp);
        d.pidx = inputs.put(R.pidx.data(), R.pidx.size()); d.ekf = inputs.put(p.edge_kf, p.n_edges); d.emp = inputs.put(p.edge_mp, p.n_edges);
        d.obs = inputs.put(p.obs, 3 * (size_t)p.n_edges); d.invs2 = inputs.put(p.inv_sigma2, p.n_edges);
        d.mpStart = inputs.put(R.mpStart.data(), R.mpStart.size()); d.mpEdge = inputs.put(R.mpEdge.data(), R.mpEdge.size());
        d.poseStart = inputs.put(R.poseStart.data(), R.poseStart.size()); d.poseEdge = inputs.put(R.poseEdge.data(), R.poseEdge.size(), 1);
        d.pairStart = inputs.put(R.pairStart.data(), R.pairStart.size());
        d.ptItem = reinterpret_cast<const int4*>(inputs.put(R.ptItem.data(), R.ptItem.size(), 1));
        d.poseSlot = inputs.put(R.poseSlot.data(), R.poseSlot.size());
        d.taskStart = inputs.put(R.taskStart.data(), R.taskStart.size()); d.blockTask = inputs.put(R.blockTask.data(), R.blockTask.size());
        d.blockP1 = inputs.put(R.blockP1.data(), R.blockP1.size(), 1); d.blockP2 = inputs.put(R.blockP2.data(), R.blockP2.size(), 1);
    }
    lay.in_bytes = inputs.bytes();
    lay.desc_bytes = (sizeof(LbaDev) * n + 255) / 256 * 256;
    PackRegion work{dev ? dev + lay.in_bytes + lay.desc_bytes : nullptr, nullptr, 256};
    for (int i = 0; i < n; ++i) {
        LbaDev& d = D[i];
        const size_t nKF = d.nKF, nMP = d.nMP, nE = d.nE, nP = d.nP, nn = d.n;
        d.pose = work.take<double>(7 * nKF); d.point = work.take<double>(3 * nMP); d.poseSave = work.take<double>(7 * nKF); d.pointSave = work.take<double>(3 * nMP);
        d.Hpl = work.take<double>(18 * nE); d.W = work.take<double>(27 * (d.nFreeEdges + 1));
        d.posePart = work.take<double>(27 * (nP * LBA_PCH + 1));
        d.HsBlocks = work.take<double>(36 * (d.nPairBlocks + 1));
        d.bs = work.take<double>(nn + 1); d.xp = work.take<double>(nn + 1);
        d.partials = work.take<double>(64); d.flags = work.take<int>(16);
        d.taskSum = work.take<double>(36 * (d.nTasks + 2)); d.BD = work.take<double>(18 * (nE + 1));
        d.Hll = work.take<double>(9 * nMP); d.bl = work.take<double>(3 * nMP); d.Dinv = work.take<double>(9 * nMP); d.db = work.take<double>(3 * nMP);
        d.Hpp = work.take<double>(36 * nP + 1); d.bp = work.take<double>(6 * nP + 1); d.xl = work.take<double>(3 * nMP);
        d.HsGlobal = work.take<double>(nn > LBA_SMEM_N ? nn * nn : 1);
        d.err = work.take<double>(nE); d.depthPos = work.take<uint8_t>(nE); d.stats = work.take<double>(32);
    }
    lay.work_bytes = work.off + 256;
    if (dev) memcpy(host + lay.in_bytes, D.data(), sizeof(LbaDev) * n);
    return lay;
}

}  // namespace orb
