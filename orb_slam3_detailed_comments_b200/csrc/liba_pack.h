// liba_pack.h -- host-side flattening of a liba_problem into one blob laid out for liba_core.cuh.  Pure host C++ so that the
// CUDA wrapper (liba.cu) and the CPU emulation harness (tests/host_emul) share it.
//   [io]   state, point, err, lerr, out_scalars, dpos            host -> device before, device -> host after
//   [in]   obs, invs2, links, pidx, ekf, emp, the CSRs, co-observation lists    host -> device before
//   [work] saved state, normal equations, Schur scratch    zero-filled on the device
// The host range of io | in must be zero before the fill: its padding and the outputs in io are uploaded as they are.
#pragma once
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>

#include "../../include/orbslam3_b200.h"
#include "liba_core.cuh"
#include "pack.h"

namespace orb {

struct LibaLayout { size_t io_bytes = 0, in_bytes = 0, work_bytes = 0, total = 0; };

static_assert(sizeof(liba_link) == 1080 && sizeof(LibaLink) == 1080, "liba_link layout");

// devBase == nullptr: sizes only.  Pointers inside *dev are relative to devBase (== host for the CPU emulation).
// Returns total == 0 when two links join the same keyframe pair (the gather in liba_build assumes at most one; the reference
// creates one EdgeInertial per keyframe and its mPrevKF, Optimizer.cc:2430-2500).
inline LibaLayout liba_pack(const liba_problem& p, uint8_t* host, uint8_t* devBase, LibaDev* dev) {
    const int nKF = p.n_kf, nMP = p.n_mp, nE = p.n_edges, nL = p.n_links;
    std::vector<int32_t> pidx(nKF);
    int nFree = 0;
    for (int k = 0; k < nKF; ++k) pidx[k] = p.fixed[k] ? -1 : nFree++;
    const size_t sp = 15 * (size_t)nFree, sl = 3 * (size_t)nMP;

    // CSRs: edges by map point, edges by keyframe, links by keyframe
    auto csr = [](int nRows, int n, auto rowOf, std::vector<int32_t>& off, std::vector<int32_t>& ent, auto entOf) {
        off.assign(nRows + 1, 0);
        for (int i = 0; i < n; ++i) ++off[rowOf(i) + 1];
        for (int r = 0; r < nRows; ++r) off[r + 1] += off[r];
        ent.resize(n ? n : 1);
        std::vector<int32_t> cur(off.begin(), off.end() - 1);
        for (int i = 0; i < n; ++i) ent[cur[rowOf(i)]++] = entOf(i);
    };
    std::vector<int32_t> ptOff, ptEdge, kfOff, kfEdge, klOff, klEnt;
    csr(nMP, nE, [&](int e) { return p.edge_mp[e]; }, ptOff, ptEdge, [](int e) { return e; });
    csr(nKF, nE, [&](int e) { return p.edge_kf[e]; }, kfOff, kfEdge, [](int e) { return e; });
    csr(nKF, 2 * nL, [&](int i) { return (i & 1) ? p.links[i >> 1].k2 : p.links[i >> 1].k1; }, klOff, klEnt, [](int i) { return i; });
    LibaLayout lay;
    for (int k = 0; k < nKF; ++k)          // one link per keyframe pair
        for (int a = klOff[k]; a < klOff[k + 1]; ++a)
            for (int b = a + 1; b < klOff[k + 1]; ++b) {
                const liba_link &A = p.links[klEnt[a] >> 1], &B = p.links[klEnt[b] >> 1];
                if ((A.k1 == B.k1 && A.k2 == B.k2) || (A.k1 == B.k2 && A.k2 == B.k1)) return lay;
            }
    if (nFree > 0xffff) return lay;

    // co-observation lists per upper block pair (p1 <= p2), ordered by map point
    std::vector<int32_t> pairCount((size_t)nFree * nFree, 0), pairP, pairOff(1, 0), coE1, coE2;
    auto forEachCo = [&](auto fn) {
        for (int l = 0; l < nMP; ++l)
            for (int a = ptOff[l]; a < ptOff[l + 1]; ++a)
                for (int b = ptOff[l]; b < ptOff[l + 1]; ++b) {
                    const int pa = pidx[p.edge_kf[ptEdge[a]]], pb = pidx[p.edge_kf[ptEdge[b]]];
                    if (pa >= 0 && pb >= 0 && pa <= pb) fn(pa, pb, ptEdge[a], ptEdge[b]);
                }
    };
    forEachCo([&](int pa, int pb, int, int) { ++pairCount[(size_t)pa * nFree + pb]; });
    std::vector<int32_t> pairIdx((size_t)nFree * nFree, -1);
    for (int a = 0; a < nFree; ++a)
        for (int b = a; b < nFree; ++b)
            if (pairCount[(size_t)a * nFree + b]) {
                pairIdx[(size_t)a * nFree + b] = (int32_t)pairP.size();
                pairP.push_back(a << 16 | b);
                pairOff.push_back(pairOff.back() + pairCount[(size_t)a * nFree + b]);
            }
    const int nPairs = (int)pairP.size();
    const size_t nCo = (size_t)pairOff.back();
    coE1.resize(nCo ? nCo : 1); coE2.resize(nCo ? nCo : 1);
    {
        std::vector<int32_t> cur(pairOff.begin(), pairOff.end() - 1);
        forEachCo([&](int pa, int pb, int e1, int e2) { const int q = pairIdx[(size_t)pa * nFree + pb]; coE1[cur[q]] = e1; coE2[cur[q]++] = e2; });
    }

    PackRegion r{devBase, host, 16};
    LibaDev d;
    d.state = r.put(p.state, 21 * (size_t)nKF); d.point = r.put(p.point, sl);
    d.err = r.take<double>(nE); d.lerr = r.take<double>(3 * (size_t)nL); d.out_scalars = r.take<double>(8); d.dpos = r.take<uint8_t>(nE);
    lay.io_bytes = r.bytes();
    d.obs = r.put(p.obs, 3 * (size_t)nE); d.invs2 = r.put(p.inv_sigma2, nE); d.links = reinterpret_cast<const LibaLink*>(r.put(p.links, nL));
    d.pidx = r.put(pidx.data(), nKF); d.ekf = r.put(p.edge_kf, nE); d.emp = r.put(p.edge_mp, nE);
    d.pt_off = r.put(ptOff.data(), (size_t)nMP + 1); d.pt_edge = r.put(ptEdge.data(), nE);
    d.kf_off = r.put(kfOff.data(), (size_t)nKF + 1); d.kf_edge = r.put(kfEdge.data(), nE);
    d.kl_off = r.put(klOff.data(), (size_t)nKF + 1); d.kl_ent = r.put(klEnt.data(), 2 * (size_t)nL);
    d.pair_p = r.put(pairP.data(), nPairs); d.pair_off = r.put(pairOff.data(), (size_t)nPairs + 1);
    d.co_e1 = r.put(coE1.data(), nCo); d.co_e2 = r.put(coE2.data(), nCo);
    lay.in_bytes = r.bytes() - lay.io_bytes;
    d.state_saved = r.take<double>(21 * (size_t)nKF); d.point_saved = r.take<double>(sl);
    d.Hpp = r.take<double>(sp * sp); d.Hs = r.take<double>(sp * sp);
    d.b = r.take<double>(sp + sl); d.bs = r.take<double>(sp);
    d.x = r.take<double>(sp + sl); d.y = r.take<double>(sp);
    d.Hll = r.take<double>(9 * (size_t)nMP); d.Dinv = r.take<double>(9 * (size_t)nMP);
    d.W = r.take<double>(18 * (size_t)nE); d.WD = r.take<double>(18 * (size_t)nE);
    d.Wdb = r.take<double>(6 * (size_t)nE); d.Epp = r.take<double>(27 * (size_t)nE);
    d.Lblk = r.take<double>(930 * (size_t)nL);
    d.flag = r.take<int>(4); d.partials = r.take<double>(16); d.part = r.take<double>((size_t)LIBA_CHUNKS * std::max((size_t)27 * nKF, (size_t)36 * nPairs));
    d.part_b = r.take<double>((size_t)LIBA_CHUNKS * 6 * nKF); d.Ypan = r.take<double>(15 * sp);
    lay.total = r.bytes();
    lay.work_bytes = lay.total - lay.io_bytes - lay.in_bytes;
    if (!dev) return lay;

    d.nKF = nKF; d.nMP = nMP; d.nE = nE; d.nL = nL; d.nFree = nFree; d.sp = (int)sp; d.nPairs = nPairs;
    for (int i = 0; i < 9; ++i) d.Rcb[i] = p.Tcb[i];
    for (int i = 0; i < 3; ++i) d.tcb[i] = p.Tcb[9 + i];
    m3_T(d.Rcb, d.Rbc);
    m3_vec(d.Rbc, d.tcb, d.tbc);
    for (int i = 0; i < 3; ++i) d.tbc[i] = -d.tbc[i];
    d.fx = p.fx; d.fy = p.fy; d.cx = p.cx; d.cy = p.cy; d.bf = p.bf;
    d.lambda_init = p.lambda_init;
    d.max_iters = p.max_iters;
    d.red = nullptr;
    d.t_id = 0; d.t_stride = 1; d.l_id = 0; d.l_stride = 1; d.rank = 0; d.cs = 1;      // a team of one thread; the launcher overrides per thread
    *dev = d;
    return lay;
}

// io region -> liba_result
inline void liba_unpack(const liba_problem& p, const uint8_t* host, const LibaDev& d, const uint8_t* devBase, liba_result* r) {
    auto H = [&](const void* devPtr) { return reinterpret_cast<const double*>(host + (reinterpret_cast<const uint8_t*>(devPtr) - devBase)); };
    memcpy(r->state, H(d.state), 8 * 21 * (size_t)p.n_kf);
    memcpy(r->point, H(d.point), 8 * 3 * (size_t)p.n_mp);
    if (r->edge_chi2) memcpy(r->edge_chi2, H(d.err), 8 * (size_t)p.n_edges);
    if (r->link_chi2) memcpy(r->link_chi2, H(d.lerr), 8 * 3 * (size_t)p.n_links);
    if (r->edge_depth_positive) memcpy(r->edge_depth_positive, host + (d.dpos - devBase), (size_t)p.n_edges);
    const double* o = H(d.out_scalars);
    r->iterations = (int32_t)o[0]; r->trials = (int32_t)o[1]; r->lambda = o[2]; r->chi2 = o[3]; r->chi2_initial = o[4];
    r->chi2_last_trial = o[5];
}

}  // namespace orb
