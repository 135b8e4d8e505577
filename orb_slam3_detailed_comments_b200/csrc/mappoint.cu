// mappoint.cu -- the two MapPoint maintenance routines that feed the projection searches, batched over map points:
//   MapPoint::ComputeDistinctiveDescriptors  /root/reference/src/MapPoint.cc:438-520
//       the observation descriptor whose median Hamming distance to the others is smallest (first minimum)
//   MapPoint::UpdateNormalAndDepth           /root/reference/src/MapPoint.cc:567-640
//       mean viewing direction and the scale-invariance distances mfMaxDistance / mfMinDistance
// (LocalMapping calls both for every new / fused map point: LocalMapping.cc:300-340, 860-875; pinhole keyframes.)
#include <algorithm>
#include <vector>

#include "extractor.h"
#include "devmath.cuh"

using namespace orb;
using namespace orbdev;

namespace orb {

// One warp per map point.  Row i of the distance matrix is never stored: lane i histograms its N distances (0..256) in
// shared memory and walks the histogram to the element of rank (int)(0.5 (N - 1)) -- what sort() + vDists[0.5*(N-1)] returns.
__global__ void __launch_bounds__(32) k_distinctive(const int* __restrict__ ooff, const uint8_t* __restrict__ odesc, int* __restrict__ best_out) {
    __shared__ uint16_t s_hist[32][258];
    const int mp = blockIdx.x, lane = threadIdx.x;
    const int o0 = ooff[mp], N = ooff[mp + 1] - o0;
    if (N <= 0) {
        if (lane == 0) best_out[mp] = -1;     // vDescriptors.empty(): the descriptor is left untouched
        return;
    }
    const int k = (int)(0.5 * (double)(N - 1));
    uint32_t best = 0xffffffffu;              // median << 20 | row: strict '<' keeps the first minimum
    for (int i = lane; i < N; i += 32) {
        uint16_t* hist = s_hist[lane];
        for (int b = 0; b < 257; ++b) hist[b] = 0;
        const uint4* di = reinterpret_cast<const uint4*>(odesc + (size_t)(o0 + i) * 32);
        const uint4 a0 = __ldg(di), a1 = __ldg(di + 1);
        for (int j = 0; j < N; ++j) {
            const uint4* dj = reinterpret_cast<const uint4*>(odesc + (size_t)(o0 + j) * 32);
            const uint4 b0 = __ldg(dj), b1 = __ldg(dj + 1);
            const int d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                          __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
            hist[d] += 1;                     // Distances[i][i] = 0 included
        }
        int acc = 0, median = 256;
        for (int b = 0; b < 257; ++b) {
            acc += hist[b];
            if (acc > k) { median = b; break; }
        }
        best = min(best, ((uint32_t)median << 20) | (uint32_t)i);
    }
    best = __reduce_min_sync(0xffffffffu, best);
    if (lane == 0) best_out[mp] = (int)(best & 0xfffffu);
}

// One thread per map point: the sums run in observation order like the reference's map walk.
__global__ void __launch_bounds__(128) k_normal_depth(int np, const int* __restrict__ ooff, const float* __restrict__ ocenter,
                                                     const float* __restrict__ pos, const float* __restrict__ refc, const int* __restrict__ reflevel,
                                                     const float* __restrict__ scale, int nLevels, float* __restrict__ normal, float* __restrict__ maxd,
                                                     float* __restrict__ mind) {
    const int mp = blockIdx.x * blockDim.x + threadIdx.x;
    if (mp >= np) return;
    const int o0 = ooff[mp], N = ooff[mp + 1] - o0;
    if (N <= 0) return;                       // observations.empty(): nothing changes
    const float X = pos[3 * (size_t)mp], Y = pos[3 * (size_t)mp + 1], Z = pos[3 * (size_t)mp + 2];
    float nx = 0.f, ny = 0.f, nz = 0.f;
    for (int o = o0; o < o0 + N; ++o) {
        const float vx = fsub(X, ocenter[3 * (size_t)o]), vy = fsub(Y, ocenter[3 * (size_t)o + 1]), vz = fsub(Z, ocenter[3 * (size_t)o + 2]);
        const float nrm = fsqrt(fadd(fmul(vx, vx), fadd(fmul(vy, vy), fmul(vz, vz))));     // Eigen: x^2 + (y^2 + z^2)
        nx = fadd(nx, fdiv(vx, nrm)); ny = fadd(ny, fdiv(vy, nrm)); nz = fadd(nz, fdiv(vz, nrm));
    }
    const float px = fsub(X, refc[3 * (size_t)mp]), py = fsub(Y, refc[3 * (size_t)mp + 1]), pz = fsub(Z, refc[3 * (size_t)mp + 2]);
    const float dist = fsqrt(fadd(fmul(px, px), fadd(fmul(py, py), fmul(pz, pz))));
    const float mx = fmul(dist, scale[reflevel[mp]]);
    maxd[mp] = mx;
    mind[mp] = fdiv(mx, scale[nLevels - 1]);
    const float fn = (float)N;
    normal[3 * (size_t)mp] = fdiv(nx, fn); normal[3 * (size_t)mp + 1] = fdiv(ny, fn); normal[3 * (size_t)mp + 2] = fdiv(nz, fn);
}

}  // namespace orb

extern "C" orb_status orbp_distinctive_descriptors(orbx_handle* h, int32_t n_points, const int32_t* obs_offset, const uint8_t* obs_desc,
                                                   int32_t* best_index_out) {
    if (!h || n_points < 0 || !obs_offset || !best_index_out) return set_error(ORB_ERR_INVALID, "bad arguments");
    if (n_points == 0) return ORB_OK;
    const int nobs = obs_offset[n_points];
    if (nobs < 0 || (nobs > 0 && !obs_desc)) return set_error(ORB_ERR_INVALID, "bad observation table");
    for (int i = 0; i < n_points; ++i)
        if (obs_offset[i + 1] - obs_offset[i] > 65535) return set_error(ORB_ERR_UNSUPPORTED, "map point with more than 65535 observations");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    cudaStream_t st = h->stream;
    const int* d_off; const uint8_t* d_desc; int* d_best;
    auto layout = [&](Carve& c) {
        d_off = stage_in(c, obs_offset, (size_t)n_points + 1, false);
        d_best = stage_out(c, best_index_out, n_points, false);
        d_desc = stage_in(c, obs_desc, (size_t)nobs * 32, false);
    };
    const Carve c = carve_scratch(h->po_bytes, h->d_po, h->capturing, st, layout);
    if (c.status != ORB_OK) return c.status;
    k_distinctive<<<n_points, 32, 0, st>>>(d_off, d_desc, d_best);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return copy_out(c);
}

extern "C" orb_status orbp_update_normal_and_depth(orbx_handle* h, int32_t n_points, const int32_t* obs_offset, const float* obs_center,
                                                   const float* world_pos, const float* ref_center, const int32_t* ref_level,
                                                   float* normal_out, float* max_dist_out, float* min_dist_out) {
    if (!h || n_points < 0 || !obs_offset || !world_pos || !ref_center || !ref_level || !normal_out || !max_dist_out || !min_dist_out)
        return set_error(ORB_ERR_INVALID, "bad arguments");
    if (n_points == 0) return ORB_OK;
    const int nobs = obs_offset[n_points];
    if (nobs < 0 || (nobs > 0 && !obs_center)) return set_error(ORB_ERR_INVALID, "bad observation table");
    for (int i = 0; i < n_points; ++i)
        if (ref_level[i] < 0 || ref_level[i] >= h->cfg.n_levels) return set_error(ORB_ERR_INVALID, "reference level outside the pyramid");
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const size_t np = (size_t)n_points;
    cudaStream_t st = h->stream;
    const int *d_off, *d_lv; const float *d_oc, *d_pos, *d_rc, *d_sc; float *d_n, *d_mx, *d_mn;
    auto layout = [&](Carve& c) {
        d_off = stage_in(c, obs_offset, np + 1, false); d_oc = stage_in(c, obs_center, (size_t)nobs * 3, false);
        d_pos = stage_in(c, world_pos, np * 3, false); d_rc = stage_in(c, ref_center, np * 3, false);
        d_lv = stage_in(c, ref_level, np, false); d_sc = stage_in(c, h->scale.data(), (size_t)h->cfg.n_levels, false);
        // outputs start from the caller's current values: points without observations keep them
        d_n = stage_in(c, normal_out, np * 3, false); d_mx = stage_in(c, max_dist_out, np, false); d_mn = stage_in(c, min_dist_out, np, false);
        c.copy_back(normal_out, d_n, np * 3); c.copy_back(max_dist_out, d_mx, np); c.copy_back(min_dist_out, d_mn, np);
    };
    const Carve c = carve_scratch(h->po_bytes, h->d_po, h->capturing, st, layout);
    if (c.status != ORB_OK) return c.status;
    k_normal_depth<<<(n_points + 127) / 128, 128, 0, st>>>(n_points, d_off, d_oc, d_pos, d_rc, d_lv, d_sc, h->cfg.n_levels, d_n, d_mx, d_mn);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return copy_out(c);
}
