// triangulation.cu -- ORBmatcher::SearchForTriangulation (/root/reference/src/ORBmatcher.cc:1045-1323) for
// single-camera keyframes (no mpCamera2), with Pinhole::epipolarConstrain (src/CameraModels/Pinhole.cpp:186-209).
//
// The reference never sets vbMatched2 (upstream omission kept, SURVEY 8a'), so queries are independent: for a KF1
// feature the result is, among the KF2 features of the same vocabulary node that pass the gates, the one with the
// smallest Hamming distance (<= TH_LOW), ties going to the LATER candidate ("dist > bestDist -> skip").  One warp
// per query: lanes stride over KF2's features (staged in shared memory), __popc Hamming, per-pair epipole and
// epipolar-line tests in non-contracted float32, shuffle arg-min on (distance, reversed index).  A second kernel
// applies the rotation histogram (factor 1/30) and ComputeThreeMaxima.
#include <algorithm>
#include <vector>

#include "extractor.h"
#include "devmath.cuh"

using namespace orb;
using namespace orbdev;

namespace orb {

struct TriParams {
    int nq, N2;
    const orbx_keypoint* kp1;
    const uint8_t* desc1;
    const int* node1;
    const uint8_t* stereo1;
    const orbx_keypoint* kp2;
    const uint8_t* desc2;
    const int* node2;
    const uint8_t* valid2;
    const uint8_t* stereo2;
    float F12[9], ep[2];
    float scale[ORB_MAX_LEVELS], sigma2[ORB_MAX_LEVELS];
    int coarse, checkOri;
    int* match;      // [nq]
    int* bins;       // [nq] rotation bin of the accepted match or -1
    int* nmatches;   // [1]
};

#define TRI_WARPS 8
#define TRI_QPB 64

__global__ void __launch_bounds__(TRI_WARPS * 32) k_tri_match(const __grid_constant__ TriParams P) {
    extern __shared__ __align__(16) unsigned char tri_smem[];
    float* s_x = reinterpret_cast<float*>(tri_smem);
    float* s_y = s_x + P.N2;
    int* s_node = reinterpret_cast<int*>(s_y + P.N2);
    uint8_t* s_oct = reinterpret_cast<uint8_t*>(s_node + P.N2);
    uint8_t* s_flag = s_oct + P.N2;   // bit0 valid (no map point [& stereo when bOnlyStereo]), bit1 stereo
    for (int i = threadIdx.x; i < P.N2; i += blockDim.x) {
        const orbx_keypoint k = P.kp2[i];
        s_x[i] = k.x; s_y[i] = k.y; s_node[i] = P.node2[i]; s_oct[i] = (uint8_t)k.octave;
        s_flag[i] = (P.valid2[i] ? 1 : 0) | (P.stereo2[i] ? 2 : 0);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int qbase = blockIdx.x * TRI_QPB;
    for (int q = qbase + warp; q < min(qbase + TRI_QPB, P.nq); q += TRI_WARPS) {
        const orbx_keypoint k1 = P.kp1[q];
        const int node = P.node1[q];
        const bool st1 = P.stereo1[q] != 0;
        const uint4* q4 = reinterpret_cast<const uint4*>(P.desc1 + 32 * (size_t)q);
        const uint4 a0 = __ldg(q4), a1 = __ldg(q4 + 1);
        // epipolar line of kp1 in image 2: (a, b, c) = (x1, y1, 1) F12
        const float la = fadd(fadd(fmul(k1.x, P.F12[0]), fmul(k1.y, P.F12[3])), P.F12[6]);
        const float lb = fadd(fadd(fmul(k1.x, P.F12[1]), fmul(k1.y, P.F12[4])), P.F12[7]);
        const float lc = fadd(fadd(fmul(k1.x, P.F12[2]), fmul(k1.y, P.F12[5])), P.F12[8]);
        const float den = fadd(fmul(la, la), fmul(lb, lb));
        uint32_t best = 0xffffffffu;   // dist << 16 | (0xffff - idx2): smaller distance wins, then the LATER index
        if (node >= 0) {
            for (int i = lane; i < P.N2; i += 32) {
                if (s_node[i] != node) continue;
                const int fl = s_flag[i];
                if (!(fl & 1)) continue;
                const uint4* d4 = reinterpret_cast<const uint4*>(P.desc2 + 32 * (size_t)i);
                const uint4 b0 = __ldg(d4), b1 = __ldg(d4 + 1);
                const uint32_t d = __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
                                   __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
                if (d > 50u) continue;   // TH_LOW
                if (!st1 && !(fl & 2)) {   // both monocular: reject points close to the epipole (ORBmatcher.cc:1189-1200)
                    const float ex = fsub(P.ep[0], s_x[i]), ey = fsub(P.ep[1], s_y[i]);
                    if (fadd(fmul(ex, ex), fmul(ey, ey)) < fmul(100.f, P.scale[s_oct[i]])) continue;
                }
                bool ok = P.coarse != 0;
                if (!ok && den != 0.f) {
                    const float num = fadd(fadd(fmul(la, s_x[i]), fmul(lb, s_y[i])), lc);
                    const float dsqr = fdiv(fmul(num, num), den);
                    ok = (double)dsqr < 3.84 * (double)P.sigma2[s_oct[i]];
                }
                if (!ok) continue;
                const uint32_t key = (d << 16) | (uint32_t)(0xffff - i);
                best = min(best, key);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (lane == 0) {
            int m = -1, bin = -1;
            if (best != 0xffffffffu) {
                m = 0xffff - (int)(best & 0xffffu);
                if (P.checkOri) {
                    float rot = fsub(k1.angle, P.kp2[m].angle);
                    if (rot < 0.0f) rot = fadd(rot, 360.0f);
                    bin = (int)roundf(fmul(rot, 1.0f / 30));
                    if (bin == 30) bin = 0;
                }
            }
            P.match[q] = m;
            P.bins[q] = bin;
        }
    }
}

__global__ void __launch_bounds__(256) k_tri_rotation(const __grid_constant__ TriParams P) {
    __shared__ int s_hist[30], s_keep[30], s_nm;
    if (threadIdx.x < 30) s_hist[threadIdx.x] = 0;
    if (threadIdx.x == 0) s_nm = 0;
    __syncthreads();
    int local = 0;
    for (int q = threadIdx.x; q < P.nq; q += blockDim.x) {
        if (P.match[q] >= 0) {
            ++local;
            if (P.checkOri) atomicAdd(&s_hist[P.bins[q]], 1);
        }
    }
    if (local) atomicAdd(&s_nm, local);
    __syncthreads();
    if (threadIdx.x == 0) {
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
        for (int q = threadIdx.x; q < P.nq; q += blockDim.x)
            if (P.match[q] >= 0 && !s_keep[min(max(P.bins[q], 0), 29)]) {
                P.match[q] = -1;
                ++removed;
            }
        if (removed) atomicSub(&s_nm, removed);
    }
    __syncthreads();
    if (threadIdx.x == 0) P.nmatches[0] = s_nm;
}

}  // namespace orb

extern "C" orb_status orbm_search_triangulation(orbx_handle* h, const orbm_triangulation* T, int32_t* match12_out,
                                                int32_t* nmatches_out) {
    if (!h || !T || !match12_out || T->n_queries < 0 || T->n2 < 0) return set_error(ORB_ERR_INVALID, "bad arguments");
    orb_status s;
    if ((s = check_frame_rows(T->n2, "keyframe")) != ORB_OK) return s;
    ORB_CUDA(cudaSetDevice(h->cfg.device));
    const int nq = T->n_queries, N2 = T->n2;
    if (nmatches_out) *nmatches_out = 0;
    if (nq == 0 || N2 == 0) {
        for (int i = 0; i < nq; ++i) match12_out[i] = -1;
        return ORB_OK;
    }
    if (!T->kp1 || !T->desc1 || !T->node1 || !T->stereo1 || !T->kp2 || !T->desc2 || !T->node2 || !T->valid2 || !T->stereo2)
        return set_error(ORB_ERR_INVALID, "missing triangulation arrays");
    TriParams P{};
    P.nq = nq; P.N2 = N2;
    for (int i = 0; i < 9; ++i) P.F12[i] = T->F12[i];
    P.ep[0] = T->epipole2[0]; P.ep[1] = T->epipole2[1];
    for (int l = 0; l < ORB_MAX_LEVELS; ++l) {
        P.scale[l] = l < h->cfg.n_levels ? h->scale[l] : 1.f;
        P.sigma2[l] = l < h->cfg.n_levels ? h->sigma2[l] : 1.f;
    }
    P.coarse = T->coarse; P.checkOri = T->check_orientation;
    const size_t smem = (size_t)N2 * 14 + 16;
    static const size_t triStatic = static_smem(k_tri_match);
    if ((s = check_smem(h, smem, triStatic, "k_tri_match")) != ORB_OK) return s;
    auto layout = [&](Carve& c) {
        P.kp1 = stage_in(c, T->kp1, nq, false); P.desc1 = stage_in(c, T->desc1, (size_t)nq * 32, false);
        P.node1 = stage_in(c, T->node1, nq, false); P.stereo1 = stage_in(c, T->stereo1, nq, false);
        P.kp2 = stage_in(c, T->kp2, N2, false); P.desc2 = stage_in(c, T->desc2, (size_t)N2 * 32, false);
        P.node2 = stage_in(c, T->node2, N2, false); P.valid2 = stage_in(c, T->valid2, N2, false); P.stereo2 = stage_in(c, T->stereo2, N2, false);
        P.match = stage_out(c, match12_out, nq, false);
        P.bins = c.take<int>(nq);
        P.nmatches = stage_out(c, nmatches_out, 1, false);
    };
    const Carve c = carve_scratch(h->stage_bytes, h->d_stage, h->capturing, h->stream, layout);
    if (c.status != ORB_OK) return c.status;
    ORB_CUDA(cudaFuncSetAttribute(k_tri_match, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max(smem, (size_t)1024)));
    k_tri_match<<<(nq + TRI_QPB - 1) / TRI_QPB, TRI_WARPS * 32, smem, h->stream>>>(P);
    ORB_LAUNCHED();
    k_tri_rotation<<<1, 256, 0, h->stream>>>(P);
    ORB_LAUNCHED();
    ORB_CUDA(cudaGetLastError());
    return copy_out(c);
}
