// quadtree_v1.cuh -- the body of k_quadtree_v1 (DistributeOctTree, one CTA per (level, image); quadtree_core.cuh), written once for
// both sort elements: k_quadtree_v1 (32-bit element, regions up to 2048 px) and k_quadtree_v1_k64 (64-bit element, regions up to
// 4096 px), both in extractor_kernels.cuh.
#pragma once
#include "common.cuh"
#include "quadtree_core.cuh"

namespace orb {
using namespace orbdev;

template <typename E>
__device__ __forceinline__ int qt_run_v1(E* arr, void* ws, int cap, int n, int npow, const uint32_t* __restrict__ src,
                                         const QtGeom& q, uint32_t* out) {
    QT_PROF_BEGIN();
    if (npow < 256) npow = 256;     // qt_bitonic_sort_w sorts whole 256-element warp blocks (every sort buffer holds >= 2048 elements)
    for (int i = threadIdx.x; i < npow; i += blockDim.x) arr[i] = (i < n) ? qt_element<E>(src[i], q) : ~(E)0;
    __syncthreads();
    QT_TICK(q, 0)
    qt_bitonic_sort_w(arr, npow);
    QT_TICK(q, 1)
    QtWork w;
    qt_work_carve(w, ws, cap);
    return qt_distribute_v<1>(arr, n, q, w, out);
}

// The body of k_quadtree_v1 for either sort element (quadtree_core.cuh QtForm).  sortCapSmem counts elements; the global sort scratch
// of a level holds pow2_ceil(candCap) elements at sortOff (uint32 slots, 8-byte aligned for the 64-bit form).
template <typename E>
__device__ __forceinline__ void qt_v1_body(const ExtractGeom& g, int batch, int levelBegin, const uint32_t* __restrict__ cand,
                                           const int* __restrict__ candCnt, uint32_t* __restrict__ sortScratch,
                                           char* __restrict__ nodeScratch, int64_t nodeScratchStride, int sortCapSmem, int nodesInSmem,
                                           int nodeCapMax, uint32_t* __restrict__ lvlKp, int* __restrict__ lvlCnt, int* __restrict__ err) {
    extern __shared__ __align__(16) unsigned char qt_smem[];
    const int l = levelBegin + blockIdx.x / batch, img = blockIdx.x % batch;
    const LevelGeom& G = g.lv[l];
    int n = candCnt[img * g.nlevels + l];
    if (n > G.candCap) n = G.candCap;
    QtGeom q;
    q.regionW = G.maxBX - 16; q.regionH = G.maxBY - 16;
    q.nIni = G.nIni; q.hX = G.hX; q.N = G.quota;
    q.wCell = G.wCell; q.hCell = G.hCell; q.nCols = G.nCols;
#if defined(QT_PROFILE)
    q.prof_base = l == 0 ? 0 : 16;
#endif
    int npow = 2;
    while (npow < n) npow <<= 1;
    const uint32_t* src = cand + (int64_t)img * g.candTotal + G.candOff;
    uint32_t* out = lvlKp + (int64_t)img * g.kpTotal + G.kpOff;
    int cap = qt_node_cap(G.quota);
    if (cap > nodeCapMax) cap = nodeCapMax;
    E* garr = reinterpret_cast<E*>(sortScratch + (int64_t)img * g.sortTotal + G.sortOff);
    void* gws = nodeScratch + ((int64_t)l * batch + img) * nodeScratchStride;
    int S;
    if (npow <= sortCapSmem) {
        E* sarr = reinterpret_cast<E*>(qt_smem);
        if (nodesInSmem) S = qt_run_v1(sarr, qt_smem + (size_t)sortCapSmem * sizeof(E), cap, n, npow, src, q, out);
        else S = qt_run_v1(sarr, gws, cap, n, npow, src, q, out);
    } else {
        if (nodesInSmem) S = qt_run_v1(garr, qt_smem + (size_t)sortCapSmem * sizeof(E), cap, n, npow, src, q, out);
        else S = qt_run_v1(garr, gws, cap, n, npow, src, q, out);
    }
    if (threadIdx.x == 0) {
        if (S < 0 || S > G.kpCap) {
            atomicExch(&err[1], 1);
            S = 0;
        }
        lvlCnt[img * g.nlevels + l] = S;
    }
}

// the kernels' parameter list (k_quadtree_v1 and k_quadtree_v1_k64 take the same arguments as k_quadtree)
#define QT_V1_PARAMS const __grid_constant__ ExtractGeom g, int batch, int levelBegin, const uint32_t* __restrict__ cand,                   \
                     const int* __restrict__ candCnt, uint32_t* __restrict__ sortScratch, char* __restrict__ nodeScratch,                \
                     int64_t nodeScratchStride, int sortCapSmem, int nodesInSmem, int nodeCapMax, uint32_t* __restrict__ lvlKp,          \
                     int* __restrict__ lvlCnt, int* __restrict__ err
#define QT_V1_ARGS g, batch, levelBegin, cand, candCnt, sortScratch, nodeScratch, nodeScratchStride, sortCapSmem, nodesInSmem, nodeCapMax, \
                   lvlKp, lvlCnt, err

// k_quadtree_v1_k64 runs 512 threads per CTA: the 128 registers a thread may then hold keep the 64-bit sort network out of local
// memory (at 1024 threads, 64 registers, it spills).
#define QT_K64_THREADS 512

}  // namespace orb
