// quadtree_k64.cu -- k_quadtree_v1_k64: k_quadtree_v1 (quadtree_v1.cuh) on the 64-bit, 12-depth sort element, for the level group whose
// region side exceeds 2048 px (it always holds level 0; levels of 2048 px or less never run it).  Its own library,
// liborbslam3_b200_qt64.so, linked by liborbslam3_b200.so.
#include "common.cuh"
#include "quadtree_v1.cuh"

namespace orb {

template <int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) k_quadtree_v1_k64(QT_V1_PARAMS) { qt_v1_body<uint64_t>(QT_V1_ARGS); }

cudaError_t qt_k64_set_smem(size_t bytes) {
    return cudaFuncSetAttribute(k_quadtree_v1_k64<QT_K64_THREADS, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

cudaError_t launch_quadtree_k64(int blocks, size_t smem, cudaStream_t st, const ExtractGeom& g, int batch, int levelBegin,
                                const uint32_t* cand, const int* candCnt, uint32_t* sortScratch, char* nodeScratch,
                                int64_t nodeScratchStride, int sortCapSmem, int nodesInSmem, int nodeCapMax, uint32_t* lvlKp, int* lvlCnt,
                                int* err) {
    return launch_p(k_quadtree_v1_k64<QT_K64_THREADS, 1>, dim3(blocks), dim3(QT_K64_THREADS), smem, st, g, batch, levelBegin, cand, candCnt,
                    sortScratch, nodeScratch, nodeScratchStride, sortCapSmem, nodesInSmem, nodeCapMax, lvlKp, lvlCnt, err);
}

}  // namespace orb
