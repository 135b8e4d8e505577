// common.cuh -- shared declarations of the sm_90a hot-path library (liborbslam3_b200.so)
#pragma once
#include <utility>
#include <cstdlib>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>

#include "../../include/orbslam3_b200.h"

namespace orb {

extern thread_local std::string g_last_error;
extern std::atomic<long long> g_launches;

inline orb_status set_error(orb_status s, const std::string& msg) {
    g_last_error = msg;
    return s;
}

#define ORB_CUDA(call)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (call);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            char _b[512];                                                                           \
            snprintf(_b, sizeof(_b), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
            return orb::set_error(ORB_ERR_CUDA, _b);                                                \
        }                                                                                           \
    } while (0)

#define ORB_LAUNCHED() (++orb::g_launches)

// Launch with the device's highest stream priority (ORB_PRIO=1) -- for the latency-bound kernels of the step (one CTA per image or
// per frame: quadtree, ordering, stereo, the searches).  With several batches in flight on different streams their few CTAs then
// take the next free SM slots instead of queueing behind the hundreds of thousands of CTAs of another batch's FAST / blur launch,
// so the dependent-latency chains run under the issue-bound kernels.  The attribute is kept by stream capture (graph kernel nodes).
inline int launch_priority() {
    static const int prio = [] {
        const char* v = getenv("ORB_PRIO");
        if (!v || atoi(v) == 0) return 0;
        int least = 0, greatest = 0;
        cudaDeviceGetStreamPriorityRange(&least, &greatest);
        return greatest;
    }();
    return prio;
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_p(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributePriority;
    at[0].val.priority = launch_priority();
    cfg.attrs = at; cfg.numAttrs = launch_priority() != 0 ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

inline int device_sm_count(int device) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
    return n > 0 ? n : 1;
}

// One thread-block cluster of `cs` CTAs per problem (solvers k_lba, k_liba): one or two problems get 16 CTAs each (the non-portable
// cluster size), larger batches 8, 4 or 2 while all their clusters fit the SMs at once, then one CTA each.
inline int cluster_size_for(int n_problems, int sms) {
    if (n_problems <= 2) return 16;
    int cs = 8;
    while (cs > 1 && n_problems * cs > sms) cs >>= 1;
    return cs;
}

inline void cluster_config(cudaLaunchConfig_t& cfg, cudaLaunchAttribute& at, int grid, int cs, int threads, size_t smem, cudaStream_t st) {
    cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    at.id = cudaLaunchAttributeClusterDimension;
    at.val.clusterDim.x = cs; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
    cfg.attrs = &at; cfg.numAttrs = 1;
}

// n_problems clusters of cs CTAs; the CTAs of a problem are consecutive in x
template <typename... KArgs, typename... Args>
inline cudaError_t launch_cluster(void (*kern)(KArgs...), int n_problems, int cs, int threads, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg;
    cudaLaunchAttribute at;
    cluster_config(cfg, at, n_problems * cs, cs, threads, smem, st);
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// Halve a thread-block cluster size (*cs) until the device can co-schedule one cluster of `kern` with this block and dynamic shared
// memory: a 16-CTA (non-portable) cluster needs 16 SMs with room for the block inside one GPC, which not every H100 GPC has.  A
// failing query is returned as the error it is, never taken for "does not fit".
template <typename... KArgs>
inline cudaError_t fit_cluster_size(void (*kern)(KArgs...), int* cs, int threads, size_t smem) {
    while (*cs > 1) {
        cudaLaunchConfig_t cfg;
        cudaLaunchAttribute at;
        cluster_config(cfg, at, *cs, *cs, threads, smem, nullptr);
        int n = 0;
        const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
        if (e != cudaSuccess) return e;
        if (n > 0) break;
        *cs >>= 1;
    }
    return cudaSuccess;
}

#define ORB_MAX_LEVELS 12

// geometry of one pyramid level (level-major device layout: all images of level l are contiguous)
struct LevelGeom {
    uint8_t* base;        // level image of batch item 0 (level 0 may alias a caller's device buffer)
    uint8_t* blur;        // blurred copy (ORBextractor.cc:1629-1637)
    int64_t img_stride;   // bytes between consecutive images of this level
    int64_t blur_stride;
    int w, h, pitch, blur_pitch;
    // FAST cell grid, ORBextractor.cc:1073-1095
    int nCols, nRows, wCell, hCell, maxBX, maxBY, cellBase;
    // blur tiles
    int tilesX, tilesY, tileBase;
    // DistributeOctTree
    int quota, nIni;
    float hX;
    int candOff, candCap;   // uint32 slots inside one image's candidate block
    int kpOff, kpCap;       // uint32 slots inside one image's level-keypoint block
    int sortOff;            // uint32 slots inside one image's global sort scratch (power-of-two sized)
    // resize taps (int2 per destination column / row), tapOff = columns, tapOff + w = rows
    int tapOff;
    int area2x;             // cv::resize INTER_AREA fast path (exact 2x decimation)
    float scale;            // mvScaleFactor[level]
    float inv_scale;        // mvInvScaleFactor[level]
    float patch;            // (float)(int)(31 * scale)
};

struct ExtractGeom {
    int nlevels, totalCells, totalTiles;
    int candTotal, kpTotal, sortTotal;  // per-image block sizes (uint32 slots)
    int iniTh, minTh;
    int fastRows;                       // max over the levels of hCell + 6: rows of the FAST cell staging arrays
    LevelGeom lv[ORB_MAX_LEVELS];
};

}  // namespace orb
