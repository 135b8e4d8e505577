// scratch.h -- per-call device scratch: one carver, one growth policy, one host-to-device staging helper (host code only)
//
// An entry point describes its scratch block once, as a `layout` function of a Carve that assigns every device pointer.
// carve_scratch runs it with a null base to measure, grows the buffer to fit and runs it again on the buffer, so the size
// always matches what the layout takes.
//
// Some calls nest, so a call never carves the arena its caller carves.  Which entry points use which buffer:
//
// | Buffer | Entry points |
// |---|---|
// | `h->d_stage` | every matcher.cu entry point, `orbm_search_triangulation`, `orbo_pose_optimization`, `orbo_pose_edges` (its count array) |
// | `h->d_po` | `orbo_pose_optimization_frames` (it calls the two above), `orbv_transform`, `orbp_distinctive_descriptors`, `orbp_update_normal_and_depth`, `orbm_hamming_knn2` |
// | `orbr_state::d_buf` | `orbr_submit` (it calls the searches and pose calls above) |
// | `h->d_xl` | the frame blocks of the matcher searches' global-memory form (matcher.cu `launch_proj`) |
//
// Captured CUDA graphs hold pointers into these buffers, so a buffer only grows in an eager call: growth inside a capture is refused.
//
// The two bundle-adjustment solvers (`lba_solve*`, `liba_solve`) are not carved: each lays a batch out in its handle's `d_buf` with
// a pinned mirror in `h_buf` (pack.h), both grown by the functions below.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace orb {

struct Carve {
    uint8_t* base;               // nullptr: measure only
    cudaStream_t stream = nullptr;
    size_t off = 0;
    orb_status status = ORB_OK;  // first failed copy of stage_in
    // 256-byte aligned; at least one element, so no two arrays share an address
    template <typename T>
    T* take(size_t n) {
        off = (off + 255) / 256 * 256;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += std::max<size_t>(n, 1) * sizeof(T);
        return p;
    }
};

// Device callers get their own pointer back; host arrays get a slot in the block and are copied there on the carve's stream.
template <typename T>
T* stage_in(Carve& c, const T* src, size_t n, bool on_device) {
    if (!src) return nullptr;
    if (on_device) return const_cast<T*>(src);
    T* dst = c.take<T>(n);
    if (dst && n && c.status == ORB_OK) {
        const cudaError_t e = cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, c.stream);
        if (e != cudaSuccess) c.status = set_error(ORB_ERR_CUDA, std::string("stage_in: cudaMemcpyAsync -> ") + cudaGetErrorString(e));
    }
    return dst;
}

// Grow only, never shrink.  A quarter of headroom keeps calls whose sizes vary a little from reallocating every time.
inline size_t scratch_alloc_bytes(size_t need) {
    const size_t MiB = (size_t)1 << 20;
    return (need + need / 4 + MiB - 1) / MiB * MiB;
}

inline orb_status grow_device(size_t& bytes, uint8_t*& ptr, size_t need, bool capturing) {
    if (need <= bytes) return ORB_OK;
    if (capturing) return set_error(ORB_ERR_INVALID, "scratch must be sized by one eager call with the same bounds before a graph capture");
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    bytes = 0;
    const size_t want = scratch_alloc_bytes(need);
    ORB_CUDA(cudaMalloc((void**)&ptr, want));
    bytes = want;
    return ORB_OK;
}

inline orb_status grow_pinned(size_t& bytes, uint8_t*& ptr, size_t need) {
    if (need <= bytes) return ORB_OK;
    if (ptr) cudaFreeHost(ptr);
    ptr = nullptr;
    bytes = 0;
    const size_t want = scratch_alloc_bytes(need);
    ORB_CUDA(cudaMallocHost((void**)&ptr, want));
    bytes = want;
    return ORB_OK;
}

// What a solver handle (lba_handle, liba_handle) holds besides its own state.
struct SolverHandle {
    int device = 0;
    cudaStream_t stream = nullptr;
    uint8_t* d_buf = nullptr;   // device block of a batch
    size_t d_bytes = 0;
    uint8_t* h_buf = nullptr;   // its pinned mirror
    size_t h_bytes = 0;
    int n_sms = 1;
};

// Creates *out on `device` with its own stream; `kern` may then be launched in clusters of up to 16 CTAs and with up to
// `max_smem` bytes of dynamic shared memory (0: the default limit).
template <typename H, typename... KArgs>
orb_status solver_create(int32_t device, void (*kern)(KArgs...), size_t max_smem, H** out) {
    if (!out) return set_error(ORB_ERR_INVALID, "null argument");
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev)
        return set_error(ORB_ERR_NO_DEVICE, "no usable CUDA device (this library has no CPU fallback)");
    ORB_CUDA(cudaSetDevice(device));
    ORB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    if (max_smem) ORB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)max_smem));
    H* h = new H();
    h->device = device;
    h->n_sms = device_sm_count(device);
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete h;
        return set_error(ORB_ERR_CUDA, "cudaStreamCreate failed");
    }
    *out = h;
    return ORB_OK;
}

// Waits for the handle's work and frees what solver_create and the solves allocated; the caller frees its own state, then deletes.
inline void solver_release(SolverHandle* h) {
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    if (h->d_buf) cudaFree(h->d_buf);
    if (h->h_buf) cudaFreeHost(h->h_buf);
    if (h->stream) cudaStreamDestroy(h->stream);
}

// measure `layout`, grow the buffer to fit, carve it: returns the first error of the growth or of a stage_in copy
template <typename F>
orb_status carve_scratch(size_t& bytes, uint8_t*& ptr, bool capturing, cudaStream_t stream, F&& layout) {
    Carve m{nullptr, stream};
    layout(m);
    const orb_status s = grow_device(bytes, ptr, m.off, capturing);
    if (s != ORB_OK) return s;
    Carve c{ptr, stream};
    layout(c);
    return c.status;
}

}  // namespace orb
