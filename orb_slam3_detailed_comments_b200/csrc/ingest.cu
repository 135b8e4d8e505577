// ingest.cu -- k_ingest, the camera-image stage in front of the extractor, in a shared object of its own
// (lib/liborbslam3_b200_ingest.so).  liborbslam3_b200.so opens it on the first colour or resized batch (extractor.cu
// ingest_launcher), so the main library's kernels stay exactly the GPU-validated set that tests/golden/sass_fingerprints.json
// pins; this one is pinned by tests/golden/ingest_sass_fingerprint.json.  Grey batches of the extracted size never load it.
#include <cuda_runtime.h>

#include "resize_core.cuh"

namespace orb {

// colour conversion and resize of a batch of camera images into level 0 (resize_core.cuh ig_pixels4).  256 threads cover 1024 px x
// 1 row; blockIdx.z is the image.
__global__ void __launch_bounds__(256) k_ingest(const __grid_constant__ orbdev::IngestPlan P) {
    const int dx4 = 4 * (blockIdx.x * 256 + threadIdx.x), dy = blockIdx.y;
    if (dx4 >= P.dw) return;
    const uint32_t v = orbdev::ig_pixels4(P, P.src + (int64_t)blockIdx.z * P.src_image, dx4, dy);
    *reinterpret_cast<uint32_t*>(P.dst + (int64_t)blockIdx.z * P.dst_image + (int64_t)dy * P.dpitch + dx4) = v;
}

}  // namespace orb

// Queues k_ingest for `batch` images on `stream` (a stream of `device`; no synchronisation, so it can be captured): returns the launch's
// error.  This object carries its own CUDA runtime; the context is the device's primary context, which the caller's runtime uses too.
extern "C" cudaError_t orb_ingest_launch(const orbdev::IngestPlan* P, int32_t batch, int32_t device, cudaStream_t stream) {
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return e;
    orb::k_ingest<<<dim3((P->dw + 1023) / 1024, P->dh, batch), 256, 0, stream>>>(*P);
    return cudaGetLastError();
}
