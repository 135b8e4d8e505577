// rgbd.cu -- k_stereo_rgbd, Frame::ComputeStereoFromRGBD of a batch of RGB-D frames, in a shared object of its own
// (lib/liborbslam3_b200_rgbd.so).  liborbslam3_b200.so opens it on the first RGB-D batch (extractor.cu side_symbol), so the main
// library's kernels stay exactly the GPU-validated set that tests/golden/sass_fingerprints.json pins; this one is pinned by
// tests/golden/rgbd_sass_fingerprint.json.  Other sensors never load it.
#include <cuda_runtime.h>

#include "rgbd_core.cuh"

namespace orb {

// One thread per keypoint row of each image (rgbd_core.cuh rgbd_row); blockIdx.y is the image.  Only the sampled depth pixels are
// read and converted.
__global__ void __launch_bounds__(128) k_stereo_rgbd(const __grid_constant__ orbdev::RgbdPlan P) {
    const int img = blockIdx.y, i = blockIdx.x * 128 + threadIdx.x;
    if (i >= P.nkp[img]) return;
    const int row = P.offsets[img] + i;
    const float x = P.kps[row].x, y = P.kps[row].y;
    float u, d;
    orbdev::rgbd_row(P.depth + (int64_t)img * P.image_stride, P.stride, P.format, P.scaled != 0, P.factor, x, y, P.bf, &u, &d);
    P.uright[row] = u;
    P.depth_out[row] = d;
}

}  // namespace orb

// Queues k_stereo_rgbd for `n_images` images of at most `rows_per_image` keypoints on `stream` (a stream of `device`; no synchronisation,
// so it can be captured): returns the launch's error.  The context is the device's primary context, which the caller's runtime uses too.
extern "C" cudaError_t orb_rgbd_launch(const orbdev::RgbdPlan* P, int32_t n_images, int32_t rows_per_image, int32_t device, cudaStream_t stream) {
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return e;
    orb::k_stereo_rgbd<<<dim3((rows_per_image + 127) / 128, n_images), 128, 0, stream>>>(*P);
    return cudaGetLastError();
}
