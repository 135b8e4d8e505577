// rgbd_core.cuh -- one keypoint of Frame::ComputeStereoFromRGBD over a raw depth map, with Tracking::GrabImageRGBD's conversion of the
// sampled pixel only.  The identical source runs as k_stereo_rgbd's per-thread body (csrc/stereo.cu) and on the host
// (tests/host_emul/rgbd_emul.cpp, against a numpy restatement and the oracle).
#pragma once
#include "../../include/orbslam3_b200.h"
#include "devmath.cuh"

namespace orbdev {

// Tracking::GrabImageRGBD: `if (fabs(mDepthMapFactor - 1.0f) > 1e-5 || imDepth.type() != CV_32F) imDepth.convertTo(imDepth, CV_32F,
// mDepthMapFactor)`.  The float difference is compared in double, as the reference's expression promotes it.
ORB_HD bool rgbd_scaled(int format, float factor) {
    const float diff = fsub(factor, 1.0f);
    return format != ORB_DEPTH_F32 || (double)(diff < 0.0f ? -diff : diff) > 1e-5;
}

// A camera with zero distortion: mvKeysUn = mvKeys.  d = imDepth.at<float>(v, u) with u, v the keypoint truncated to int; convertTo's
// 16U -> 32F or 32F -> 32F scaling with a zero offset is one rounded product.  d > 0 (false for NaN): mvDepth = d, mvuRight = x - bf / d.
ORB_HD void rgbd_row(const uint8_t* map, int64_t stride, int format, bool scaled, float factor, float x, float y, float bf, float* uright,
                     float* depth) {
    const uint8_t* row = map + (int64_t)(int)y * stride;
    const int u = (int)x;
    float d = format == ORB_DEPTH_U16 ? (float)reinterpret_cast<const uint16_t*>(row)[u] : reinterpret_cast<const float*>(row)[u];
    if (scaled) d = fmul(d, factor);
    if (d > 0.0f) {
        *depth = d;
        *uright = fsub(x, fdiv(bf, d));
    } else {
        *depth = -1.0f;
        *uright = -1.0f;
    }
}

// k_stereo_rgbd's arguments: the depth maps of a batch and the compact keypoint rows of the extractor handle
struct RgbdPlan {
    const uint8_t* depth;        // map of image b at depth + b * image_stride
    int64_t image_stride, stride;
    int format, scaled;
    float factor, bf;
    const orbx_keypoint* kps;    // compact rows; image b's are [offsets[b], offsets[b] + nkp[b])
    const int* offsets;
    const int* nkp;
    float* uright;               // row-aligned with kps
    float* depth_out;
};

}  // namespace orbdev
