// oracle/rgbd_oracle.cpp -- TEST INFRASTRUCTURE (see oracle.h).
// CPU restatement of Tracking::GrabImageRGBD's depth conversion and Frame::ComputeStereoFromRGBD for a camera with zero distortion
// (mvKeysUn = mvKeys).  The whole map is converted first, as the reference does: `if (fabs(mDepthMapFactor - 1.0f) > 1e-5 ||
// imDepth.type() != CV_32F) imDepth.convertTo(imDepth, CV_32F, mDepthMapFactor)`; then every keypoint samples imDepth.at<float>(v, u)
// with v, u truncated to int.
#include <cmath>
#include <cstdint>
#include <vector>

#include "oracle.h"

using orb_oracle::KeyPoint;

// format 1: uint16 map, 2: float map; stride in bytes.  Writes mvuRight / mvDepth of the N keypoints (-1 where d <= 0 or NaN).
extern "C" void orc_stereo_from_rgbd(const KeyPoint* kps, int N, const void* map, int format, long long stride, int W, int H, float factor,
                                     float mbf, float* uRight, float* depth) {
    const bool is_f32 = format == 2;
    const bool convert = std::fabs(factor - 1.0f) > 1e-5 || !is_f32;
    std::vector<float> im((size_t)W * H);
    for (int v = 0; v < H; ++v) {
        const uint8_t* row = (const uint8_t*)map + (size_t)v * stride;
        for (int u = 0; u < W; ++u) {
            const float raw = is_f32 ? ((const float*)row)[u] : (float)((const uint16_t*)row)[u];
            im[(size_t)v * W + u] = convert ? raw * factor : raw;
        }
    }
    for (int i = 0; i < N; ++i) {
        uRight[i] = depth[i] = -1.0f;
        const int u = (int)kps[i].x, v = (int)kps[i].y;
        const float d = im[(size_t)v * W + u];
        if (d > 0) {
            depth[i] = d;
            uRight[i] = kps[i].x - mbf / d;
        }
    }
}
