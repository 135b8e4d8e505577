// k_stereo_rgbd's per-thread body (csrc/rgbd_core.cuh rgbd_row) and GrabImageRGBD's factor rule compiled for the host:
// tests/test_rgbd_cpu.py runs them against a numpy restatement and the oracle.
#include <cstdint>

#include "../../orb_slam3_detailed_comments_b200/csrc/rgbd_core.cuh"

extern "C" int emul_rgbd_scaled(int format, float factor) { return orbdev::rgbd_scaled(format, factor) ? 1 : 0; }

// n keypoints at (xy[2i], xy[2i + 1]) over one map
extern "C" void emul_rgbd(const float* xy, int n, const uint8_t* map, int format, long long stride, float factor, float bf, float* uright,
                          float* depth) {
    const bool scaled = orbdev::rgbd_scaled(format, factor);
    for (int i = 0; i < n; ++i) orbdev::rgbd_row(map, stride, format, scaled, factor, xy[2 * i], xy[2 * i + 1], bf, &uright[i], &depth[i]);
}
