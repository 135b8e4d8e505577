// tests/host/pose_stub.cc -- TEST INFRASTRUCTURE (CPU tier): orbo_pose_optimization over the oracle (orc_pose_optimization) instead of the
// GPU, so that host/Optimizer_pose_b200.cc -- the feature walk, mvbOutlier, SetPose, the return value -- can run without a GPU next to the
// reference's own function (oracle/_ref part 5; tests/test_host_pose_vs_ref.py).  Never linked into the product.
#include <cstdint>
#include <vector>

#include "orbslam3_b200.h"

extern "C" int orc_pose_optimization(int n, const double* Xw, const double* obs, const double* invs2, const double* cam5, double* pose7, uint8_t* outlier,
                                     double* stats);

extern "C" {
const char* orb_last_error(void) { return "pose_stub"; }
orbx_handle* orb_b200_handle_of(const void*) { static int dummy; return reinterpret_cast<orbx_handle*>(&dummy); }

orb_status orbo_pose_optimization(orbx_handle*, const orbo_pose_problems* in, double* pose_out, uint8_t* outlier_out, int32_t* inliers_out, int32_t* stats_out) {
    if (in->on_device) return ORB_ERR_INVALID;
    const double cam5[5] = {in->fx, in->fy, in->cx, in->cy, in->bf};
    for (int f = 0; f < in->n_frames; ++f) {
        const int e0 = in->edge_offset[f], n = in->edge_offset[f + 1] - e0;
        std::vector<double> Xw(3 * (size_t)n + 3), obs(3 * (size_t)n + 3), w(n + 1);
        for (int i = 0; i < 3 * n; ++i) { Xw[i] = in->world_pos[3 * (size_t)e0 + i]; obs[i] = in->obs[3 * (size_t)e0 + i]; }
        for (int i = 0; i < n; ++i) w[i] = in->inv_sigma2[e0 + i];
        double pose[7], stats[4];
        for (int i = 0; i < 7; ++i) pose[i] = in->pose[7 * f + i];
        std::vector<uint8_t> out(n + 1);
        inliers_out[f] = orc_pose_optimization(n, Xw.data(), obs.data(), w.data(), cam5, pose, out.data(), stats);
        for (int i = 0; i < 7; ++i) pose_out[7 * f + i] = pose[i];
        for (int i = 0; i < n; ++i) outlier_out[e0 + i] = out[i];
        if (stats_out) for (int i = 0; i < 4; ++i) stats_out[4 * f + i] = (int32_t)stats[i];
    }
    return ORB_OK;
}
}
