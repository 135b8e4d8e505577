// Optimizer_pose_b200.cc -- Optimizer::PoseOptimization(Frame*) (/root/reference/src/Optimizer.cc:55-412) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/Optimizer.h (signature :48).  The tracking thread calls it after every projection
// search (Tracking.cc:3222, 3443, 3522).  What stays on the host is the walk over the frame's features under MapPoint::mGlobalMutex
// (:104-290): one edge per feature that holds a map point, in feature order, mvbOutlier cleared; and the result: mvbOutlier per
// feature, SetPose, the return value.  The four optimize(10) rounds with their chi2 classification, levels and dropped kernels are one
// kernel launch (k_pose_opt, csrc/poseopt.cu) behind orbo_pose_optimization, on the workspace of the frame's own extractor.
// A tracker that keeps the search results on the device uses orbo_pose_optimization_frames / orbr_submit instead (no host walk at all).
// Not built: two-camera rigs (Nleft != -1: EdgeSE3ProjectXYZOnlyPoseToBody, :190-287) -- such a frame is refused.
#include <mutex>
#include <vector>

#include "Optimizer.h"        // the reference's header
#include "orb_b200_host.h"

namespace ORB_SLAM3 {

int Optimizer::PoseOptimization(Frame* pFrame) {
    if (pFrame->mpCamera2 || pFrame->Nleft != -1) throw orb_b200::Error("PoseOptimization: a frame with a second camera (Nleft != -1) is not built on the GPU path");
    orbx_handle* h = orb_b200_handle_of(pFrame->mpORBextractorLeft);
    if (!h) throw orb_b200::Error("PoseOptimization: the frame's ORBextractor was not created by the GPU-path unit");
    const int N = pFrame->N;
    std::vector<float> world_pos, obs, inv_sigma2;
    std::vector<int> feature;     // vnIndexEdgeMono / vnIndexEdgeStereo, in one list (feature order)
    world_pos.reserve(3 * (size_t)N); obs.reserve(3 * (size_t)N); inv_sigma2.reserve(N); feature.reserve(N);
    {
        std::unique_lock<std::mutex> lock(MapPoint::mGlobalMutex);
        for (int i = 0; i < N; ++i) {
            MapPoint* pMP = pFrame->mvpMapPoints[i];
            if (!pMP) continue;
            pFrame->mvbOutlier[i] = false;
            const cv::KeyPoint& kpUn = pFrame->mvKeysUn[i];
            const float ur = pFrame->mvuRight[i];
            const Eigen::Vector3f X = pMP->GetWorldPos();
            world_pos.push_back(X(0)); world_pos.push_back(X(1)); world_pos.push_back(X(2));
            obs.push_back(kpUn.pt.x); obs.push_back(kpUn.pt.y); obs.push_back(ur < 0 ? -1.0f : ur);   // < 0: EdgeSE3ProjectXYZOnlyPose, else the stereo edge
            inv_sigma2.push_back(pFrame->mvInvLevelSigma2[kpUn.octave]);
            feature.push_back(i);
        }
    }
    const int nInitialCorrespondences = (int)feature.size();
    if (nInitialCorrespondences < 3) return 0;   // :292-293

    const Sophus::SE3<float> Tcw = pFrame->GetPose();
    const float pose[7] = {Tcw.unit_quaternion().x(), Tcw.unit_quaternion().y(), Tcw.unit_quaternion().z(), Tcw.unit_quaternion().w(),
                           Tcw.translation()(0), Tcw.translation()(1), Tcw.translation()(2)};
    const int32_t edge_offset[2] = {0, nInitialCorrespondences};
    orbo_pose_problems in;
    in.n_frames = 1; in.on_device = 0; in.edge_offset = edge_offset; in.pose = pose;
    in.world_pos = world_pos.data(); in.obs = obs.data(); in.inv_sigma2 = inv_sigma2.data();
    in.fx = pFrame->fx; in.fy = pFrame->fy; in.cx = pFrame->cx; in.cy = pFrame->cy; in.bf = pFrame->mbf;
    in.n_edges_max = nInitialCorrespondences;
    double pose_out[7];
    std::vector<uint8_t> outlier(nInitialCorrespondences);
    int32_t inliers = 0;
    orb_b200::check(orbo_pose_optimization(h, &in, pose_out, outlier.data(), &inliers, nullptr), "orbo_pose_optimization");

    for (int e = 0; e < nInitialCorrespondences; ++e) pFrame->mvbOutlier[feature[e]] = outlier[e] != 0;
    const Eigen::Quaterniond q(pose_out[3], pose_out[0], pose_out[1], pose_out[2]);      // SE3quat_recov (:405-410)
    const Eigen::Vector3d t(pose_out[4], pose_out[5], pose_out[6]);
    pFrame->SetPose(Sophus::SE3<float>(q.cast<float>(), t.cast<float>()));
    return inliers;   // nInitialCorrespondences - nBad
}

}  // namespace ORB_SLAM3
