// ORBmatcher_reloc_b200.cc -- ORBmatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const set<MapPoint*>& sAlreadyFound, th, ORBdist)
// (/root/reference/src/ORBmatcher.cc:2196-2330) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  Tracking::Relocalization runs it after the first PnP inliers to pick up
// the candidate keyframe's remaining map points (Tracking.cc:3758, 3773).  On the host: the queries -- the keyframe's good map points that are
// not in sAlreadyFound, in feature order, with their world position, raw mfMinDistance / mfMaxDistance, descriptor and the keyframe
// feature's angle -- and which frame features hold a map point on entry; after the call, CurrentFrame.mvpMapPoints[bestIdx2] = pMP for
// every match the rotation check kept.  The frame searched is the one its extractor produced last, on the device (ORBM_KF_PROJ_RELOC with a
// device target).  Nleft != -1 rigs are not built.
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "marshal.h"

namespace ORB_SLAM3 {

int ORBmatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th, const int ORBdist) {
    const char* who = "ORBmatcher::SearchByProjection(CurrentFrame, pKF, sAlreadyFound)";
    orbx_handle* h = orb_b200::resident_frame(CurrentFrame, who);
    const Sophus::SE3f Tcw = CurrentFrame.GetPose();
    const Eigen::Vector3f Ow = Tcw.inverse().translation();
    const std::vector<MapPoint*> vpMPs = pKF->GetMapPointMatches();
    std::vector<MapPoint*> qmp;
    orb_b200::PointQueries<MapPoint> Q(false);
    std::vector<float> angle;
    for (size_t i = 0; i < vpMPs.size(); ++i) {
        MapPoint* pMP = vpMPs[i];
        if (!pMP || pMP->isBad() || sAlreadyFound.count(pMP)) continue;       // :2214-2218
        Q.push(pMP);
        angle.push_back(pKF->mvKeysUn[i].angle);
        qmp.push_back(pMP);
    }
    const int nq = (int)qmp.size();
    if (nq == 0 || CurrentFrame.N == 0) return 0;
    std::vector<uint8_t> claimed(CurrentFrame.N);
    for (int i = 0; i < CurrentFrame.N; ++i) claimed[i] = CurrentFrame.mvpMapPoints[i] ? 1 : 0;   // :2264-2265
    const std::array<float, 7> T7 = orb_b200::pose7(Tcw);
    const float O3[3] = {Ow(0), Ow(1), Ow(2)};
    const int32_t target_image = 0, query_offset[2] = {0, nq};
    orbm_kf_queries q;
    std::memset(&q, 0, sizeof(q));
    q.n_targets = 1; q.target_image = &target_image; q.feat_claimed = claimed.data(); q.Tcw = T7.data(); q.Ow = O3; q.query_offset = query_offset;
    Q.fill(q);
    q.angle = angle.data();
    const orbm_camera cam = orb_b200::camera_of(CurrentFrame);
    std::vector<int32_t> best(nq, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_keyframe(h, &cam, &q, ORBM_KF_PROJ_RELOC, th, (float)ORBdist, mbCheckOrientation ? 1 : 0, best.data(), &nmatches),
                    "orbm_search_keyframe");
    for (int k = 0; k < nq; ++k)
        if (best[k] >= 0) CurrentFrame.mvpMapPoints[best[k]] = qmp[k];      // :2285 (the rotation check's removals, :2309-2326, are already applied)
    return nmatches;
}

}  // namespace ORB_SLAM3
