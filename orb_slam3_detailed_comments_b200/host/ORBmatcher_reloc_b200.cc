// ORBmatcher_reloc_b200.cc -- ORBmatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const set<MapPoint*>& sAlreadyFound, th, ORBdist)
// (/root/reference/src/ORBmatcher.cc:2196-2330) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  Tracking::Relocalization runs it after the first PnP inliers to pick up
// the candidate keyframe's remaining map points (Tracking.cc:3758, 3773).  On the host: the queries -- the keyframe's good map points that are
// not in sAlreadyFound, in feature order, with their world position, RAW mfMinDistance / mfMaxDistance (protected members, read through
// a derived class), descriptor and the keyframe feature's angle -- and which frame features hold a map point on entry; after the call,
// CurrentFrame.mvpMapPoints[bestIdx2] = pMP for every match the rotation check kept.  The frame searched is the one its extractor produced
// last, on the device (ORBM_KF_PROJ_RELOC with a device target).  Nleft != -1 rigs are not built.
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "orb_b200_host.h"

namespace {
struct MapPointAccess : ORB_SLAM3::MapPoint {
    static float min_distance(const ORB_SLAM3::MapPoint& p) { return p.*(&MapPointAccess::mfMinDistance); }
    static float max_distance(const ORB_SLAM3::MapPoint& p) { return p.*(&MapPointAccess::mfMaxDistance); }
};
}  // namespace

namespace ORB_SLAM3 {

int ORBmatcher::SearchByProjection(Frame& CurrentFrame, KeyFrame* pKF, const std::set<MapPoint*>& sAlreadyFound, const float th, const int ORBdist) {
    const char* who = "ORBmatcher::SearchByProjection(CurrentFrame, pKF, sAlreadyFound)";
    if (CurrentFrame.Nleft != -1) throw orb_b200::Error(std::string(who) + ": Nleft != -1 (fisheye stereo rig) is not built on the GPU path");
    orbx_handle* h = orb_b200_handle_of(CurrentFrame.mpORBextractorLeft);
    if (!h) throw orb_b200::Error(std::string(who) + ": the frame's extractor is not a GPU-path extractor");
    int32_t n = 0;
    orb_b200::check(orbx_counts(h, &n, nullptr, nullptr), "orbx_counts");
    if (n != CurrentFrame.N) throw orb_b200::Error(std::string(who) + ": the frame is not the one its extractor produced last");
    const Sophus::SE3f Tcw = CurrentFrame.GetPose();
    const Eigen::Vector3f Ow = Tcw.inverse().translation();
    const std::vector<MapPoint*> vpMPs = pKF->GetMapPointMatches();
    std::vector<MapPoint*> qmp;
    std::vector<float> xw, maxd, mind, angle;
    std::vector<uint8_t> qdesc;
    for (size_t i = 0; i < vpMPs.size(); ++i) {
        MapPoint* pMP = vpMPs[i];
        if (!pMP || pMP->isBad() || sAlreadyFound.count(pMP)) continue;       // :2214-2218
        const Eigen::Vector3f X = pMP->GetWorldPos();
        for (int c = 0; c < 3; ++c) xw.push_back(X(c));
        maxd.push_back(MapPointAccess::max_distance(*pMP));
        mind.push_back(MapPointAccess::min_distance(*pMP));
        angle.push_back(pKF->mvKeysUn[i].angle);
        const cv::Mat d = pMP->GetDescriptor();
        const size_t o = qdesc.size();
        qdesc.resize(o + 32);
        std::memcpy(&qdesc[o], d.ptr<unsigned char>(), 32);
        qmp.push_back(pMP);
    }
    const int nq = (int)qmp.size();
    if (nq == 0 || CurrentFrame.N == 0) return 0;
    std::vector<uint8_t> claimed(CurrentFrame.N);
    for (int i = 0; i < CurrentFrame.N; ++i) claimed[i] = CurrentFrame.mvpMapPoints[i] ? 1 : 0;   // :2264-2265
    const float T7[7] = {Tcw.unit_quaternion().x(), Tcw.unit_quaternion().y(), Tcw.unit_quaternion().z(), Tcw.unit_quaternion().w(),
                         Tcw.translation()(0), Tcw.translation()(1), Tcw.translation()(2)};
    const float O3[3] = {Ow(0), Ow(1), Ow(2)};
    const int32_t target_image = 0, query_offset[2] = {0, nq};
    orbm_kf_queries q;
    std::memset(&q, 0, sizeof(q));
    q.n_targets = 1; q.target_image = &target_image; q.feat_claimed = claimed.data(); q.Tcw = T7; q.Ow = O3; q.query_offset = query_offset;
    q.world_pos = xw.data(); q.max_dist = maxd.data(); q.min_dist = mind.data(); q.desc_q = qdesc.data(); q.angle = angle.data();
    orbm_camera cam;
    cam.fx = Frame::fx; cam.fy = Frame::fy; cam.cx = Frame::cx; cam.cy = Frame::cy; cam.bf = CurrentFrame.mbf; cam.b = CurrentFrame.mb;
    cam.min_x = Frame::mnMinX; cam.max_x = Frame::mnMaxX; cam.min_y = Frame::mnMinY; cam.max_y = Frame::mnMaxY;
    std::vector<int32_t> best(nq, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_keyframe(h, &cam, &q, ORBM_KF_PROJ_RELOC, th, (float)ORBdist, mbCheckOrientation ? 1 : 0, best.data(), &nmatches),
                    "orbm_search_keyframe");
    for (int k = 0; k < nq; ++k)
        if (best[k] >= 0) CurrentFrame.mvpMapPoints[best[k]] = qmp[k];      // :2285 (the rotation check's removals, :2309-2326, are already applied)
    return nmatches;
}

}  // namespace ORB_SLAM3
