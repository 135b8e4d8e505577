// ORBmatcher_sim3_b200.cc -- the loop-closing / map-merging searches that project map points into a keyframe through a Sim3 pose
// (/root/reference/src/ORBmatcher.cc) on the GPU:
//   SearchByProjection(KeyFrame* pKF, Sophus::Sim3f& Scw, const vector<MapPoint*>& vpPoints, vector<MapPoint*>& vpMatched, int th, float ratioHamming)   :495-618
//   the overload with vpPointsKFs / vpMatchedKF                                                                                                        :620-732
//   Fuse(KeyFrame* pKF, Sophus::Sim3f& Scw, const vector<MapPoint*>& vpPoints, float th, vector<MapPoint*>& vpReplacePoint)                               :1546-1687
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  On the host: Tcw = SE3f(Scw.rotationMatrix(), Scw.translation() /
// Scw.scale()) and the camera centre in the caller's own Sophus, the skips (isBad(), already matched / already in the keyframe), the query
// arrays (raw mfMinDistance / mfMaxDistance through a derived class) and the side effects in query order: vpMatched[bestIdx] = pMP, or
// vpReplacePoint[iMP] = the keyframe's point / AddObservation + AddMapPoint.  Everything between is orbm_search_keyframe
// (ORBM_KF_PROJ_SIM3 / ORBM_KF_FUSE_SIM3).
#include <cstring>
#include <set>
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "orb_b200_host.h"

extern "C" orbx_handle* orb_b200_keyframe_search_handle(void);   // ORBmatcher_bow_b200.cc

namespace {
struct MapPointAccess : ORB_SLAM3::MapPoint {
    static float min_distance(const ORB_SLAM3::MapPoint& p) { return p.*(&MapPointAccess::mfMinDistance); }
    static float max_distance(const ORB_SLAM3::MapPoint& p) { return p.*(&MapPointAccess::mfMaxDistance); }
};

struct Sim3Search {
    std::vector<int> src;
    std::vector<int32_t> best;
    int32_t nmatches = 0;
};

// the part the two functions share: queries = vpPoints minus the skipped ones; one search of the keyframe's features
Sim3Search search(ORB_SLAM3::KeyFrame* pKF, Sophus::Sim3f& Scw, const std::vector<ORB_SLAM3::MapPoint*>& vpPoints, const std::set<ORB_SLAM3::MapPoint*>& skip,
                  const uint8_t* feat_claimed, int variant, float th, float hamming_max, bool checkOri, const char* who) {
    using namespace ORB_SLAM3;
    if (pKF->mpCamera2) throw orb_b200::Error(std::string(who) + ": a keyframe with a second camera is not built on the GPU path");
    orbx_handle* h = orb_b200_keyframe_search_handle();
    if (!h) throw orb_b200::Error(std::string(who) + ": no device workspace yet (orb_b200_use_handle_for_keyframe_searches)");
    const Sophus::SE3f Tcw = Sophus::SE3f(Scw.rotationMatrix(), Scw.translation() / Scw.scale());
    const Eigen::Vector3f Ow = Tcw.inverse().translation();
    Sim3Search R;
    std::vector<float> xw, nrm, maxd, mind;
    std::vector<uint8_t> qdesc;
    for (int i = 0; i < (int)vpPoints.size(); ++i) {
        MapPoint* pMP = vpPoints[i];
        if (pMP->isBad() || skip.count(pMP)) continue;
        const Eigen::Vector3f X = pMP->GetWorldPos(), n = pMP->GetNormal();
        for (int c = 0; c < 3; ++c) { xw.push_back(X(c)); nrm.push_back(n(c)); }
        maxd.push_back(MapPointAccess::max_distance(*pMP));
        mind.push_back(MapPointAccess::min_distance(*pMP));
        const cv::Mat d = pMP->GetDescriptor();
        const size_t o = qdesc.size();
        qdesc.resize(o + 32);
        std::memcpy(&qdesc[o], d.ptr<unsigned char>(), 32);
        R.src.push_back(i);
    }
    const int nq = (int)R.src.size(), N = (int)pKF->mvKeysUn.size();
    R.best.assign(nq > 0 ? nq : 1, -1);
    if (nq == 0 || N == 0) return R;
    std::vector<orbx_keypoint> kp(N);
    std::vector<uint8_t> desc((size_t)N * 32);
    for (int i = 0; i < N; ++i) {
        const cv::KeyPoint& k = pKF->mvKeysUn[i];
        kp[i].x = k.pt.x; kp[i].y = k.pt.y; kp[i].size = k.size; kp[i].angle = k.angle; kp[i].response = k.response; kp[i].octave = k.octave; kp[i].class_id = k.class_id;
        std::memcpy(&desc[(size_t)i * 32], pKF->mDescriptors.ptr<unsigned char>(i), 32);
    }
    const float T7[7] = {Tcw.unit_quaternion().x(), Tcw.unit_quaternion().y(), Tcw.unit_quaternion().z(), Tcw.unit_quaternion().w(),
                         Tcw.translation()(0), Tcw.translation()(1), Tcw.translation()(2)};
    const float O3[3] = {Ow(0), Ow(1), Ow(2)};
    const int32_t feat_offset[2] = {0, N}, query_offset[2] = {0, nq};
    orbm_kf_queries q;
    std::memset(&q, 0, sizeof(q));
    q.n_targets = 1; q.feat_offset = feat_offset; q.kp = kp.data(); q.desc = desc.data(); q.uright = pKF->mvuRight.data(); q.feat_claimed = feat_claimed;
    q.Tcw = T7; q.Ow = O3; q.query_offset = query_offset;
    q.world_pos = xw.data(); q.normal = nrm.data(); q.max_dist = maxd.data(); q.min_dist = mind.data(); q.desc_q = qdesc.data();
    orbm_camera cam;
    cam.fx = pKF->fx; cam.fy = pKF->fy; cam.cx = pKF->cx; cam.cy = pKF->cy; cam.bf = pKF->mbf; cam.b = pKF->mb;
    cam.min_x = (float)pKF->mnMinX; cam.max_x = (float)pKF->mnMaxX; cam.min_y = (float)pKF->mnMinY; cam.max_y = (float)pKF->mnMaxY;
    orb_b200::check(orbm_search_keyframe(h, &cam, &q, variant, th, hamming_max, checkOri ? 1 : 0, R.best.data(), &R.nmatches), "orbm_search_keyframe");
    return R;
}
}  // namespace

namespace ORB_SLAM3 {

// ORBmatcher.cc:495-618
int ORBmatcher::SearchByProjection(KeyFrame* pKF, Sophus::Sim3f& Scw, const std::vector<MapPoint*>& vpPoints, std::vector<MapPoint*>& vpMatched, int th,
                                   float ratioHamming) {
    std::set<MapPoint*> spAlreadyFound(vpMatched.begin(), vpMatched.end());
    spAlreadyFound.erase(static_cast<MapPoint*>(NULL));
    std::vector<uint8_t> claimed(vpMatched.size());
    for (size_t i = 0; i < vpMatched.size(); ++i) claimed[i] = vpMatched[i] ? 1 : 0;          // :589-590
    const Sim3Search R = search(pKF, Scw, vpPoints, spAlreadyFound, claimed.data(), ORBM_KF_PROJ_SIM3, (float)th, (float)TH_LOW * ratioHamming, mbCheckOrientation,
                                "ORBmatcher::SearchByProjection(pKF, Scw, vpPoints, vpMatched)");
    for (size_t k = 0; k < R.src.size(); ++k)
        if (R.best[k] >= 0) vpMatched[R.best[k]] = vpPoints[R.src[k]];                        // :609-613
    return R.nmatches;
}

// ORBmatcher.cc:620-732: the same search; the keyframe each point came from is recorded next to it
int ORBmatcher::SearchByProjection(KeyFrame* pKF, Sophus::Sim3<float>& Scw, const std::vector<MapPoint*>& vpPoints, const std::vector<KeyFrame*>& vpPointsKFs,
                                   std::vector<MapPoint*>& vpMatched, std::vector<KeyFrame*>& vpMatchedKF, int th, float ratioHamming) {
    std::set<MapPoint*> spAlreadyFound(vpMatched.begin(), vpMatched.end());
    spAlreadyFound.erase(static_cast<MapPoint*>(NULL));
    std::vector<uint8_t> claimed(vpMatched.size());
    for (size_t i = 0; i < vpMatched.size(); ++i) claimed[i] = vpMatched[i] ? 1 : 0;
    const Sim3Search R = search(pKF, Scw, vpPoints, spAlreadyFound, claimed.data(), ORBM_KF_PROJ_SIM3, (float)th, (float)TH_LOW * ratioHamming, mbCheckOrientation,
                                "ORBmatcher::SearchByProjection(pKF, Scw, vpPoints, vpPointsKFs, vpMatched, vpMatchedKF)");
    for (size_t k = 0; k < R.src.size(); ++k)
        if (R.best[k] >= 0) {                                                                 // :724-728
            vpMatched[R.best[k]] = vpPoints[R.src[k]];
            vpMatchedKF[R.best[k]] = vpPointsKFs[R.src[k]];
        }
    return R.nmatches;
}

// ORBmatcher.cc:1546-1687
int ORBmatcher::Fuse(KeyFrame* pKF, Sophus::Sim3f& Scw, const std::vector<MapPoint*>& vpPoints, float th, std::vector<MapPoint*>& vpReplacePoint) {
    const std::set<MapPoint*> spAlreadyFound = pKF->GetMapPoints();
    const Sim3Search R = search(pKF, Scw, vpPoints, spAlreadyFound, nullptr, ORBM_KF_FUSE_SIM3, th, (float)TH_LOW, mbCheckOrientation,
                                "ORBmatcher::Fuse(pKF, Scw, vpPoints)");
    int nFused = 0;
    for (size_t k = 0; k < R.src.size(); ++k) {                                              // :1662-1681, in the order of vpPoints
        if (R.best[k] < 0) continue;
        const int iMP = R.src[k];
        MapPoint* pMP = vpPoints[iMP];
        MapPoint* pMPinKF = pKF->GetMapPoint((size_t)R.best[k]);
        if (pMPinKF) {
            if (!pMPinKF->isBad()) vpReplacePoint[iMP] = pMPinKF;
        } else {
            pMP->AddObservation(pKF, R.best[k]);
            pKF->AddMapPoint(pMP, (size_t)R.best[k]);
        }
        ++nFused;
    }
    return nFused;
}

}  // namespace ORB_SLAM3
