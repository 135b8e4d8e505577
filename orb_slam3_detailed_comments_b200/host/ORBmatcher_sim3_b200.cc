// ORBmatcher_sim3_b200.cc -- the loop-closing / map-merging searches that project map points into a keyframe through a Sim3 pose
// (/root/reference/src/ORBmatcher.cc) on the GPU:
//   SearchByProjection(KeyFrame* pKF, Sophus::Sim3f& Scw, const vector<MapPoint*>& vpPoints, vector<MapPoint*>& vpMatched, int th, float ratioHamming)   :495-618
//   the overload with vpPointsKFs / vpMatchedKF                                                                                                        :620-732
//   Fuse(KeyFrame* pKF, Sophus::Sim3f& Scw, const vector<MapPoint*>& vpPoints, float th, vector<MapPoint*>& vpReplacePoint)                               :1546-1687
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  On the host: Tcw = SE3f(Scw.rotationMatrix(), Scw.translation() /
// Scw.scale()) and the camera centre in the caller's own Sophus, the skips (isBad(), already matched / already in the keyframe), the query
// arrays and the side effects in query order: vpMatched[bestIdx] = pMP, or vpReplacePoint[iMP] = the keyframe's point / AddObservation +
// AddMapPoint.  Everything between is orbm_search_keyframe (ORBM_KF_PROJ_SIM3 / ORBM_KF_FUSE_SIM3).
#include <set>
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "marshal.h"

namespace {
// the part the three members share: Tcw and the camera centre from Scw, queries = vpPoints minus the bad and the skipped ones, one search of
// the keyframe's features
orb_b200::KeyFrameSearch search(ORB_SLAM3::KeyFrame* pKF, Sophus::Sim3f& Scw, const std::vector<ORB_SLAM3::MapPoint*>& vpPoints,
                                const std::set<ORB_SLAM3::MapPoint*>& skip, const uint8_t* feat_claimed, int variant, float th, float hamming_max,
                                bool checkOri, const char* who) {
    if (pKF->mpCamera2) throw orb_b200::Error(std::string(who) + ": a keyframe with a second camera is not built on the GPU path");
    const Sophus::SE3f Tcw = Sophus::SE3f(Scw.rotationMatrix(), Scw.translation() / Scw.scale());
    return orb_b200::search_keyframe(pKF, Tcw, Tcw.inverse().translation(), vpPoints,
                                     [&skip](ORB_SLAM3::MapPoint* pMP) { return pMP->isBad() || skip.count(pMP); }, feat_claimed, variant, th,
                                     hamming_max, checkOri, who);
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
    const orb_b200::KeyFrameSearch R = search(pKF, Scw, vpPoints, spAlreadyFound, claimed.data(), ORBM_KF_PROJ_SIM3, (float)th, (float)TH_LOW * ratioHamming, mbCheckOrientation,
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
    const orb_b200::KeyFrameSearch R = search(pKF, Scw, vpPoints, spAlreadyFound, claimed.data(), ORBM_KF_PROJ_SIM3, (float)th, (float)TH_LOW * ratioHamming, mbCheckOrientation,
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
    const orb_b200::KeyFrameSearch R = search(pKF, Scw, vpPoints, spAlreadyFound, nullptr, ORBM_KF_FUSE_SIM3, th, (float)TH_LOW, mbCheckOrientation,
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
