// ORBmatcher_fuse_b200.cc -- ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th, bRight) (/root/reference/src/ORBmatcher.cc:1325-1544)
// on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  LocalMapping::SearchInNeighbors runs it twice per neighbour for every
// new keyframe (LocalMapping.cc:703, 746).  On the host: the caller-side skips (NULL, isBad(), IsInKeyFrame), the query arrays, and the
// map mutations in query order from the best feature of every query -- Replace in the direction of the point with more observations, or
// AddObservation + AddMapPoint (:1508-1532).  Projection, the image / distance / viewing-angle gates, PredictScale, the radius search over
// the keyframe's grid, the level and stereo chi2 gates and the best Hamming distance are orbm_search_keyframe (ORBM_KF_FUSE_POSE).
// bRight (the second camera of a fisheye rig) is not built.
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "marshal.h"

namespace ORB_SLAM3 {

int ORBmatcher::Fuse(KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th, const bool bRight) {
    const char* who = "ORBmatcher::Fuse(KeyFrame*, vpMapPoints)";
    if (bRight || pKF->mpCamera2) throw orb_b200::Error(std::string(who) + ": the second camera of a rig is not built on the GPU path");
    const orb_b200::KeyFrameSearch R = orb_b200::search_keyframe(
        pKF, pKF->GetPose(), pKF->GetCameraCenter(), vpMapPoints,
        [pKF](MapPoint* pMP) { return !pMP || pMP->isBad() || pMP->IsInKeyFrame(pKF); },   // :1362-1379
        nullptr, ORBM_KF_FUSE_POSE, th, (float)TH_LOW, mbCheckOrientation, who);
    int nFused = 0;
    for (size_t k = 0; k < R.src.size(); ++k) {                               // :1508-1532, in the order of vpMapPoints
        if (R.best[k] < 0) continue;
        MapPoint* pMP = vpMapPoints[R.src[k]];
        if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;                 // a repeated pointer the loop already fused (the reference re-tests at :1368-1377)
        MapPoint* pMPinKF = pKF->GetMapPoint((size_t)R.best[k]);
        if (pMPinKF) {
            if (!pMPinKF->isBad()) {
                if (pMPinKF->Observations() > pMP->Observations()) pMP->Replace(pMPinKF);
                else pMPinKF->Replace(pMP);
            }
        } else {
            pMP->AddObservation(pKF, R.best[k]);
            pKF->AddMapPoint(pMP, (size_t)R.best[k]);
        }
        ++nFused;
    }
    return nFused;
}

}  // namespace ORB_SLAM3
