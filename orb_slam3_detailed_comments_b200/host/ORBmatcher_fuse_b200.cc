// ORBmatcher_fuse_b200.cc -- ORBmatcher::Fuse(KeyFrame*, const vector<MapPoint*>&, th, bRight) (/root/reference/src/ORBmatcher.cc:1325-1544)
// on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  LocalMapping::SearchInNeighbors runs it twice per neighbour for every
// new keyframe (LocalMapping.cc:703, 746).  On the host: the caller-side skips (NULL, isBad(), IsInKeyFrame), the query arrays, and the
// map mutations in query order from the best feature of every query -- Replace in the direction of the point with more observations, or
// AddObservation + AddMapPoint (:1508-1532).  Projection, the image / distance / viewing-angle gates, PredictScale, the radius search over
// the keyframe's grid, the level and stereo chi2 gates and the best Hamming distance are orbm_search_keyframe (ORBM_KF_FUSE_POSE).
// The search needs MapPoint's RAW mfMinDistance / mfMaxDistance (the gate applies 0.8f / 1.2f itself, PredictScale divides the raw value):
// they are protected members, read through a derived class (no change to the reference's header), without mMutexPos -- like every
// member this function reads from the mapping thread that owns it.  bRight (the second camera of a fisheye rig) is not built.
#include <cstring>
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
}  // namespace

namespace ORB_SLAM3 {

int ORBmatcher::Fuse(KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPoints, const float th, const bool bRight) {
    const char* who = "ORBmatcher::Fuse(KeyFrame*, vpMapPoints)";
    if (bRight || pKF->mpCamera2) throw orb_b200::Error(std::string(who) + ": the second camera of a rig is not built on the GPU path");
    orbx_handle* h = orb_b200_keyframe_search_handle();
    if (!h) throw orb_b200::Error(std::string(who) + ": no device workspace yet (orb_b200_use_handle_for_keyframe_searches)");
    const int nMPs = (int)vpMapPoints.size();
    std::vector<int> src;
    std::vector<float> xw, nrm, maxd, mind;
    std::vector<uint8_t> qdesc;
    for (int i = 0; i < nMPs; ++i) {
        MapPoint* pMP = vpMapPoints[i];
        if (!pMP || pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;         // :1362-1379
        const Eigen::Vector3f X = pMP->GetWorldPos(), n = pMP->GetNormal();
        for (int c = 0; c < 3; ++c) { xw.push_back(X(c)); nrm.push_back(n(c)); }
        maxd.push_back(MapPointAccess::max_distance(*pMP));
        mind.push_back(MapPointAccess::min_distance(*pMP));
        const cv::Mat d = pMP->GetDescriptor();
        const size_t o = qdesc.size();
        qdesc.resize(o + 32);
        std::memcpy(&qdesc[o], d.ptr<unsigned char>(), 32);
        src.push_back(i);
    }
    const int nq = (int)src.size(), N = (int)pKF->mvKeysUn.size();
    if (nq == 0 || N == 0) return 0;
    std::vector<orbx_keypoint> kp(N);
    std::vector<uint8_t> desc((size_t)N * 32);
    for (int i = 0; i < N; ++i) {
        const cv::KeyPoint& k = pKF->mvKeysUn[i];
        kp[i].x = k.pt.x; kp[i].y = k.pt.y; kp[i].size = k.size; kp[i].angle = k.angle; kp[i].response = k.response; kp[i].octave = k.octave; kp[i].class_id = k.class_id;
        std::memcpy(&desc[(size_t)i * 32], pKF->mDescriptors.ptr<unsigned char>(i), 32);
    }
    const Sophus::SE3f Tcw = pKF->GetPose();
    const Eigen::Vector3f Ow = pKF->GetCameraCenter();
    const float T7[7] = {Tcw.unit_quaternion().x(), Tcw.unit_quaternion().y(), Tcw.unit_quaternion().z(), Tcw.unit_quaternion().w(),
                         Tcw.translation()(0), Tcw.translation()(1), Tcw.translation()(2)};
    const float O3[3] = {Ow(0), Ow(1), Ow(2)};
    const int32_t feat_offset[2] = {0, N}, query_offset[2] = {0, nq};
    orbm_kf_queries q;
    std::memset(&q, 0, sizeof(q));
    q.n_targets = 1; q.feat_offset = feat_offset; q.kp = kp.data(); q.desc = desc.data(); q.uright = pKF->mvuRight.data();
    q.Tcw = T7; q.Ow = O3; q.query_offset = query_offset;
    q.world_pos = xw.data(); q.normal = nrm.data(); q.max_dist = maxd.data(); q.min_dist = mind.data(); q.desc_q = qdesc.data();
    orbm_camera cam;
    cam.fx = pKF->fx; cam.fy = pKF->fy; cam.cx = pKF->cx; cam.cy = pKF->cy; cam.bf = pKF->mbf; cam.b = pKF->mb;
    cam.min_x = (float)pKF->mnMinX; cam.max_x = (float)pKF->mnMaxX; cam.min_y = (float)pKF->mnMinY; cam.max_y = (float)pKF->mnMaxY;
    std::vector<int32_t> best(nq, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_keyframe(h, &cam, &q, ORBM_KF_FUSE_POSE, th, (float)TH_LOW, mbCheckOrientation ? 1 : 0, best.data(), &nmatches),
                    "orbm_search_keyframe");
    int nFused = 0;
    for (int k = 0; k < nq; ++k) {                                            // :1508-1532, in the order of vpMapPoints
        if (best[k] < 0) continue;
        MapPoint* pMP = vpMapPoints[src[k]];
        if (pMP->isBad() || pMP->IsInKeyFrame(pKF)) continue;                 // a repeated pointer the loop already fused (the reference re-tests at :1368-1377)
        MapPoint* pMPinKF = pKF->GetMapPoint((size_t)best[k]);
        if (pMPinKF) {
            if (!pMPinKF->isBad()) {
                if (pMPinKF->Observations() > pMP->Observations()) pMP->Replace(pMPinKF);
                else pMPinKF->Replace(pMP);
            }
        } else {
            pMP->AddObservation(pKF, best[k]);
            pKF->AddMapPoint(pMP, (size_t)best[k]);
        }
        ++nFused;
    }
    return nFused;
}

}  // namespace ORB_SLAM3
