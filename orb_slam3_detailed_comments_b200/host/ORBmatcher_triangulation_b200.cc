// ORBmatcher_triangulation_b200.cc -- ORBmatcher::SearchForTriangulation (/root/reference/src/ORBmatcher.cc:1045-1323) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  LocalMapping::CreateNewMapPoints runs it for every new keyframe
// against its best covisible neighbours (LocalMapping.cc:379).  On the host: the relative pose, the epipole and the fundamental matrix in
// the caller's own Sophus / Eigen float arithmetic (:1052-1073 and Pinhole::epipolarConstrain's F12, Pinhole.cpp:191-194, which the
// reference recomputes for every candidate pair), the FeatureVector merge order of keyframe 1's features without a map point, the
// vocabulary node / validity / stereo flags of keyframe 2's features, and the pair list in ascending idx1.  The search itself -- per-node
// candidates, Hamming gate, epipole gate, epipolar-line gate at the candidate's level, vbMatched2 claims, rotation histogram -- is
// orbm_search_triangulation.  Keyframes with a second camera (fisheye rigs) are not built.
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "orb_b200_host.h"

extern "C" void orb_b200_use_handle_for_keyframe_searches(orbx_handle* h);   // ORBmatcher_bow_b200.cc
extern "C" orbx_handle* orb_b200_keyframe_search_handle(void);

namespace ORB_SLAM3 {

namespace {
void put_keypoint(orbx_keypoint& o, const cv::KeyPoint& k) {
    o.x = k.pt.x; o.y = k.pt.y; o.size = k.size; o.angle = k.angle; o.response = k.response; o.octave = k.octave; o.class_id = k.class_id;
}
}  // namespace

int ORBmatcher::SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<std::pair<size_t, size_t> >& vMatchedPairs, const bool bOnlyStereo,
                                       const bool bCoarse) {
    const char* who = "ORBmatcher::SearchForTriangulation";
    if (pKF1->mpCamera2 || pKF2->mpCamera2) throw orb_b200::Error(std::string(who) + ": a keyframe with a second camera is not built on the GPU path");
    orbx_handle* h = orb_b200_keyframe_search_handle();
    if (!h) throw orb_b200::Error(std::string(who) + ": no device workspace yet (orb_b200_use_handle_for_keyframe_searches)");

    // :1052-1073, Pinhole.cpp:119-130 (project) and :191-194 (F12)
    const Sophus::SE3f T1w = pKF1->GetPose(), T2w = pKF2->GetPose(), Tw2 = pKF2->GetPoseInverse();
    const Eigen::Vector3f Cw = pKF1->GetCameraCenter();
    const Eigen::Vector3f C2 = T2w * Cw;
    const float epx = pKF2->fx * C2(0) / C2(2) + pKF2->cx, epy = pKF2->fy * C2(1) / C2(2) + pKF2->cy;
    const Sophus::SE3f T12 = T1w * Tw2;
    const Eigen::Matrix3f R12 = T12.rotationMatrix();
    const Eigen::Vector3f t12 = T12.translation();
    const Eigen::Matrix3f t12x = Sophus::SO3f::hat(t12);
    Eigen::Matrix3f K1 = Eigen::Matrix3f::Zero(), K2 = Eigen::Matrix3f::Zero();      // Pinhole::toK_()
    K1(0, 0) = pKF1->fx; K1(0, 2) = pKF1->cx; K1(1, 1) = pKF1->fy; K1(1, 2) = pKF1->cy; K1(2, 2) = 1.f;
    K2(0, 0) = pKF2->fx; K2(0, 2) = pKF2->cx; K2(1, 1) = pKF2->fy; K2(1, 2) = pKF2->cy; K2(2, 2) = 1.f;
    const Eigen::Matrix3f F12 = K1.transpose().inverse() * t12x * R12 * K2.inverse();

    const std::vector<MapPoint*> vpMP1 = pKF1->GetMapPointMatches(), vpMP2 = pKF2->GetMapPointMatches();
    const int N1 = (int)vpMP1.size(), N2 = (int)vpMP2.size();
    // queries: keyframe-1 features without a map point (stereo ones when bOnlyStereo), FeatureVector order
    std::vector<int> src;
    std::vector<orbx_keypoint> kp1;
    std::vector<uint8_t> desc1, stereo1;
    std::vector<int32_t> node1;
    for (DBoW2::FeatureVector::const_iterator it = pKF1->mFeatVec.begin(); it != pKF1->mFeatVec.end(); ++it)
        for (size_t k = 0; k < it->second.size(); ++k) {
            const int idx1 = (int)it->second[k];
            if (vpMP1[idx1]) continue;                                   // :1111-1114
            const bool bStereo1 = pKF1->mvuRight[idx1] >= 0;
            if (bOnlyStereo && !bStereo1) continue;                       // :1118-1120
            src.push_back(idx1);
            orbx_keypoint kk;
            put_keypoint(kk, pKF1->mvKeysUn[idx1]);
            kp1.push_back(kk);
            const size_t o = desc1.size();
            desc1.resize(o + 32);
            std::memcpy(&desc1[o], pKF1->mDescriptors.ptr<unsigned char>(idx1), 32);
            node1.push_back((int32_t)it->first);
            stereo1.push_back(bStereo1 ? 1 : 0);
        }
    vMatchedPairs.clear();
    const int nq = (int)src.size();
    if (nq == 0 || N2 == 0) return 0;
    std::vector<orbx_keypoint> kp2(N2);
    std::vector<uint8_t> desc2((size_t)N2 * 32), valid2(N2), stereo2(N2);
    std::vector<int32_t> node2(N2, -1);
    for (int i = 0; i < N2; ++i) {
        put_keypoint(kp2[i], pKF2->mvKeysUn[i]);
        std::memcpy(&desc2[(size_t)i * 32], pKF2->mDescriptors.ptr<unsigned char>(i), 32);
        stereo2[i] = pKF2->mvuRight[i] >= 0 ? 1 : 0;
        valid2[i] = (!vpMP2[i] && (!bOnlyStereo || stereo2[i])) ? 1 : 0;  // :1137-1146
    }
    for (DBoW2::FeatureVector::const_iterator it = pKF2->mFeatVec.begin(); it != pKF2->mFeatVec.end(); ++it)
        for (size_t k = 0; k < it->second.size(); ++k)
            if ((int)it->second[k] < N2) node2[it->second[k]] = (int32_t)it->first;
    orbm_triangulation t;
    t.n_queries = nq; t.n2 = N2;
    t.kp1 = kp1.data(); t.desc1 = desc1.data(); t.node1 = node1.data(); t.stereo1 = stereo1.data();
    t.kp2 = kp2.data(); t.desc2 = desc2.data(); t.node2 = node2.data(); t.valid2 = valid2.data(); t.stereo2 = stereo2.data();
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) t.F12[3 * r + c] = F12(r, c);
    t.epipole2[0] = epx; t.epipole2[1] = epy;
    t.coarse = bCoarse ? 1 : 0; t.check_orientation = mbCheckOrientation ? 1 : 0;
    std::vector<int32_t> match12(nq, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_triangulation(h, &t, match12.data(), &nmatches), "orbm_search_triangulation");
    std::vector<int> vMatches12(N1, -1);
    for (int k = 0; k < nq; ++k) vMatches12[src[k]] = match12[k];
    vMatchedPairs.reserve(nmatches);                                      // :1311-1320
    for (int i = 0; i < N1; ++i)
        if (vMatches12[i] >= 0) vMatchedPairs.push_back(std::make_pair((size_t)i, (size_t)vMatches12[i]));
    return nmatches;
}

}  // namespace ORB_SLAM3
