// ORBmatcher_bow_b200.cc -- the two bag-of-words searches of ORB_SLAM3::ORBmatcher (/root/reference/src/ORBmatcher.cc) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h, next to ORBmatcher_b200.cc (constructor, constants, the per-frame
// projection searches):
//   SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>& vpMapPointMatches)        ORBmatcher.cc:259-493  (TrackReferenceKeyFrame, Relocalization)
//   SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12)        ORBmatcher.cc:892-1043 (loop closing / place recognition)
// Only marshaling happens here: the FeatureVector merge order of the query side (ascending vocabulary node, ascending feature index
// inside a node, features that hold a good map point), the vocabulary node of every target feature, and the map points written back.
// The first overload reads the frame's keypoints and descriptors from the DEVICE (the frame its extractor produced last); the second
// takes both keyframes from the host.  Nleft != -1 rigs (fisheye pairs) are not built.
#include <cstring>
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "marshal.h"

// The workspace of the keyframe-to-keyframe searches (orb_b200_host.h).
static orbx_handle* g_keyframe_search_handle = nullptr;
extern "C" void orb_b200_use_handle_for_keyframe_searches(orbx_handle* h) { g_keyframe_search_handle = h; }
extern "C" orbx_handle* orb_b200_keyframe_search_handle(void) { return g_keyframe_search_handle; }   // SearchForTriangulation uses the same one

namespace ORB_SLAM3 {

namespace {

struct QuerySide {            // the keyframe whose map points are looked for
    std::vector<int> src;     // keyframe feature of every query
    std::vector<int32_t> node;
    std::vector<float> angle;
    std::vector<uint8_t> desc;
};

QuerySide query_side(KeyFrame* pKF, const std::vector<MapPoint*>& vpMapPointsKF, const char* who) {
    if (pKF->mpCamera2 || pKF->NLeft != -1) throw orb_b200::Error(std::string(who) + ": a keyframe with a second camera is not built on the GPU path");
    QuerySide q;
    for (DBoW2::FeatureVector::const_iterator it = pKF->mFeatVec.begin(); it != pKF->mFeatVec.end(); ++it)
        for (size_t k = 0; k < it->second.size(); ++k) {
            const unsigned int idx = it->second[k];
            MapPoint* pMP = vpMapPointsKF[idx];
            if (!pMP || pMP->isBad()) continue;
            q.src.push_back((int)idx);
            q.node.push_back((int32_t)it->first);
            q.angle.push_back(pKF->mvKeysUn[idx].angle);
            const size_t o = q.desc.size();
            q.desc.resize(o + 32);
            std::memcpy(&q.desc[o], pKF->mDescriptors.ptr<unsigned char>((int)idx), 32);
        }
    return q;
}

}  // namespace

// ORBmatcher.cc:259-493
int ORBmatcher::SearchByBoW(KeyFrame* pKF, Frame& F, std::vector<MapPoint*>& vpMapPointMatches) {
    const char* who = "ORBmatcher::SearchByBoW(KeyFrame*, Frame&)";
    orbx_handle* h = orb_b200::resident_frame(F, who);
    if (!g_keyframe_search_handle) g_keyframe_search_handle = h;
    const std::vector<MapPoint*> vpMapPointsKF = pKF->GetMapPointMatches();
    vpMapPointMatches = std::vector<MapPoint*>(F.N, static_cast<MapPoint*>(NULL));
    const QuerySide Q = query_side(pKF, vpMapPointsKF, who);
    const int nq = (int)Q.src.size();
    if (nq == 0 || F.N == 0) return 0;
    const std::vector<int32_t> feature_node = orb_b200::node_of_features(F.mFeatVec, F.N);
    const int32_t frame_image = 0, query_offset[2] = {0, nq};
    orbm_bow_queries q;
    q.n_frames = 1; q.on_device = 0; q.frame_image = &frame_image; q.query_offset = query_offset;
    q.query_node = Q.node.data(); q.query_angle = Q.angle.data(); q.desc = Q.desc.data(); q.feature_node = feature_node.data();
    std::vector<int32_t> fmatch(F.N, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_bow(h, &q, mfNNratio, mbCheckOrientation ? 1 : 0, fmatch.data(), &nmatches), "orbm_search_bow");
    for (int i = 0; i < F.N; ++i)
        if (fmatch[i] >= 0) vpMapPointMatches[i] = vpMapPointsKF[Q.src[fmatch[i]]];
    return nmatches;
}

// ORBmatcher.cc:892-1043
int ORBmatcher::SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, std::vector<MapPoint*>& vpMatches12) {
    const char* who = "ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*)";
    const std::vector<MapPoint*> vpMapPoints1 = pKF1->GetMapPointMatches(), vpMapPoints2 = pKF2->GetMapPointMatches();
    vpMatches12 = std::vector<MapPoint*>(vpMapPoints1.size(), static_cast<MapPoint*>(NULL));
    const QuerySide Q = query_side(pKF1, vpMapPoints1, who);
    if (pKF2->mpCamera2 || pKF2->NLeft != -1) throw orb_b200::Error(std::string(who) + ": a keyframe with a second camera is not built on the GPU path");
    const int nq = (int)Q.src.size(), n2 = (int)vpMapPoints2.size();
    if (nq == 0 || n2 == 0) return 0;
    const orb_b200::Features F2 = orb_b200::features_of(pKF2->mvKeysUn, pKF2->mDescriptors, n2);
    std::vector<uint8_t> valid2(n2);
    for (int i = 0; i < n2; ++i) valid2[i] = (vpMapPoints2[i] && !vpMapPoints2[i]->isBad()) ? 1 : 0;
    const std::vector<int32_t> node2 = orb_b200::node_of_features(pKF2->mFeatVec, n2);
    const int32_t feat_offset[2] = {0, n2}, query_offset[2] = {0, nq};
    orbm_bow_kf_queries q;
    q.n_pairs = 1; q.feat_offset = feat_offset; q.kp2 = F2.kp.data(); q.desc2 = F2.desc.data(); q.node2 = node2.data(); q.valid2 = valid2.data();
    q.query_offset = query_offset; q.query_node = Q.node.data(); q.query_angle = Q.angle.data(); q.desc1 = Q.desc.data();
    std::vector<int32_t> match12(nq, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_bow_keyframes(orb_b200::keyframe_search_handle(who), &q, mfNNratio, mbCheckOrientation ? 1 : 0, match12.data(), &nmatches), "orbm_search_bow_keyframes");
    for (int k = 0; k < nq; ++k)
        if (match12[k] >= 0) vpMatches12[Q.src[k]] = vpMapPoints2[match12[k]];
    return nmatches;
}

}  // namespace ORB_SLAM3
