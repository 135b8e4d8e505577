// marshal.h -- the conversions between the reference's Frame / KeyFrame / MapPoint objects and the C ABI structs, written once for the
// host units that stand in for members of ORBmatcher, Frame and Optimizer.  Include it after the reference header the unit implements
// (ORBmatcher.h, Optimizer.h or Frame.h): that header declares the classes, Sophus and Eigen used here.
//
// A helper that reads a member the reference declares but not every unit's skeleton section provides (refshim/ref_skeleton.h: KeyFrame's
// image bounds, MapPoint's raw distances, the FeatureVector) is a template, so that the access is checked only where it is instantiated.
#pragma once
#include <array>
#include <cstring>
#include <string>
#include <vector>

#include "orb_b200_host.h"

namespace orb_b200 {

inline orbx_keypoint keypoint_of(const cv::KeyPoint& k) {
    orbx_keypoint o;
    o.x = k.pt.x; o.y = k.pt.y; o.size = k.size; o.angle = k.angle; o.response = k.response; o.octave = k.octave; o.class_id = k.class_id;
    return o;
}

// keypoints and descriptor rows of a feature list, flattened for the C ABI
struct Features {
    std::vector<orbx_keypoint> kp;
    std::vector<uint8_t> desc;
    void push(const cv::KeyPoint& k, const cv::Mat& D, int row) {
        kp.push_back(keypoint_of(k));
        const unsigned char* d = D.ptr<unsigned char>(row);
        desc.insert(desc.end(), d, d + 32);
    }
};
// the first n features
inline Features features_of(const std::vector<cv::KeyPoint>& keys, const cv::Mat& D, int n) {
    Features f;
    for (int i = 0; i < n; ++i) f.push(keys[i], D, i);
    return f;
}
// features idx[0], idx[1], ... in that order
inline Features features_of(const std::vector<cv::KeyPoint>& keys, const cv::Mat& D, const std::vector<int>& idx) {
    Features f;
    for (int i : idx) f.push(keys[i], D, i);
    return f;
}

// qx qy qz qw tx ty tz
inline std::array<float, 7> pose7(const Sophus::SE3f& T) {
    const Eigen::Quaternionf q = T.unit_quaternion();
    return {{q.x(), q.y(), q.z(), q.w(), T.translation()(0), T.translation()(1), T.translation()(2)}};
}

inline orbm_camera camera_of(const ORB_SLAM3::Frame& F) {
    orbm_camera c;
    c.fx = ORB_SLAM3::Frame::fx; c.fy = ORB_SLAM3::Frame::fy; c.cx = ORB_SLAM3::Frame::cx; c.cy = ORB_SLAM3::Frame::cy; c.bf = F.mbf; c.b = F.mb;
    c.min_x = ORB_SLAM3::Frame::mnMinX; c.max_x = ORB_SLAM3::Frame::mnMaxX; c.min_y = ORB_SLAM3::Frame::mnMinY; c.max_y = ORB_SLAM3::Frame::mnMaxY;
    return c;
}
template <class KeyFrame>
orbm_camera camera_of(const KeyFrame* pKF) {
    orbm_camera c;
    c.fx = pKF->fx; c.fy = pKF->fy; c.cx = pKF->cx; c.cy = pKF->cy; c.bf = pKF->mbf; c.b = pKF->mb;
    c.min_x = (float)pKF->mnMinX; c.max_x = (float)pKF->mnMaxX; c.min_y = (float)pKF->mnMinY; c.max_y = (float)pKF->mnMaxY;
    return c;
}

// MapPoint's RAW mfMinDistance / mfMaxDistance: the keyframe search applies 0.8f / 1.2f itself and PredictScale divides the raw value.
// They are protected members, read through a derived class (no change to the reference's header).
template <class MapPoint>
struct RawDistance : MapPoint {
    static float min_distance(const MapPoint& p) { return p.*(&RawDistance::mfMinDistance); }
    static float max_distance(const MapPoint& p) { return p.*(&RawDistance::mfMaxDistance); }
};

// The map-point queries of orbm_search_keyframe, one row per push: world position, viewing normal (when the variant reads one), raw
// distances and descriptor.  Read without mMutexPos, like every member the callers read from the thread that owns the map.
template <class MapPoint>
struct PointQueries {
    explicit PointQueries(bool with_normal) : with_normal(with_normal) {}
    void push(MapPoint* p) {
        const Eigen::Vector3f X = p->GetWorldPos();
        xw.insert(xw.end(), {X(0), X(1), X(2)});
        if (with_normal) {
            const Eigen::Vector3f n = p->GetNormal();
            nrm.insert(nrm.end(), {n(0), n(1), n(2)});
        }
        maxd.push_back(RawDistance<MapPoint>::max_distance(*p));
        mind.push_back(RawDistance<MapPoint>::min_distance(*p));
        const cv::Mat d = p->GetDescriptor();
        desc.insert(desc.end(), d.ptr<unsigned char>(), d.ptr<unsigned char>() + 32);
    }
    int size() const { return (int)maxd.size(); }
    void fill(orbm_kf_queries& q) const {
        q.world_pos = xw.data(); q.normal = with_normal ? nrm.data() : nullptr; q.max_dist = maxd.data(); q.min_dist = mind.data(); q.desc_q = desc.data();
    }
    const bool with_normal;
    std::vector<float> xw, nrm, maxd, mind;
    std::vector<uint8_t> desc;
};

// the vocabulary node of each of N features; -1: the feature is in no node of the FeatureVector
template <class FeatureVector>
std::vector<int32_t> node_of_features(const FeatureVector& fv, int N) {
    std::vector<int32_t> node(N > 0 ? N : 1, -1);
    for (const auto& kv : fv)
        for (unsigned int i : kv.second)
            if ((int)i < N) node[i] = (int32_t)kv.first;
    return node;
}

// The handle of the extractor that produced F, when F is what it produced last: F's keypoints, descriptors, mvuRight and grid are then
// on the device.  Nleft != -1 rigs (fisheye pairs) are not built.
inline orbx_handle* resident_frame(const ORB_SLAM3::Frame& F, const char* who) {
    if (F.Nleft != -1) throw Error(std::string(who) + ": Nleft != -1 (fisheye stereo rig) is not built on the GPU path");
    orbx_handle* h = orb_b200_handle_of(F.mpORBextractorLeft);
    if (!h) throw Error(std::string(who) + ": the frame's extractor is not a GPU-path extractor");
    int32_t n = 0;
    check(orbx_counts(h, &n, nullptr, nullptr), "orbx_counts");
    if (n != F.N) throw Error(std::string(who) + ": the frame is not the one its extractor produced last");
    return h;
}

inline orbx_handle* keyframe_search_handle(const char* who) {
    orbx_handle* h = orb_b200_keyframe_search_handle();
    if (!h) throw Error(std::string(who) + ": no device workspace yet (orb_b200_use_handle_for_keyframe_searches)");
    return h;
}

// One orbm_search_keyframe over a host keyframe's features for the points of vpPoints that skip(pMP) keeps: Fuse(pKF, vpMapPoints) and
// the Sim3 members.  Tcw and Ow come from the caller, in its own float arithmetic.  src[k] is the vpPoints index of query k and best[k]
// its keyframe feature, or -1.
struct KeyFrameSearch {
    std::vector<int> src;
    std::vector<int32_t> best;
    int32_t nmatches = 0;
};
template <class KeyFrame, class MapPoint, class Skip>
KeyFrameSearch search_keyframe(KeyFrame* pKF, const Sophus::SE3f& Tcw, const Eigen::Vector3f& Ow, const std::vector<MapPoint*>& vpPoints, Skip skip,
                               const uint8_t* feat_claimed, int variant, float th, float hamming_max, bool checkOri, const char* who) {
    orbx_handle* h = keyframe_search_handle(who);
    KeyFrameSearch R;
    PointQueries<MapPoint> Q(true);
    for (int i = 0; i < (int)vpPoints.size(); ++i) {
        if (skip(vpPoints[i])) continue;
        Q.push(vpPoints[i]);
        R.src.push_back(i);
    }
    const int nq = Q.size(), N = (int)pKF->mvKeysUn.size();
    R.best.assign(nq, -1);
    if (nq == 0 || N == 0) return R;
    const Features F = features_of(pKF->mvKeysUn, pKF->mDescriptors, N);
    const std::array<float, 7> T7 = pose7(Tcw);
    const float O3[3] = {Ow(0), Ow(1), Ow(2)};
    const int32_t feat_offset[2] = {0, N}, query_offset[2] = {0, nq};
    orbm_kf_queries q;
    std::memset(&q, 0, sizeof(q));
    q.n_targets = 1; q.feat_offset = feat_offset; q.kp = F.kp.data(); q.desc = F.desc.data(); q.uright = pKF->mvuRight.data(); q.feat_claimed = feat_claimed;
    q.Tcw = T7.data(); q.Ow = O3; q.query_offset = query_offset;
    Q.fill(q);
    const orbm_camera cam = camera_of(pKF);
    check(orbm_search_keyframe(h, &cam, &q, variant, th, hamming_max, checkOri ? 1 : 0, R.best.data(), &R.nmatches), "orbm_search_keyframe");
    return R;
}

}  // namespace orb_b200
