// ORBmatcher_b200.cc -- the per-frame members of ORB_SLAM3::ORBmatcher (/root/reference/src/ORBmatcher.cc) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  Provides the constructor, the three static constants,
// DescriptorDistance and the two searches the tracking thread runs on every frame:
//   SearchByProjection(Frame&, const vector<MapPoint*>&, th, bFarPoints, thFarPoints)   ORBmatcher.cc:45-239   (Tracking.cc:4062)
//   SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, th, bMono)          ORBmatcher.cc:1950-2184 (Tracking.cc:3389)
// Link this object BEFORE the reference's ORBmatcher.o with -Wl,--allow-multiple-definition (GNU ld keeps the first definition),
// or exclude those bodies from ORBmatcher.cc; the remaining eleven searches keep the reference's code or take the C-ABI recipes
// of INTEGRATION.md (every one of them has a kernel: orbm_search_keyframe, orbm_search_bow*, orbm_search_triangulation, ...).
//
// Both searches read the frame's keypoints, descriptors, mvuRight and grid from the DEVICE: the frame searched is the frame the
// GPU-path extractor behind F.mpORBextractorLeft produced last (true at both call sites: the current frame), so nothing but the
// query side (a few KB per call) is uploaded.  Only marshaling happens here; Nleft != -1 rigs (fisheye pairs) are not built.
#include <cmath>
#include <cstring>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "orb_b200_host.h"

namespace ORB_SLAM3 {

const int ORBmatcher::TH_HIGH = 100;        // ORBmatcher.cc:35-37
const int ORBmatcher::TH_LOW = 50;
const int ORBmatcher::HISTO_LENGTH = 30;

ORBmatcher::ORBmatcher(float nnratio, bool checkOri) : mfNNratio(nnratio), mbCheckOrientation(checkOri) {}

// ORBmatcher.cc:2383-2403: one pair of 256-bit descriptors.  (A scalar utility for host callers such as MapPoint.cc:496; the
// batched distances of every search are __popc inside the kernels.)
int ORBmatcher::DescriptorDistance(const cv::Mat& a, const cv::Mat& b) {
    unsigned long long x[4], y[4];
    std::memcpy(x, a.ptr<unsigned char>(), 32);
    std::memcpy(y, b.ptr<unsigned char>(), 32);
    int d = 0;
    for (int i = 0; i < 4; ++i) d += __builtin_popcountll(x[i] ^ y[i]);
    return d;
}

namespace {
orbm_camera camera_of(const Frame& F) {
    orbm_camera c;
    c.fx = Frame::fx; c.fy = Frame::fy; c.cx = Frame::cx; c.cy = Frame::cy; c.bf = F.mbf; c.b = F.mb;
    c.min_x = Frame::mnMinX; c.max_x = Frame::mnMaxX; c.min_y = Frame::mnMinY; c.max_y = Frame::mnMaxY;
    return c;
}
orbx_handle* device_frame(const Frame& F, const char* who) {
    if (F.Nleft != -1) throw orb_b200::Error(std::string(who) + ": Nleft != -1 (fisheye stereo rig) is not built on the GPU path");
    orbx_handle* h = orb_b200_handle_of(F.mpORBextractorLeft);
    if (!h) throw orb_b200::Error(std::string(who) + ": the frame's extractor is not a GPU-path extractor");
    int32_t n = 0;
    orb_b200::check(orbx_counts(h, &n, nullptr, nullptr), "orbx_counts");
    if (n != F.N) throw orb_b200::Error(std::string(who) + ": the frame is not the one its extractor produced last");
    return h;
}
}  // namespace

// ORBmatcher.cc:45-239
int ORBmatcher::SearchByProjection(Frame& F, const std::vector<MapPoint*>& vpMapPoints, const float th, const bool bFarPoints,
                                   const float thFarPoints) {
    orbx_handle* h = device_frame(F, "ORBmatcher::SearchByProjection(Frame&, vpMapPoints)");
    const int nq = (int)vpMapPoints.size();
    if (nq == 0) return 0;
    std::vector<float> px(nq), py(nq), pxr(nq), vcos(nq), depth(nq);
    std::vector<int32_t> level(nq);
    std::vector<uint8_t> desc((size_t)nq * 32), in_view(nq), claimed(F.N, 0);
    for (int i = 0; i < nq; ++i) {
        MapPoint* pMP = vpMapPoints[i];
        // :52-58 -- the far-point gate is applied by the kernel from track_depth
        in_view[i] = (pMP->mbTrackInView && !pMP->isBad()) ? 1 : 0;
        px[i] = pMP->mTrackProjX; py[i] = pMP->mTrackProjY; pxr[i] = pMP->mTrackProjXR;
        level[i] = pMP->mnTrackScaleLevel; vcos[i] = pMP->mTrackViewCos; depth[i] = pMP->mTrackDepth;
        if (in_view[i]) {
            const cv::Mat d = pMP->GetDescriptor();
            std::memcpy(&desc[(size_t)i * 32], d.ptr<unsigned char>(), 32);
        }
    }
    for (int idx = 0; idx < F.N; ++idx)   // :101-103
        if (F.mvpMapPoints[idx] && F.mvpMapPoints[idx]->Observations() > 0) claimed[idx] = 1;
    const int32_t frame_image = 0, query_offset[2] = {0, nq};
    orbm_local_queries q;
    q.n_frames = 1; q.on_device = 0; q.frame_image = &frame_image; q.query_offset = query_offset;
    q.proj_x = px.data(); q.proj_y = py.data(); q.proj_xr = pxr.data(); q.level = level.data(); q.view_cos = vcos.data();
    q.track_depth = depth.data(); q.desc = desc.data(); q.feature_claimed = claimed.data(); q.in_view = in_view.data();
    const orbm_camera cam = camera_of(F);
    std::vector<int32_t> match(nq, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_local_points(h, &cam, &q, th, mfNNratio, bFarPoints ? 1 : 0, thFarPoints, match.data(), &nmatches),
                    "orbm_search_local_points");
    for (int i = 0; i < nq; ++i)
        if (match[i] >= 0) F.mvpMapPoints[match[i]] = vpMapPoints[i];   // :152
    return nmatches;
}

// ORBmatcher.cc:1950-2184
int ORBmatcher::SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, const float th, const bool bMono) {
    orbx_handle* h = device_frame(CurrentFrame, "ORBmatcher::SearchByProjection(CurrentFrame, LastFrame)");
    if (LastFrame.Nleft != -1) throw orb_b200::Error("SearchByProjection(CurrentFrame, LastFrame): Nleft != -1 is not built");
    // :1964-1971, in the caller's own Sophus / Eigen float arithmetic
    const Sophus::SE3f Tcw = CurrentFrame.GetPose();
    const Eigen::Vector3f twc = Tcw.inverse().translation();
    const Sophus::SE3f Tlw = LastFrame.GetPose();
    const Eigen::Vector3f tlc = Tlw * twc;
    const bool bForward = tlc(2) > CurrentFrame.mb && !bMono;
    const bool bBackward = -tlc(2) > CurrentFrame.mb && !bMono;
    std::vector<int> src;                       // LastFrame feature of every query (:1975-1981)
    src.reserve(LastFrame.N);
    for (int i = 0; i < LastFrame.N; ++i)
        if (LastFrame.mvpMapPoints[i] && !LastFrame.mvbOutlier[i]) src.push_back(i);
    const int nq = (int)src.size();
    if (nq == 0) return 0;
    std::vector<float> pos((size_t)nq * 3), angle(nq);
    std::vector<int32_t> octave(nq);
    std::vector<uint8_t> desc((size_t)nq * 32), obs(nq);
    for (int k = 0; k < nq; ++k) {
        const int i = src[k];
        MapPoint* pMP = LastFrame.mvpMapPoints[i];
        const Eigen::Vector3f x = pMP->GetWorldPos();
        pos[3 * k] = x(0); pos[3 * k + 1] = x(1); pos[3 * k + 2] = x(2);
        octave[k] = LastFrame.mvKeys[i].octave;        // :1995
        angle[k] = LastFrame.mvKeysUn[i].angle;        // :2080
        const cv::Mat d = pMP->GetDescriptor();
        std::memcpy(&desc[(size_t)k * 32], d.ptr<unsigned char>(), 32);
        obs[k] = pMP->Observations() > 0 ? 1 : 0;
    }
    const Eigen::Quaternionf qc = Tcw.unit_quaternion();
    const float T7[7] = {qc.x(), qc.y(), qc.z(), qc.w(), Tcw.translation()(0), Tcw.translation()(1), Tcw.translation()(2)};
    const int32_t frame_image = 0, query_offset[2] = {0, nq}, direction = bForward ? 1 : (bBackward ? 2 : 0);
    orbm_last_queries q;
    q.n_frames = 1; q.on_device = 0; q.frame_image = &frame_image; q.query_offset = query_offset; q.Tcw = T7; q.direction = &direction;
    q.world_pos = pos.data(); q.last_octave = octave.data(); q.last_angle = angle.data(); q.desc = desc.data(); q.obs_positive = obs.data();
    const orbm_camera cam = camera_of(CurrentFrame);
    std::vector<int32_t> fmatch(CurrentFrame.N > 0 ? CurrentFrame.N : 1, -1);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_last_frame(h, &cam, &q, th, mbCheckOrientation ? 1 : 0, fmatch.data(), &nmatches), "orbm_search_last_frame");
    for (int idx = 0; idx < CurrentFrame.N; ++idx)   // :2068 and the rotation-consistency removals :2163-2177 are already applied
        if (fmatch[idx] >= 0) CurrentFrame.mvpMapPoints[idx] = LastFrame.mvpMapPoints[src[fmatch[idx]]];
    return nmatches;
}

// protected helpers the reference's remaining members call (ORBmatcher.cc:241-247, 2335-2381)
float ORBmatcher::RadiusByViewingCos(const float& viewCos) { return viewCos > 0.998f ? 2.5f : 4.0f; }

void ORBmatcher::ComputeThreeMaxima(std::vector<int>* histo, const int L, int& ind1, int& ind2, int& ind3) {
    int max1 = 0, max2 = 0, max3 = 0;
    for (int i = 0; i < L; ++i) {
        const int s = (int)histo[i].size();
        if (s > max1) { max3 = max2; max2 = max1; max1 = s; ind3 = ind2; ind2 = ind1; ind1 = i; }
        else if (s > max2) { max3 = max2; max2 = s; ind3 = ind2; ind2 = i; }
        else if (s > max3) { max3 = s; ind3 = i; }
    }
    if (max2 < 0.1f * (float)max1) { ind2 = -1; ind3 = -1; }
    else if (max3 < 0.1f * (float)max1) ind3 = -1;
}

}  // namespace ORB_SLAM3
