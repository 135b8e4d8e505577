// Frame_stereo_b200.cc -- Frame::ComputeStereoMatches (/root/reference/src/Frame.cc:1102-1358) and Frame::ComputeStereoFromRGBD on the GPU.
//
// Replaces those two members of the reference's Frame.cc (compile Frame.cc with the members' bodies excluded, or link this object
// first with -Wl,--allow-multiple-definition; INTEGRATION.md).  The frame's extractor objects are ours (host/ORBextractor_b200.cc), so
// its pyramids, keypoints and descriptors are already resident on the device.  ComputeStereoMatches runs the row-band candidate
// search, the Hamming match, the 11x11 SAD refinement with its parabola and the 2.1 x median filter there (k_stereo_match_v1 /
// k_stereo_median); ComputeStereoFromRGBD samples the depth map at every keypoint there (k_stereo_rgbd).  Only mvuRight / mvDepth
// (2 x N floats) come back, and they stay on the device for the ORBmatcher members that search this frame next.
#include <vector>

#include "Frame.h"            // the reference's header in a real build; refshim/ref_skeleton.h in the compile check
#include "marshal.h"

namespace ORB_SLAM3 {

void Frame::ComputeStereoMatches() {
    mvuRight = std::vector<float>(N, -1.0f);      // Frame.cc:1114-1115
    mvDepth = std::vector<float>(N, -1.0f);
    orbx_handle* hl = orb_b200_handle_of(mpORBextractorLeft);
    orbx_handle* hr = orb_b200_handle_of(mpORBextractorRight);
    if (!hl || !hr) throw orb_b200::Error("Frame::ComputeStereoMatches: the frame's extractors are not GPU-path extractors");
    if (N == 0) return;
    orb_b200::check(orbm_stereo_pair(hl, hr, mbf, mb, mvuRight.data(), mvDepth.data(), N), "orbm_stereo_pair");
}

// The RGB-D constructor calls this after ExtractORB(0, imGray, 0, 0) and UndistortKeyPoints, which is an identity copy for a camera with
// zero distortion: the keypoints sampled are the frame's mvKeys on the device.  imDepth is the map Tracking::GrabImageRGBD has already
// converted to CV_32F (scaled by mDepthMapFactor unless that is within 1e-5 of 1), so it goes up as it is, with factor 1.
void Frame::ComputeStereoFromRGBD(const cv::Mat& imDepth) {
    mvuRight = std::vector<float>(N, -1.0f);
    mvDepth = std::vector<float>(N, -1.0f);
    if (N == 0) return;
    orbx_handle* h = orb_b200::resident_frame(*this, "Frame::ComputeStereoFromRGBD");
    int32_t w = 0, hh = 0;
    orb_b200::check(orbx_level_size(h, 0, &w, &hh), "orbx_level_size");
    if (imDepth.type() != CV_32F || imDepth.cols != w || imDepth.rows != hh)
        throw orb_b200::Error("Frame::ComputeStereoFromRGBD: the depth map must be CV_32F and of the image's size (Tracking::GrabImageRGBD)");
    const size_t stride = (size_t)imDepth.step;
    orb_b200::check(orbm_stereo_rgbd_batch(h, 1, imDepth.ptr<float>(0), ORB_DEPTH_F32, (int32_t)stride, stride * (size_t)hh, 1.0f, 0, mbf),
                    "orbm_stereo_rgbd_batch");
    orb_b200::check(orbm_stereo_download(h, mvuRight.data(), mvDepth.data(), N), "orbm_stereo_download");
}

}  // namespace ORB_SLAM3
