// Frame_stereo_b200.cc -- Frame::ComputeStereoMatches (/root/reference/src/Frame.cc:1102-1358) on the GPU.
//
// Replaces that one member of the reference's Frame.cc (compile Frame.cc with the member's body excluded, or link this object
// first with -Wl,--allow-multiple-definition; INTEGRATION.md).  Both extractor objects of the frame are ours
// (host/ORBextractor_b200.cc), so the two pyramids, keypoints and descriptors of this frame are already resident on the device:
// the row-band candidate search, the Hamming match, the 11x11 SAD refinement with its parabola and the 2.1 x median filter
// (k_stereo_match_v1 / k_stereo_median) run there, and only mvuRight / mvDepth (2 x N floats) come back.
#include <vector>

#include "Frame.h"            // the reference's header in a real build; refshim/ref_skeleton.h in the compile check
#include "orb_b200_host.h"

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

}  // namespace ORB_SLAM3
