// ORBmatcher_init_b200.cc -- ORBmatcher::SearchForInitialization (/root/reference/src/ORBmatcher.cc:734-890) on the GPU.
//
// Compiled against the reference's UNMODIFIED include/ORBmatcher.h.  Monocular initialisation (Tracking.cc:2588) runs it on every frame
// until a map exists: the reference frame F1 (host memory) against the current frame F2, which is the frame its extractor produced last
// and therefore still on the device -- else F2's own arrays are uploaded.  On the host: vnMatches12 sized to F1, the search call, and the
// refresh of vbPrevMatched from the matches (:880-884).  Windows around vbPrevMatched, the level-0 rule, ratio test, match stealing through
// vnMatches21 / vMatchedDistance and the rotation histogram are orbm_search_initialization.
#include <string>
#include <vector>

#include "ORBmatcher.h"        // the reference's header
#include "marshal.h"

namespace ORB_SLAM3 {

int ORBmatcher::SearchForInitialization(Frame& F1, Frame& F2, std::vector<cv::Point2f>& vbPrevMatched, std::vector<int>& vnMatches12, int windowSize) {
    const char* who = "ORBmatcher::SearchForInitialization";
    if (F1.Nleft != -1 || F2.Nleft != -1) throw orb_b200::Error(std::string(who) + ": Nleft != -1 (fisheye stereo rig) is not built on the GPU path");
    orbx_handle* h = orb_b200_handle_of(F2.mpORBextractorLeft);
    if (!h) throw orb_b200::Error(std::string(who) + ": the frame's extractor is not a GPU-path extractor");
    const int n1 = (int)F1.mvKeysUn.size(), n2 = (int)F2.mvKeysUn.size();
    vnMatches12 = std::vector<int>(n1, -1);
    if (n1 == 0 || n2 == 0) return 0;
    const orb_b200::Features f1 = orb_b200::features_of(F1.mvKeysUn, F1.mDescriptors, n1);
    std::vector<float> prev((size_t)n1 * 2);
    for (int i = 0; i < n1; ++i) { prev[2 * i] = vbPrevMatched[i].x; prev[2 * i + 1] = vbPrevMatched[i].y; }
    orbm_init_queries q;
    q.n1 = n1; q.kp1 = f1.kp.data(); q.desc1 = f1.desc.data(); q.prev_matched = prev.data();
    int32_t resident = -1;
    orb_b200::check(orbx_counts(h, &resident, nullptr, nullptr), "orbx_counts");
    orb_b200::Features f2;
    if (resident == F2.N && F2.N == n2) {      // F2 is what its extractor produced last: search it where it lies
        q.n2 = 0; q.kp2 = nullptr; q.desc2 = nullptr; q.target_image = 0;
    } else {
        f2 = orb_b200::features_of(F2.mvKeysUn, F2.mDescriptors, n2);
        q.n2 = n2; q.kp2 = f2.kp.data(); q.desc2 = f2.desc.data(); q.target_image = -1;
    }
    const orbm_camera cam = orb_b200::camera_of(F2);
    int32_t nmatches = 0;
    orb_b200::check(orbm_search_initialization(h, &cam, &q, windowSize, mfNNratio, mbCheckOrientation ? 1 : 0, vnMatches12.data(), &nmatches),
                    "orbm_search_initialization");
    for (int i1 = 0; i1 < n1; ++i1)            // :880-884
        if (vnMatches12[i1] >= 0) vbPrevMatched[i1] = F2.mvKeysUn[vnMatches12[i1]].pt;
    return nmatches;
}

}  // namespace ORB_SLAM3
