// tests/host/bow_stub.cc -- TEST INFRASTRUCTURE (CPU tier): orbm_search_bow / orbm_search_bow_keyframes over the oracle instead of the GPU,
// so that host/ORBmatcher_bow_b200.cc (FeatureVector merge order, per-feature nodes, written map points) can run without a GPU next to
// the reference's own functions (oracle/_ref part 2; tests/test_host_bow_vs_ref.py).  The frame "resident on the device" is the one
// the driver registers with bow_stub_set_frame.  Never linked into the product.
#include <cstdint>
#include <vector>

#include "orbslam3_b200.h"

extern "C" int orc_search_bow(const orbx_keypoint* kps, const uint8_t* desc, const int* feat_node, int N, int nq, const int* qnode, const float* qangle,
                              const uint8_t* qdesc, float nnratio, int checkOri, int* feat_match);
extern "C" int orc_search_bow_kf(const orbx_keypoint* kp2, const uint8_t* desc2, const int* node2, const uint8_t* valid2, int n2, int nq, const int* qnode,
                                 const float* qangle, const uint8_t* desc1, float nnratio, int checkOri, int* match12);

extern "C" int orc_search_triangulation(int nq, const orbx_keypoint* kp1, const uint8_t* desc1, const int* node1, const uint8_t* stereo1, int N2,
                                        const orbx_keypoint* kp2, const uint8_t* desc2, const int* node2, const uint8_t* valid2, const uint8_t* stereo2,
                                        const float* F12, const float* ep2, const float* scaleFactors, const float* sigma2, int bCoarse, int checkOri, int* match12);

extern "C" int orc_search_initialization(const orbx_keypoint* kp1, const uint8_t* desc1, int n1, const float* prevMatched, const orbx_keypoint* kp2,
                                         const uint8_t* desc2, int n2, const float* bounds4, int windowSize, float nnratio, int checkOri, int* matches12);

static std::vector<orbx_keypoint> g_kps;
static std::vector<uint8_t> g_desc;

extern "C" {
void bow_stub_set_frame(const orbx_keypoint* kps, const uint8_t* desc, int n) { g_kps.assign(kps, kps + n); g_desc.assign(desc, desc + 32 * (size_t)n); }
const char* orb_last_error(void) { return "bow_stub"; }
orbx_handle* orb_b200_handle_of(const void*) { static int dummy; return reinterpret_cast<orbx_handle*>(&dummy); }
orb_status orbx_counts(orbx_handle*, int32_t* n_total, int32_t*, int32_t*) { *n_total = (int32_t)g_kps.size(); return ORB_OK; }

orb_status orbm_search_bow(orbx_handle*, const orbm_bow_queries* q, float nnratio, int32_t check, int32_t* fm, int32_t* nm) {
    if (q->n_frames != 1 || q->on_device || q->frame_image[0] != 0) return ORB_ERR_INVALID;
    const int nq = q->query_offset[1] - q->query_offset[0];
    nm[0] = orc_search_bow(g_kps.data(), g_desc.data(), q->feature_node, (int)g_kps.size(), nq, q->query_node, q->query_angle, q->desc, nnratio, check, fm);
    return ORB_OK;
}
orb_status orbm_search_initialization(orbx_handle*, const orbm_camera* cam, const orbm_init_queries* q, int32_t window, float nnratio, int32_t check, int32_t* m12,
                                      int32_t* nm) {
    const float bounds[4] = {cam->min_x, cam->max_x, cam->min_y, cam->max_y};
    const bool resident = q->kp2 == nullptr;      // the registered frame plays the image on the device
    if (resident && q->target_image != 0) return ORB_ERR_INVALID;
    nm[0] = orc_search_initialization(q->kp1, q->desc1, q->n1, q->prev_matched, resident ? g_kps.data() : q->kp2, resident ? g_desc.data() : q->desc2,
                                      resident ? (int)g_kps.size() : q->n2, bounds, window, nnratio, check, m12);
    return ORB_OK;
}
orb_status orbm_search_triangulation(orbx_handle*, const orbm_triangulation* t, int32_t* m12, int32_t* nm) {
    float sf[8], s2[8];                    // the handle's level tables: scaleFactor 1.2, 8 levels (ORBextractor.cc:484-494)
    sf[0] = 1.0f; s2[0] = 1.0f;
    for (int i = 1; i < 8; ++i) { sf[i] = (float)(sf[i - 1] * 1.2f); s2[i] = sf[i] * sf[i]; }
    nm[0] = orc_search_triangulation(t->n_queries, t->kp1, t->desc1, t->node1, t->stereo1, t->n2, t->kp2, t->desc2, t->node2, t->valid2, t->stereo2, t->F12,
                                     t->epipole2, sf, s2, t->coarse, t->check_orientation, m12);
    return ORB_OK;
}
orb_status orbm_search_bow_keyframes(orbx_handle*, const orbm_bow_kf_queries* q, float nnratio, int32_t check, int32_t* m12, int32_t* nm) {
    if (q->n_pairs != 1) return ORB_ERR_INVALID;
    const int n2 = q->feat_offset[1], nq = q->query_offset[1];
    nm[0] = orc_search_bow_kf(q->kp2, q->desc2, q->node2, q->valid2, n2, nq, q->query_node, q->query_angle, q->desc1, nnratio, check, m12);
    return ORB_OK;
}
}
