// tests/host/fuse_stub.cc -- TEST INFRASTRUCTURE (CPU tier): orbm_search_keyframe over the oracle (orc_search_keyframe) instead of the GPU, so that
// host/ORBmatcher_fuse_b200.cc (caller-side skips, raw distances through the protected-member access, map mutations in query order) can run
// without a GPU next to the reference's own function (oracle/_ref part 2; tests/test_host_fuse_vs_ref.py).  Never linked into the product.
#include <cmath>
#include <cstdint>
#include <vector>

#include "orbslam3_b200.h"

extern "C" int orc_search_keyframe(int variant, const orbx_keypoint* kps, const uint8_t* desc, const float* uright, int N, const float* bounds4,
                                   const float* scaleFactors, const float* invLevelSigma2, int nLevels, float logScaleFactor, const float* cam6,
                                   const float* Tcw7, const float* Ow, const float* S8, int nq, const float* xw, const float* normal, const float* maxDist,
                                   const float* minDist, const uint8_t* qdesc, const float* qangle, uint8_t* claimed, float th, float thr, int checkOri,
                                   int* match);
static float g_logsf = 0;
static std::vector<orbx_keypoint> g_kps;
static std::vector<uint8_t> g_desc;
static std::vector<float> g_ur;

extern "C" {
void fuse_stub_set_log_scale_factor(float v) { g_logsf = v; }     // the handle's mfLogScaleFactor (glibc logf(1.2f), taken from the test)
void fuse_stub_set_frame(const orbx_keypoint* kps, const uint8_t* desc, const float* ur, int n) { g_kps.assign(kps, kps + n); g_desc.assign(desc, desc + 32 * (size_t)n); g_ur.assign(ur, ur + n); }
orbx_handle* orb_b200_handle_of(const void*) { static int dummy; return reinterpret_cast<orbx_handle*>(&dummy); }
orb_status orbx_counts(orbx_handle*, int32_t* n_total, int32_t*, int32_t*) { *n_total = (int32_t)g_kps.size(); return ORB_OK; }
const char* orb_last_error(void) { return "fuse_stub"; }
orbx_handle* orb_b200_keyframe_search_handle(void) { static int dummy; return reinterpret_cast<orbx_handle*>(&dummy); }
orb_status orbm_search_keyframe(orbx_handle*, const orbm_camera* cam, const orbm_kf_queries* q, int32_t variant, float th, float hamming_max, int32_t check,
                                int32_t* match, int32_t* nm) {
    if (q->n_targets != 1) return ORB_ERR_INVALID;
    const bool resident = q->kp == nullptr;            // the registered frame plays the image on the device
    if (resident && q->target_image[0] != 0) return ORB_ERR_INVALID;
    const int N = resident ? (int)g_kps.size() : q->feat_offset[1];
    std::vector<uint8_t> claimed(N + 1, 0);
    if (q->feat_claimed) claimed.assign(q->feat_claimed, q->feat_claimed + N);
    float sf[8], isg[8];                      // the handle's level tables: scaleFactor 1.2, 8 levels (ORBextractor.cc:484-494)
    sf[0] = 1.0f;
    for (int i = 1; i < 8; ++i) sf[i] = (float)(sf[i - 1] * 1.2f);
    for (int i = 0; i < 8; ++i) isg[i] = 1.0f / (sf[i] * sf[i]);
    const float bounds[4] = {cam->min_x, cam->max_x, cam->min_y, cam->max_y};
    const float cam6[6] = {cam->fx, cam->fy, cam->cx, cam->cy, cam->bf, cam->b};
    nm[0] = orc_search_keyframe(variant, resident ? g_kps.data() : q->kp, resident ? g_desc.data() : q->desc, resident ? g_ur.data() : q->uright, N, bounds, sf, isg, 8, g_logsf, cam6, q->Tcw, q->Ow, q->Sim3,
                                q->query_offset[1], q->world_pos, q->normal, q->max_dist, q->min_dist, q->desc_q, q->angle, q->feat_claimed ? claimed.data() : nullptr, th, hamming_max, check, match);
    return ORB_OK;
}
}
