// tests/host/voc_stub.cc -- TEST INFRASTRUCTURE (CPU tier): orbv_create / orbv_transform over the oracle (orc_bow_transform) instead of the
// GPU, so that host/Frame_bow_b200.cc (vocabulary flattening through the protected-member access, BowVector / FeatureVector filling) can
// run without a GPU (tests/test_host_voc_cpu.py).  The frame "resident on the device" is registered by the driver.  Never linked into
// the product.
#include <cstdint>
#include <vector>

#include "orbslam3_b200.h"

extern "C" int orc_bow_transform(int n_nodes, int L, const int* child_offset, const int* child_ids, const uint8_t* node_desc, const int* node_word,
                                 const double* node_weight, int levelsup, int n, const uint8_t* desc, int* word, int* node, double* weight, int* bow_word,
                                 double* bow_weight);

struct orbv_vocabulary {
    int n, L;
    std::vector<int> co, ci, word;
    std::vector<uint8_t> desc;
    std::vector<double> weight;
};
static std::vector<uint8_t> g_desc;
static int g_creates = 0;

extern "C" {
void voc_stub_set_frame(const uint8_t* desc, int n) { g_desc.assign(desc, desc + 32 * (size_t)n); }
int voc_stub_creates() { return g_creates; }
const char* orb_last_error(void) { return "voc_stub"; }
orbx_handle* orb_b200_handle_of(const void*) { static int dummy; return reinterpret_cast<orbx_handle*>(&dummy); }
orb_status orbx_counts(orbx_handle*, int32_t* n_total, int32_t*, int32_t*) { *n_total = (int32_t)(g_desc.size() / 32); return ORB_OK; }
int32_t orbx_max_features(const orbx_handle*) { return 4096; }
orb_status orbv_create(int32_t, int32_t n_nodes, int32_t depth_levels, const int32_t* child_offset, const int32_t* child_ids, const uint8_t* node_desc,
                       const int32_t* node_word, const double* node_weight, orbv_vocabulary** out) {
    orbv_vocabulary* v = new orbv_vocabulary;
    v->n = n_nodes; v->L = depth_levels;
    v->co.assign(child_offset, child_offset + n_nodes + 1);
    v->ci.assign(child_ids, child_ids + child_offset[n_nodes]);
    v->desc.assign(node_desc, node_desc + 32 * (size_t)n_nodes);
    v->word.assign(node_word, node_word + n_nodes);
    v->weight.assign(node_weight, node_weight + n_nodes);
    *out = v; ++g_creates;
    return ORB_OK;
}
void orbv_destroy(orbv_vocabulary* v) { delete v; }
orb_status orbv_transform(orbx_handle*, const orbv_vocabulary* v, int32_t levelsup, int32_t on_device, int32_t* word, int32_t* node, double* weight,
                          int32_t* bow_count, int32_t* bow_word, double* bow_weight) {
    if (on_device) return ORB_ERR_INVALID;
    bow_count[0] = orc_bow_transform(v->n, v->L, v->co.data(), v->ci.data(), v->desc.data(), v->word.data(), v->weight.data(), levelsup,
                                     (int)(g_desc.size() / 32), g_desc.data(), word, node, weight, bow_word, bow_weight);
    return ORB_OK;
}
}
