// extractor.h -- the extractor handle (device workspace of one ORBextractor object)
#pragma once
#include <vector>

#include "common.cuh"
#include "scratch.h"

struct orbr_state;
void orbr_release(struct orbx_handle* h);   // replay.cu
orb_status batch_rows(struct orbx_handle* h, int* rows);   // extractor.cu: compact rows of the last batch (orbx_counts)
// The batch count table (extractor.cu): queue its read-back on the handle's stream; after the wait, latch its capacity flags
orb_status queue_counts(struct orbx_handle* h);
orb_status latch_counts(struct orbx_handle* h);

// Camera images as they arrive (orbx_extract_batch_device_format, orbr_step): orb_image_format, size, row and image strides in bytes
struct ImageSource { int format, w, h; int64_t stride; size_t image_stride; };
// extractor.cu: fills the zero defaults of `src` (the size of the extracted w x hh image, tight strides) and refuses, before anything is
// queued, an unknown format or a stride below a row of pixels
orb_status check_source(ImageSource& src, int w, int hh);
// extractor.cu: a batch of checked HOST images uploaded into the handle's staging block, then orbx_extract_batch_device_format
orb_status extract_batch_source(struct orbx_handle* h, const uint8_t* imgs, int batch, int w, int hh, const ImageSource& src, int lap0, int lap1);

// extractor.cu: queues on the handle's stream the copy of `batch` images of `rows` rows of `row` bytes, from `src` (row pitch `src_pitch`,
// image stride `src_image`) to tight images at `dst` (row pitch `dst_pitch`, image stride dst_pitch x rows): one 2-D copy when the source
// images are tight too, else one per image
orb_status copy_images(struct orbx_handle* h, uint8_t* dst, size_t dst_pitch, const uint8_t* src, size_t src_pitch, size_t src_image, size_t row,
                       int rows, int batch, cudaMemcpyKind kind);

// Depth maps of RGB-D frames (orbm_stereo_rgbd_batch, orbr_step): orb_depth_format, row and image strides in bytes
struct DepthSource { int format; int64_t stride; size_t image_stride; };
// stereo.cu: fills the zero defaults of `d` (tight rows of w elements, tight maps of hh rows) and refuses, before anything is queued, an
// unknown format or a stride shorter than a row (an image stride shorter than a map, for n_images > 1) or not a multiple of the element
orb_status check_depth(DepthSource& d, int n_images, int w, int hh);

struct orbx_handle {
    orbx_config cfg{};
    orb::ExtractGeom geom{};
    int cur_w = -1, cur_h = -1;
    int fast_variant = 1; // 1 (default): k_fast_cells_v2; 0: the round-1 k_fast_cells (ORB_FAST_VARIANT=0 at orbx_create)
    std::vector<uint2> cells_host;   // k_fast_cells_v2: one record per non-empty FAST cell
    uint2* d_cells = nullptr;
    int fast_R = 0, fast_PW = 0, fast_LW = 0;
    int blur_variant = 2;    // 2: k_blur_mma (both passes as u8 IMMA, default), 1: k_blur<true> (IDP.4A horizontal pass), 0: k_blur<false>
    int resize_variant = 1;  // 1: k_resize_v2 (default), 0: k_resize
    bool fast_tma = false;   // ORB_FAST_TMA=1: k_fast_cells_v2<29, true> (window rows by cp.async.bulk + mbarrier)
    int qt_variant = 1;   // 1 (default): k_quadtree_v1; 0: k_quadtree (ORB_QT_VARIANT=0 at orbx_create)
    cudaStream_t stream = nullptr;
    static const int kProfRing = 32;
    cudaEvent_t evr[kProfRing][8] = {};   // ring of per-batch stage events
    cudaEvent_t* ev = evr[0];
    int prof_count = 0;
    bool profiling = false;
    // ORBextractor.h:97-108 tables
    std::vector<float> scale, inv_scale, sigma2, inv_sigma2;
    std::vector<int> quota, umax;
    std::vector<int2> taps_host;
    // device workspace (sized for max_width x max_height x max_batch), carved from one block (orbx_create)
    uint8_t* d_ws = nullptr;
    uint8_t* d_pyr = nullptr;      // level-major pyramids (mvImagePyramid)
    uint8_t* d_blur = nullptr;     // blurred pyramids
    size_t pyr_bytes = 0;
    uint32_t* d_cand = nullptr;    // FAST candidates, packed x|y<<12|score<<24
    uint32_t* d_sort = nullptr;    // global fallback for the quadtree sort
    uint32_t* d_lvl_kp = nullptr;  // DistributeOctTree output per level
    int* d_slot = nullptr;         // output row of every emitted keypoint
    int* d_cand_cnt = nullptr;
    int* d_lvl_cnt = nullptr;
    int* d_nkp = nullptr;          // the count table: [max_batch] n, [max_batch] mono, [max_batch+1] offsets
    int* d_mono = nullptr;
    int* d_offsets = nullptr;
    int* d_err = nullptr;
    int2* d_taps = nullptr;
    orbx_keypoint* d_kps = nullptr;  // compact results of the last batch
    uint8_t* d_desc = nullptr;
    float* d_uright = nullptr;       // Frame::mvuRight / mvDepth of the last stereo or RGB-D batch (row-aligned with d_kps)
    float* d_depth = nullptr;
    int* d_sad = nullptr;
    uint32_t* d_pat = nullptr;       // rBRIEF pattern, 256 packed pairs transposed for k_orient_describe
    uint32_t* d_blur_frag = nullptr; // k_blur_mma: the lanes' constant A fragments (bm_fragments, 8 x 32 words)
    uint8_t* d_node_scratch = nullptr;   // quadtree nodes when they do not fit shared memory (!qt_nodes_in_smem)
    uint8_t* d_stage = nullptr;
    uint8_t* d_po = nullptr;         // edge lists / results of orbo_pose_optimization_frames
    size_t stage_bytes = 0, po_bytes = 0;
    bool stereo_valid = false;   // d_uright/d_depth belong to the last extracted batch
    size_t cand_slots = 0, kp_slots = 0, sort_slots = 0, taps_slots = 0, cells_slots = 0, out_rows = 0;
    int* h_counts = nullptr;       // pinned mirror of the count table, then the capacity flags (extractor.cu queue_counts)
    bool counts_valid = false;
    int q_total_bound = 0, q_frame_bound = 0, rows_bound = 0;   // orbm_set_device_query_bounds: sync-free device-pointer searches
    bool capturing = false;   // between orbx_graph_begin and orbx_graph_end
    int batch_status = 0;   // 0 ok; 1 FAST candidate overflow, 2 quadtree node overflow of the last batch (truncated results are never served)
    int last_batch = 0;
    // quadtree launch plan: up to 4 level groups with their own shared-memory size, run on parallel
    // streams (forked from / joined into `stream`)
    struct QtGroup { int level_begin, level_end, sort_cap; size_t smem; bool k64; };   // k64: k_quadtree_v1_k64 (regions over 2048 px)
    QtGroup qt_groups[4] = {};
    int qt_max_groups = 3;   // level groups (launches) of the quadtree stage: {16384+, 8192, 2048} sort capacities; ORB_QT_GROUPS=4 adds a 4096 group
                             // (measured in round 2: 16 KB less shared memory for levels 2-4, but 0.317 instead of 0.278 ms per batch -- more
                             // co-resident CTAs contend for the same SMs' barrier / shared-memory latency)
    int qt_ngroups = 0;
    cudaStream_t aux_stream[3] = {};
    cudaEvent_t ev_fork = nullptr, ev_join[3] = {};
    int qt_node_cap = 0, qt_nodes_in_smem = 1;
    size_t qt_node_stride = 0, order_smem_bytes = 0;
    orbr_state* replay = nullptr;   // orbr_submit / orbr_collect state (replay.cu)
    uint8_t* d_xl = nullptr;        // frame blocks of the matcher's global-memory form (matcher.cu launch_proj)
    size_t xl_bytes = 0;
    uint8_t* d_src = nullptr;       // host camera images of extract_batch_source, uploaded for k_ingest
    size_t src_bytes = 0;
    uint8_t* d_dmap = nullptr;      // host depth maps of orbm_stereo_rgbd_batch, uploaded for k_stereo_rgbd
    size_t dmap_bytes = 0;
    int smem_optin = 0;             // cudaDevAttrMaxSharedMemoryPerBlockOptin of the handle's device, read on first use
};

// Rows of one searched frame or keyframe that the matchers accept: an extractor handle's row capacity (n_features + 20 x n_levels)
// or a host keyframe's feature count.  Feature ids are 16-bit (65 535 would do); the resolve state of the matcher's global-memory
// form (9 B per row next to 73 KB of query staging), k_bow_vector (8 B x the next power of two) and k_tri_match (14 B per row) fit
// one CTA's shared memory on an H100 up to this many rows and no further.
#define ORB_MAX_FRAME_ROWS 16384

inline orb_status check_frame_rows(long long rows, const char* what) {
    if (rows <= ORB_MAX_FRAME_ROWS) return ORB_OK;
    return orb::set_error(ORB_ERR_UNSUPPORTED, std::string(what) + " with " + std::to_string(rows) + " feature rows: the matchers take at most " +
                                                   std::to_string(ORB_MAX_FRAME_ROWS));
}

// What the count table of the last batch says, once orbx_counts, batch_rows or orbr_collect has read it back
inline int image_features(const orbx_handle* h, int img) { return h->h_counts[img]; }
inline int image_row0(const orbx_handle* h, int img) { return h->h_counts[2 * h->cfg.max_batch + img]; }
inline int batch_total_rows(const orbx_handle* h) { return image_row0(h, h->last_batch); }

inline int smem_optin(orbx_handle* h) {
    if (h->smem_optin == 0) cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->cfg.device);
    return h->smem_optin;
}

// A kernel's static shared memory (its __shared__ arrays), which counts against the same per-block limit as the dynamic request
template <typename... A>
inline size_t static_smem(void (*kern)(A...)) {
    cudaFuncAttributes fa{};
    return cudaFuncGetAttributes(&fa, kern) == cudaSuccess ? fa.sharedSizeBytes : 0;
}

// A kernel whose dynamic shared memory grows with the frame is refused, before anything is launched, when the device cannot give it
// that much next to its static arrays: ORB_ERR_UNSUPPORTED with a message rather than a failed launch.
inline orb_status check_smem(orbx_handle* h, size_t bytes, size_t static_bytes, const char* kernel) {
    if (bytes + static_bytes <= (size_t)smem_optin(h)) return ORB_OK;
    return orb::set_error(ORB_ERR_UNSUPPORTED, std::string(kernel) + " needs " + std::to_string(bytes + static_bytes) +
                                                   " B of shared memory per block; the device allows " + std::to_string(smem_optin(h)));
}
