/* orbslam3_b200.h -- C ABI of liborbslam3_b200.so: the H100 (sm_90a) implementation of ORB-SLAM3's
 * per-frame data-parallel hot path.  Plain pointers and sizes only; every function returns an
 * orb_status (0 = ok, <0 = error) and never throws.  The caller owns all host buffers; the library owns
 * device memory per handle; one CUDA stream per handle; thread-safe across handles, not within one.
 *
 * The reference has no FFI layer: its boundary is the C++ member functions cited below.  The C++
 * shims in orb_slam3_detailed_comments_b200/host/ keep those signatures and marshal onto this ABI
 * (see INTEGRATION.md).
 */
#ifndef ORBSLAM3_B200_H
#define ORBSLAM3_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    ORB_OK = 0,
    ORB_ERR_INVALID = -1,      /* bad argument (null pointer, size out of range) */
    ORB_ERR_EMPTY = -2,        /* empty image: ORBextractor::operator() returns -1 (ORBextractor.cc:1561) */
    ORB_ERR_CUDA = -3,         /* CUDA runtime error; orb_last_error() has the text */
    ORB_ERR_CAPACITY = -4,     /* output or internal capacity exceeded */
    ORB_ERR_UNSUPPORTED = -5,  /* geometry the reference cannot process either (nIni == 0), an image side > 4128 px, a searched frame
                                  or keyframe of more than 16 384 feature rows, or a frame-sized shared-memory need above the device's */
    ORB_ERR_NO_DEVICE = -6     /* no CUDA device: there is NO CPU fallback */
} orb_status;

const char* orb_last_error(void);
int orb_device_count(void);

/* ------------------------------------------------------------------------------------------------
 * ORBextractor  (include/ORBextractor.h:43-109, src/ORBextractor.cc)
 * ---------------------------------------------------------------------------------------------- */

/* bit-compatible with cv::KeyPoint (28 bytes) */
typedef struct {
    float x, y;      /* pt, level-0 pixel coordinates (pt *= scale[octave], ORBextractor.cc:1662) */
    float size;      /* (int)(31 * scale[octave]) */
    float angle;     /* IC_Angle, degrees [0,360) */
    float response;  /* FAST score */
    int32_t octave;
    int32_t class_id; /* -1 */
} orbx_keypoint;

typedef struct {
    int32_t n_features;    /* ORBextractor ctor args, ORBextractor.h:49-50 */
    float scale_factor;
    int32_t n_levels;
    int32_t ini_th_fast;
    int32_t min_th_fast;
    int32_t max_width;     /* largest image this handle will see */
    int32_t max_height;
    int32_t max_batch;     /* images per orbx_extract_batch call (a stereo pair is 2 images) */
    int32_t device;        /* CUDA ordinal */
} orbx_config;

typedef struct orbx_handle orbx_handle;

/* replaces ORBextractor::ORBextractor (src/ORBextractor.cc:468-571) */
orb_status orbx_create(const orbx_config* cfg, orbx_handle** out);
void orbx_destroy(orbx_handle* h);

/* GetScaleFactors / GetInverseScaleFactors / GetScaleSigmaSquares / GetInverseScaleSigmaSquares and
 * mnFeaturesPerLevel / umax (ORBextractor.h:61-81,97-108).  Each array holds n_levels entries
 * (umax: 16).  Any pointer may be NULL. */
orb_status orbx_get_tables(const orbx_handle* h, float* scale, float* inv_scale, float* sigma2,
                           float* inv_sigma2, int32_t* features_per_level, int32_t* umax16);

/* replaces ORBextractor::operator() (src/ORBextractor.cc:1557-1682) for ONE host image.
 * lap0/lap1 = vLappingArea.  Writes min(n, cap) keypoints + 32-byte descriptors; *n_out = n;
 * *mono_index = the reference's return value.  Returns ORB_ERR_EMPTY for an empty image. */
orb_status orbx_extract(orbx_handle* h, const uint8_t* img, int32_t width, int32_t height, int32_t stride,
                        int32_t lap0, int32_t lap1, orbx_keypoint* kps, uint8_t* desc, int32_t cap,
                        int32_t* n_out, int32_t* mono_index);

/* Batched form: `batch` images of identical size, image b at imgs + b*image_stride_bytes (host memory,
 * pinned preferred).  Results stay ON THE DEVICE inside the handle (keypoints, descriptors, the
 * pyramids and blurred pyramids of every image) for the stereo matcher / search kernels; fetch them
 * with orbx_download.  n_out / mono_index (host, `batch` entries) may be NULL. */
orb_status orbx_extract_batch(orbx_handle* h, const uint8_t* imgs, int32_t batch, int32_t width,
                              int32_t height, int32_t stride, size_t image_stride_bytes, int32_t lap0,
                              int32_t lap1, int32_t* n_out, int32_t* mono_index);

/* Same, images already resident in device memory (no H2D inside): the `value` leg of bench.py. */
orb_status orbx_extract_batch_device(orbx_handle* h, const uint8_t* d_imgs, int32_t batch, int32_t width,
                                     int32_t height, int32_t stride, size_t image_stride_bytes,
                                     int32_t lap0, int32_t lap1);

/* Pixel layout of a camera image: 8-bit channels, interleaved.  The colour formats are converted to grey as
 * Tracking::GrabImageStereo / GrabImageMonocular do (Tracking.cc:1523-1601: cv::cvtColor with COLOR_RGB2GRAY / COLOR_BGR2GRAY
 * for 3 channels, COLOR_RGBA2GRAY / COLOR_BGRA2GRAY for 4, chosen by mbRGB); alpha is ignored. */
typedef enum {
    ORB_FORMAT_GRAY = 0,
    ORB_FORMAT_RGB = 1,
    ORB_FORMAT_BGR = 2,
    ORB_FORMAT_RGBA = 3,
    ORB_FORMAT_BGRA = 4
} orb_image_format;

/* orbx_extract_batch_device for camera images of any orb_image_format and size: d_imgs holds `batch` images of
 * src_width x src_height pixels in `format`, rows `stride` bytes apart, images image_stride_bytes apart (device memory).  Each is
 * resized to width x height first when the sizes differ (System::TrackStereo / TrackMonocular's cv::resize(INTER_LINEAR) to
 * Settings::newImSize, System.cc:286-298), channel by channel, then converted to grey, in the reference's order; the result is
 * level 0 of the image's pyramid.  Keypoints are in the coordinates of the width x height image.  width / height are bounded by the
 * handle's max_width / max_height, the source by nothing but memory.  src_width = src_height = 0 means width x height (no resize).
 * Queues everything on the handle's stream with no synchronisation (graph capture works once the size has run eagerly); refuses an
 * unknown format, a stride below src_width x channels or a size the handle cannot hold with ORB_ERR_INVALID before queuing. */
orb_status orbx_extract_batch_device_format(orbx_handle* h, const uint8_t* d_imgs, int32_t batch, int32_t width, int32_t height,
                                            int32_t stride, size_t image_stride_bytes, int32_t lap0, int32_t lap1,
                                            int32_t format, int32_t src_width, int32_t src_height);

/* Counts of the last batch: n[b] keypoints, mono_index[b]; offsets[b] = first row of image b in the
 * compact result arrays (offsets has batch+1 entries).  Synchronises the handle's stream. */
/* upper bound of the keypoints of one image (row stride of per-image outputs such as orbv_transform's BowVector) */
int32_t orbx_max_features(const orbx_handle* h);
orb_status orbx_counts(orbx_handle* h, int32_t* n, int32_t* mono_index, int32_t* offsets);

/* Copies the compact results of the last batch to the host: kps/desc hold offsets[batch] rows. */
orb_status orbx_download(orbx_handle* h, orbx_keypoint* kps, uint8_t* desc, int32_t cap_rows);

/* mvImagePyramid[level] of image b (ORBextractor.h:83): copies the ROI (no border) into dst with
 * row stride dst_stride; blurred != 0 returns the GaussianBlur'ed working copy (ORBextractor.cc:1632). */
orb_status orbx_level_size(const orbx_handle* h, int32_t level, int32_t* width, int32_t* height);
orb_status orbx_download_level(orbx_handle* h, int32_t b, int32_t level, int32_t blurred, uint8_t* dst,
                               int32_t dst_stride);
/* All n_levels of image b at once (what a host-side mvImagePyramid needs after operator()): dst[l] / dst_stride[l] per
 * level, every copy queued on the handle's stream and ONE synchronisation at the end (orbx_download_level syncs per call). */
orb_status orbx_download_pyramid(orbx_handle* h, int32_t b, int32_t blurred, uint8_t* const* dst, const int32_t* dst_stride);

/* Stage outputs of the last batch, for stage-wise parity tests.
 * candidates: FAST keypoints entering DistributeOctTree (ORBextractor.cc:1159-1165), sorted in the
 * reference order; each row = x, y (relative to minBorder), score.  level keypoints: the output of
 * DistributeOctTree in list order; each row = x, y (level pixel coords), score. */
orb_status orbx_download_candidates(orbx_handle* h, int32_t b, int32_t level, int32_t* xys, int32_t cap,
                                    int32_t* n_out);
orb_status orbx_download_level_keypoints(orbx_handle* h, int32_t b, int32_t level, int32_t* xys,
                                         int32_t cap, int32_t* n_out);

/* Timing of the last batch with CUDA events on the handle's stream (milliseconds):
 * [0] total, [1] pyramid, [2] FAST, [3] quadtree, [4] blur, [5] orientation+descriptors, [6] H2D.
 * Averages over the batches run since orbx_set_profiling(h, 1) (ring of the last 32). */
orb_status orbx_set_profiling(orbx_handle* h, int32_t on);
orb_status orbx_last_timings(orbx_handle* h, float* ms7);
/* the handle's cudaStream_t (for CUDA-event timing on the launching stream) */
void* orbx_cuda_stream(orbx_handle* h);

/* CUDA-graph replay of a step.  Everything the caller queues on the handle's stream between begin and end -- the device-pointer
 * entry points: orbx_extract_batch_device, orbm_stereo_batch, the on_device searches under orbm_set_device_query_bounds,
 * orbo_pose_* with on_device -- is captured instead of executed; orbx_graph_launch replays it with one launch.  Captured calls
 * must not synchronise or allocate: run the same step once eagerly first (it sizes every scratch buffer).  Pointers are baked
 * in: a replay reads the same input buffers and writes the same outputs, with whatever contents they hold then. */
typedef struct orbx_graph orbx_graph;
orb_status orbx_graph_begin(orbx_handle* h);
orb_status orbx_graph_end(orbx_handle* h, orbx_graph** out);
orb_status orbx_graph_launch(orbx_handle* h, orbx_graph* g);
int32_t orbx_graph_kernels(const orbx_graph* g);   /* kernel nodes per replay */
void orbx_graph_destroy(orbx_graph* g);
/* kernels launched by this library since load (bench.py's gpu_launches) */
int64_t orb_kernel_launches(void);

/* ------------------------------------------------------------------------------------------------
 * Frame::ComputeStereoMatches  (src/Frame.cc:1102-1358)
 * ---------------------------------------------------------------------------------------------- */

/* Stereo matching of the last extracted batch of ONE handle holding interleaved eyes: left = image 2p,
 * right = image 2p+1, p < n_pairs.  bf = Frame::mbf, b = Frame::mb.  Results (mvuRight / mvDepth, -1 =
 * no match) stay on the device, row-aligned with the compact keypoint rows; right-eye rows are unused. */
orb_status orbm_stereo_batch(orbx_handle* h, int32_t n_pairs, float bf, float b);
orb_status orbm_stereo_download(orbx_handle* h, float* uright, float* depth, int32_t cap_rows);

/* The reference's own arrangement: two extractor objects (mpORBextractorLeft / Right, Frame.cc:136-141),
 * image 0 of each.  Writes mvuRight / mvDepth of the N left keypoints to host arrays. */
orb_status orbm_stereo_pair(orbx_handle* left, orbx_handle* right, float bf, float b, float* uright,
                            float* depth, int32_t cap);

/* ------------------------------------------------------------------------------------------------
 * Frame::ComputeStereoFromRGBD: mvuRight / mvDepth of an RGB-D frame from its registered depth map
 * ---------------------------------------------------------------------------------------------- */

/* Element type of a depth map: 16-bit unsigned raw sensor units (CV_16U), or 32-bit float (CV_32F). */
typedef enum { ORB_DEPTH_U16 = 1, ORB_DEPTH_F32 = 2 } orb_depth_format;

/* Image b < n_images of the last extracted batch is an RGB-D frame (extracted with vLappingArea = {0, 0}); its depth map, of the extracted
 * width x height, is at depth + b * image_stride_bytes, rows stride_bytes apart (0 = tight rows / images).  Per keypoint, as the
 * reference does for a camera with zero distortion (mvKeysUn = mvKeys):
 *   Tracking::GrabImageRGBD: d = raw * depth_factor (one float rounding) unless the map is F32 and |depth_factor - 1| <= 1e-5, in which
 *     case d = raw; depth_factor is Tracking::mDepthMapFactor, the multiplier (1 / the settings' DepthMapFactor);
 *   Frame::ComputeStereoFromRGBD: d sampled at ((int)y, (int)x); d > 0: mvDepth = d, mvuRight = x - bf / d; else both -1.
 * Only the sampled pixels are converted.  Results stay on the device, row-aligned with the compact keypoint rows, and are what the
 * searches, orbo_pose_edges and orbx_pack_keyframe_device read next; orbm_stereo_download returns them; rows of images >= n_images
 * are not written.  on_device != 0: `depth` is device memory and the call queues one kernel, with no synchronisation or allocation
 * (graph capture works).  on_device == 0: host memory, copied into a buffer of the handle on its stream (the memory must stay
 * unchanged until the copy has run, as for orbx_extract_batch).  Refuses with ORB_ERR_INVALID, before queuing anything, a null
 * handle or map, n_images outside [1, last batch], an unknown format, or a stride shorter than a row (an image stride shorter than
 * an image) or not a multiple of the element size. */
orb_status orbm_stereo_rgbd_batch(orbx_handle* h, int32_t n_images, const void* depth, int32_t depth_format, int32_t stride_bytes,
                                  size_t image_stride_bytes, float depth_factor, int32_t on_device, float bf);

/* ------------------------------------------------------------------------------------------------
 * ORBmatcher::SearchByProjection family  (include/ORBmatcher.h:40-87, src/ORBmatcher.cc), Nleft == -1
 *
 * The frame whose features are searched is an image of the extractor handle's last batch (for a stereo
 * batch: the LEFT image 2p; its mvuRight comes from orbm_stereo_batch or orbm_stereo_rgbd_batch when one ran, else -1).  Several
 * frames are processed per call; frame f uses queries [query_offset[f], query_offset[f+1]).
 * on_device != 0: every array pointer of the query struct and the output pointers are DEVICE memory and
 * the call does not synchronise (except for reading the two small offset tables).
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    float fx, fy, cx, cy, bf, b;          /* Frame::fx.., mbf, mb */
    float min_x, max_x, min_y, max_y;     /* Frame::mnMinX, mnMaxX, mnMinY, mnMaxY (image bounds when rectified) */
} orbm_camera;

/* Device-pointer searches (on_device != 0) normally read the two small offset tables and the batch's row count back to size
 * their launches -- two synchronisations per call.  With bounds set (> 0) they read nothing back: total_queries bounds
 * query_offset[n_frames], max_queries_per_frame every frame's query count, total_rows the batch's compact keypoint rows (the
 * length of the caller's per-row output arrays; clamped to max_batch * orbx_max_features).  The kernels take the real counts from the device tables, so
 * results are unchanged; the calls become pure kernel launches (capturable, orbx_graph_begin).  0, 0, 0 restores the default. */
orb_status orbm_set_device_query_bounds(orbx_handle* h, int32_t total_queries, int32_t max_queries_per_frame, int32_t total_rows);

/* SearchByProjection(Frame&, const vector<MapPoint*>&, th, bFarPoints, thFarPoints)  ORBmatcher.cc:45-239.
 * One entry per map point with mbTrackInView, in vpMapPoints order, carrying the fields Frame::isInFrustum
 * wrote into it (MapPoint.h: mTrackProjX, mTrackProjY, mTrackProjXR, mnTrackScaleLevel, mTrackViewCos,
 * mTrackDepth) and MapPoint::GetDescriptor().  Local map points always have Observations() > 0. */
typedef struct {
    int32_t n_frames;
    int32_t on_device;
    const int32_t* frame_image;   /* [n_frames] image index in the last batch */
    const int32_t* query_offset;  /* [n_frames + 1] */
    const float* proj_x;
    const float* proj_y;
    const float* proj_xr;
    const int32_t* level;
    const float* view_cos;
    const float* track_depth;     /* may be NULL unless far_points */
    const uint8_t* desc;          /* 32 bytes per query */
    const uint8_t* feature_claimed; /* per compact keypoint row of the batch: F.mvpMapPoints[idx] already holds a
                                       map point with Observations() > 0; NULL = none */
    const uint8_t* in_view;       /* pMP->mbTrackInView per entry (orbf_is_in_frustum output): entries with 0 are skipped
                                     like ORBmatcher.cc:52-53 and get match -1; NULL = every entry is in view */
} orbm_local_queries;

/* match_out[q] = feature index inside its frame (F.mvpMapPoints[bestIdx] = pMP) or -1;
 * nmatches_out[f] = the reference's return value for frame f (may be NULL). */
orb_status orbm_search_local_points(orbx_handle* h, const orbm_camera* cam, const orbm_local_queries* q, float th,
                                    float nnratio, int32_t far_points, float th_far, int32_t* match_out,
                                    int32_t* nmatches_out);

/* Frame::isInFrustum(MapPoint*, viewingCosLimit)  src/Frame.cc:667-720, Nleft == -1 (Tracking::SearchLocalPoints,
 * Tracking.cc:4022).  Frame f tests points [point_offset[f], point_offset[f+1]) -- mvpLocalMapPoints after the caller-side
 * skips (already matched in this frame, isBad) -- against its pose members mRcw (row-major), mtcw, mOw
 * (Frame::UpdatePoseMatrices).  Outputs per point are the MapPoint fields the search reads: mbTrackInView, mTrackProjX,
 * mTrackProjY, mTrackProjXR, mnTrackScaleLevel, mTrackViewCos, mTrackDepth; they plug into orbm_local_queries (with
 * in_view) without compaction.  on_device != 0: all arrays are device memory, n_points_max bounds point_offset[n_frames],
 * no synchronisation. */
typedef struct {
    int32_t n_frames;
    int32_t on_device;
    const int32_t* point_offset;  /* [n_frames + 1] */
    const float* Rcw;             /* [n_frames][9] */
    const float* tcw;             /* [n_frames][3] */
    const float* Ow;              /* [n_frames][3] */
    const float* world_pos;       /* [np][3] */
    const float* normal;          /* [np][3] MapPoint::GetNormal */
    const float* max_dist;        /* MapPoint::mfMaxDistance, the RAW member (orbp_update_normal_and_depth's output): the distance gate applies
                                     GetMaxDistanceInvariance's 1.2f itself, PredictScale divides the raw value (MapPoint.cc:658-721) */
    const float* min_dist;        /* MapPoint::mfMinDistance, raw (the gate applies 0.8f) */
    int32_t n_points_max;         /* device callers: grid bound; else ignored */
} orbf_frustum_points;

orb_status orbf_is_in_frustum(orbx_handle* h, const orbm_camera* cam, const orbf_frustum_points* in, float viewing_cos_limit,
                              uint8_t* in_view_out, float* proj_x_out, float* proj_y_out, float* proj_xr_out, int32_t* level_out,
                              float* view_cos_out, float* track_depth_out);

/* SearchByProjection(Frame& CurrentFrame, const Frame& LastFrame, th, bMono)  ORBmatcher.cc:1950-2184.
 * One entry per LastFrame feature that has a map point and is not an outlier, in LastFrame order.
 * direction[f]: 0 = neither, 1 = bForward, 2 = bBackward (tlc.z vs mb, ORBmatcher.cc:1967-1971; computed
 * by the caller from the two poses exactly as the reference does).  Tcw: qx qy qz qw tx ty tz (Sophus::SE3f).
 * CurrentFrame.mvpMapPoints must be all-NULL on entry (Tracking.cc:3367). */
typedef struct {
    int32_t n_frames;
    int32_t on_device;
    const int32_t* frame_image;
    const int32_t* query_offset;
    const float* Tcw;             /* [n_frames][7] */
    const int32_t* direction;     /* [n_frames] */
    const float* world_pos;       /* [nq][3] MapPoint::GetWorldPos */
    const int32_t* last_octave;   /* LastFrame.mvKeys[i].octave */
    const float* last_angle;      /* LastFrame.mvKeysUn[i].angle */
    const uint8_t* desc;          /* MapPoint::GetDescriptor */
    const uint8_t* obs_positive;  /* pMP->Observations() > 0 */
} orbm_last_queries;

/* feature_match_out: one entry per compact keypoint row of the whole batch: the query index now held by
 * CurrentFrame.mvpMapPoints[idx], or -1.  nmatches_out[f] = the reference's return value. */
orb_status orbm_search_last_frame(orbx_handle* h, const orbm_camera* cam, const orbm_last_queries* q, float th,
                                  int32_t check_orientation, int32_t* feature_match_out, int32_t* nmatches_out);

/* SearchByBoW(KeyFrame* pKF, Frame& F, vector<MapPoint*>& vpMapPointMatches)  ORBmatcher.cc:259-493, Nleft == -1.
 * One entry per keyframe feature that holds a good map point, in the order of the FeatureVector merge join
 * (ascending vocabulary node id, ascending keyframe feature index inside a node).  feature_node: vocabulary node
 * of every frame feature (F.mFeatVec from Frame::ComputeBoW, the level-4 ancestor), one entry per compact keypoint
 * row of the batch, -1 = none.  Output as orbm_search_last_frame (query index per feature row, or -1). */
typedef struct {
    int32_t n_frames;
    int32_t on_device;
    const int32_t* frame_image;
    const int32_t* query_offset;
    const int32_t* query_node;    /* vocabulary node of the keyframe feature */
    const float* query_angle;     /* pKF->mvKeysUn[idx].angle */
    const uint8_t* desc;          /* pKF->mDescriptors.row(idx) */
    const int32_t* feature_node;
} orbm_bow_queries;

orb_status orbm_search_bow(orbx_handle* h, const orbm_bow_queries* q, float nnratio, int32_t check_orientation,
                           int32_t* feature_match_out, int32_t* nmatches_out);

/* SearchForInitialization(Frame& F1, Frame& F2, vector<cv::Point2f>& vbPrevMatched, vector<int>& vnMatches12, int windowSize)
 * ORBmatcher.cc:734-890 (monocular initialisation, Tracking.cc:2588).  F1 (the reference frame) is host memory: all its
 * mvKeysUn / descriptors (features with octave > 0 are skipped by the search itself); F2 is host memory (kp2 != NULL) or
 * image target_image of the handle's last batch.  prev_matched = vbPrevMatched (x, y per F1 feature).
 * matches12_out[i1] = F2 feature index or -1 (vnMatches12); the caller refreshes vbPrevMatched from it (:880-884). */
typedef struct {
    int32_t n1;
    const orbx_keypoint* kp1;
    const uint8_t* desc1;
    const float* prev_matched;    /* [n1][2] */
    int32_t n2;                   /* host F2 */
    const orbx_keypoint* kp2;
    const uint8_t* desc2;
    int32_t target_image;         /* device F2 when kp2 == NULL */
} orbm_init_queries;

orb_status orbm_search_initialization(orbx_handle* h, const orbm_camera* cam, const orbm_init_queries* q, int32_t window_size,
                                      float nnratio, int32_t check_orientation, int32_t* matches12_out, int32_t* nmatches_out);

/* SearchByBoW(KeyFrame* pKF1, KeyFrame* pKF2, vector<MapPoint*>& vpMatches12)  ORBmatcher.cc:892-1043, single-camera
 * keyframes (loop closing / place recognition).  Both keyframes are map state in host memory; several (pKF1, pKF2) pairs
 * per call.  Queries = the KF1 features that hold a good map point, in FeatureVector merge order (ascending node,
 * ascending feature index inside a node); side 2 = all features of KF2 with node2[i] = vocabulary node (-1 = not in
 * mFeatVec) and valid2[i] = holds a good map point.  match12_out[q] = KF2 feature index (vpMatches12[idx1] =
 * vpMapPoints2[idx2]) or -1; nmatches_out[pair] = the reference's return value. */
typedef struct {
    int32_t n_pairs;
    const int32_t* feat_offset;   /* [n_pairs + 1] keyframe-2 features of every pair back to back */
    const orbx_keypoint* kp2;     /* mvKeysUn (angle is read) */
    const uint8_t* desc2;
    const int32_t* node2;
    const uint8_t* valid2;        /* NULL = all */
    const int32_t* query_offset;  /* [n_pairs + 1] */
    const int32_t* query_node;
    const float* query_angle;     /* pKF1->mvKeysUn[idx1].angle */
    const uint8_t* desc1;
} orbm_bow_kf_queries;

orb_status orbm_search_bow_keyframes(orbx_handle* h, const orbm_bow_kf_queries* q, float nnratio, int32_t check_orientation,
                                     int32_t* match12_out, int32_t* nmatches_out);

/* Projection searches into a KeyFrame from a pose (Nleft == -1, pinhole):
 *   ORBM_KF_FUSE_POSE   Fuse(pKF, vpMapPoints, th, bRight=false)                           ORBmatcher.cc:1325-1544
 *   ORBM_KF_FUSE_SIM3   Fuse(pKF, Scw, vpPoints, th, vpReplacePoint)                       ORBmatcher.cc:1546-1687
 *   ORBM_KF_PROJ_SIM3   SearchByProjection(pKF, Scw, vpPoints, vpMatched, th, ratioHamming) ORBmatcher.cc:495-618 and the
 *                       vpPointsKFs / vpMatchedKF overload :620-732 (same search; the caller records the extra array)
 *   ORBM_KF_PROJ_RELOC  SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist)   ORBmatcher.cc:2196-2330
 *   ORBM_KF_SIM3_ONEWAY one direction of SearchBySim3(pKF1, pKF2, vpMatches12, S12, th)     ORBmatcher.cc:1689-1948:
 *                       the map points of keyframe A (good, not already matched) into keyframe B through
 *                       p_B = S_BA * (T_Aw * p_w); the caller runs both directions (two targets of one call) and keeps
 *                       the pairs that agree (:1930-1945).  Tcw = T_Aw, Sim3 = S_BA, Ow unused.
 * Several targets per call (LocalMapping::SearchInNeighbors fuses the same points into ~20 keyframes): target t
 * searches features [feat_offset[t], feat_offset[t+1]) with queries [query_offset[t], query_offset[t+1]).
 * Targets are map state in HOST memory (kp != NULL), or -- kp == NULL -- images target_image[t] of the handle's
 * last batch (the frame being relocalised is still on the device).
 * Queries = the map points that survive the caller-side skips (NULL, isBad(), IsInKeyFrame / spAlreadyFound /
 * sAlreadyFound), in the reference's order.  Tcw: qx qy qz qw tx ty tz of the SE3f the function uses (for the Sim3
 * variants SE3f(Scw.rotationMatrix(), Scw.translation()/Scw.scale())); Ow = pKF->GetCameraCenter() /
 * Tcw.inverse().translation().  The level tables (mvScaleFactors, mvInvLevelSigma2, mnScaleLevels,
 * mfLogScaleFactor = logf(scaleFactor)) are the handle's.
 * match_out[q] = feature index inside its target (bestIdx) or -1; the caller applies the side effects in query
 * order (Replace / AddObservation / vpReplacePoint / vpMatched[bestIdx] = pMP).  nmatches_out[t] = return value. */
enum { ORBM_KF_FUSE_POSE = 0, ORBM_KF_FUSE_SIM3 = 1, ORBM_KF_PROJ_SIM3 = 2, ORBM_KF_PROJ_RELOC = 3, ORBM_KF_SIM3_ONEWAY = 4 };
typedef struct {
    int32_t n_targets;
    const int32_t* target_image;  /* [n_targets] when kp == NULL, else ignored */
    const int32_t* feat_offset;   /* [n_targets + 1] when kp != NULL */
    const orbx_keypoint* kp;      /* mvKeysUn */
    const uint8_t* desc;          /* mDescriptors */
    const float* uright;          /* mvuRight (FUSE_POSE reads it; NULL = monocular) */
    const uint8_t* feat_claimed;  /* PROJ_SIM3: vpMatched[idx] != NULL, PROJ_RELOC: mvpMapPoints[i2] != NULL on entry
                                     (per feature row, host targets: same indexing as kp; device targets: compact rows); NULL = none */
    const float* Tcw;             /* [n_targets][7] */
    const float* Ow;              /* [n_targets][3] */
    const float* Sim3;            /* SIM3_ONEWAY: [n_targets][8] quaternion x y z w (non-unit, RxSO3), translation, and
                                     scale = rxso3().quaternion().squaredNorm() as the caller's Eigen evaluates it; else NULL */
    const int32_t* query_offset;  /* [n_targets + 1] */
    const float* world_pos;       /* [nq][3] MapPoint::GetWorldPos */
    const float* normal;          /* [nq][3] MapPoint::GetNormal (unused by PROJ_RELOC, may be NULL there) */
    const float* max_dist;        /* MapPoint::mfMaxDistance, the RAW member (orbp_update_normal_and_depth's output): the distance gate applies
                                     GetMaxDistanceInvariance's 1.2f itself, PredictScale divides the raw value (MapPoint.cc:658-721) */
    const float* min_dist;        /* MapPoint::mfMinDistance, raw (the gate applies 0.8f) */
    const uint8_t* desc_q;        /* MapPoint::GetDescriptor */
    const float* angle;           /* PROJ_RELOC: pKF->mvKeysUn[i].angle of the query's keyframe feature; else NULL */
} orbm_kf_queries;

/* hamming_max: TH_LOW (50), TH_LOW * ratioHamming, ORBdist, or TH_HIGH (100) for SIM3_ONEWAY. */
orb_status orbm_search_keyframe(orbx_handle* h, const orbm_camera* cam, const orbm_kf_queries* q, int32_t variant,
                                float th, float hamming_max, int32_t check_orientation, int32_t* match_out,
                                int32_t* nmatches_out);

/* SearchForTriangulation(KeyFrame* pKF1, KeyFrame* pKF2, vMatchedPairs, bOnlyStereo, bCoarse)  ORBmatcher.cc:1045-1323,
 * keyframes without a second camera.  Both keyframes are map state (host memory): queries = the KF1 features WITHOUT
 * a map point (and stereo when bOnlyStereo), in FeatureVector merge order; side 2 = all features of KF2 with
 * valid2[i] = no map point (and stereo when bOnlyStereo).  F12 = K1^-T [t12]x R12 K2^-1 (row-major, float) and the
 * epipole of camera 1 in image 2 are computed by the caller exactly as the reference does (ORBmatcher.cc:1056-1073,
 * Pinhole.cpp:190-193).  The handle only lends its stream, staging memory and scale tables.
 * match12_out[q] = KF2 feature index or -1 (the caller emits the (idx1, idx2) pairs in ascending idx1). */
typedef struct {
    int32_t n_queries, n2;
    const orbx_keypoint* kp1;     /* mvKeysUn of the query features */
    const uint8_t* desc1;
    const int32_t* node1;
    const uint8_t* stereo1;       /* mvuRight[idx1] >= 0 */
    const orbx_keypoint* kp2;
    const uint8_t* desc2;
    const int32_t* node2;         /* -1 = not in mFeatVec */
    const uint8_t* valid2;
    const uint8_t* stereo2;
    float F12[9];
    float epipole2[2];
    int32_t coarse;               /* bCoarse: skip the epipolar-line test */
    int32_t check_orientation;
} orbm_triangulation;

orb_status orbm_search_triangulation(orbx_handle* h, const orbm_triangulation* t, int32_t* match12_out,
                                     int32_t* nmatches_out);

/* ------------------------------------------------------------------------------------------------
 * cv::BFMatcher(cv::NORM_HAMMING).knnMatch(query, train, matches, 2) -- the brute-force 256-bit Hamming search of
 * Frame::ComputeStereoFishEyeMatches (src/Frame.cc:1553; BFmatcher is a member of Frame, include/Frame.h), batched over independent
 * (query, train) descriptor sets: pair p owns query rows [query_offset[p], query_offset[p+1]) and train rows likewise.
 * idx_out / dist_out: [query rows][2] = trainIdx / distance of the nearest and second nearest train row of the SAME pair, ascending
 * distance, ties by ascending trainIdx (OpenCV's order); -1 where the train set has fewer than 1 / 2 rows (knnMatch then returns a
 * shorter list).  The caller applies the reference's ratio test `m[0].distance < m[1].distance * 0.7` (Frame.cc:1560).
 * Oracle pinned against cv2's BFMatcher; GPU parity in tests/test_zz_knn_gpu.py.
 * ---------------------------------------------------------------------------------------------- */
orb_status orbm_hamming_knn2(orbx_handle* h, int32_t n_pairs, const int32_t* query_offset, const uint8_t* query_desc,
                             const int32_t* train_offset, const uint8_t* train_desc, int32_t* idx_out, int32_t* dist_out);

/* ------------------------------------------------------------------------------------------------
 * Optimizer::LocalBundleAdjustment  (include/Optimizer.h:59, src/Optimizer.cc:1740-2188)
 *
 * The C++ shim walks the covisibility graph exactly as the reference does (Optimizer.cc:1744-1855), flattens
 * the local window into this structure, and applies the result (outlier erasure, pose / point write-back,
 * Optimizer.cc:2102-2187).  The device runs what `optimizer.optimize(10)` runs: g2o Levenberg-Marquardt over
 * BlockSolver_6_3 with Huber kernels, all in fp64.
 * Known deviation (DESIGN.md section 2, part 7): the stereo edges' `const float invz = 1.0f/z` (types_six_dof_expmap.cpp:191, :340) is
 * evaluated here and in orbo_pose_optimization as 1.0f / float(z) with `bf * invz` in double; the reference rounds the DOUBLE quotient to
 * float and, in the binary edge, multiplies bf * invz in float.  Poses differ by < 1e-6, far map points by up to 8e-5 m.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n_kf, n_mp, n_edges;
    const double* pose;        /* [n_kf][7]  qx qy qz qw tx ty tz  (g2o::SE3Quat of Tcw), local + fixed keyframes */
    const uint8_t* fixed;      /* [n_kf]     1 = setFixed(true) (lFixedCameras and the map's initial keyframe) */
    const double* point;       /* [n_mp][3]  MapPoint::GetWorldPos */
    const int32_t* edge_kf;    /* [n_edges]  index into pose[] */
    const int32_t* edge_mp;    /* [n_edges]  index into point[] */
    const double* obs;         /* [n_edges][3] kpUn.pt.x, kpUn.pt.y, mvuRight (< 0 => monocular EdgeSE3ProjectXYZ) */
    const double* inv_sigma2;  /* [n_edges]  mvInvLevelSigma2[octave]: information = inv_sigma2 * I */
    double fx, fy, cx, cy, bf; /* float members of KeyFrame promoted to double (Optimizer.cc:2038-2042) */
    double lambda_init;        /* 100 when pMap->IsInertial() (Optimizer.cc:1867-1868), else 0 = auto */
    int32_t max_iters;         /* 10 */
} lba_problem;

typedef struct {
    double* pose;                  /* [n_kf][7] optimised (fixed ones unchanged) */
    double* point;                 /* [n_mp][3] */
    double* edge_chi2;             /* [n_edges] e->chi2() as left by the LAST computeActiveErrors (may be NULL) */
    uint8_t* edge_depth_positive;  /* [n_edges] e->isDepthPositive() at the final estimate (may be NULL) */
    int32_t iterations;            /* outer Levenberg iterations run */
    int32_t trials;                /* inner trials (solve calls) */
    double lambda, chi2, chi2_initial;
} lba_result;

typedef struct lba_handle lba_handle;
orb_status lba_create(int32_t device, lba_handle** out);
void lba_destroy(lba_handle* h);
/* stop_flag mirrors `bool* pbStopFlag` (polled between LM trials; may be NULL). */
orb_status lba_solve(lba_handle* h, const lba_problem* in, lba_result* out, const volatile int32_t* stop_flag);
/* The same with the reference's own flag type: stop_flag points at the one-byte C++ `bool` that LocalMapping::InterruptBA sets
 * (Optimizer.h:59 `bool* pbStopFlag`). */
orb_status lba_solve_bool(lba_handle* h, const lba_problem* in, lba_result* out, const volatile uint8_t* stop_flag);
/* independent problems, one CTA each (sequence-sharded replay: one local BA per sequence) */
orb_status lba_solve_batch(lba_handle* h, int32_t n_problems, const lba_problem* in, lba_result* out,
                           const volatile int32_t* stop_flag);

/* ------------------------------------------------------------------------------------------------
 * Optimizer::PoseOptimization(Frame*)  (include/Optimizer.h:48, src/Optimizer.cc:55-412), Nleft == -1
 *
 * The tracking thread calls it after every projection search (Tracking.cc:3222, 3443, 3522).  Several frames per call
 * (sequence-sharded replay); frame f owns edges [edge_offset[f], edge_offset[f+1]): one per feature i with
 * pFrame->mvpMapPoints[i] != NULL, in feature order -- world_pos = pMP->GetWorldPos(), obs = kpUn.pt.x, kpUn.pt.y,
 * mvuRight[i] (< 0 => monocular EdgeSE3ProjectXYZOnlyPose, else EdgeStereoSE3ProjectXYZOnlyPose), inv_sigma2 =
 * mvInvLevelSigma2[kpUn.octave].  pose = pFrame->GetPose() (qx qy qz qw tx ty tz).  All arithmetic in fp64 like g2o.
 * pose_out[f] = SE3quat_recov (the caller casts to float and calls SetPose); outlier_out[e] = pFrame->mvbOutlier of the
 * edge's feature; inliers_out[f] = the return value nInitialCorrespondences - nBad (0 and an unchanged pose when a frame
 * has fewer than 3 correspondences).  stats_out (may be NULL): rounds, LM iterations, LM trials, 0 per frame.
 * on_device != 0: every array (inputs and outputs) is device memory and the call does not synchronise. */
typedef struct {
    int32_t n_frames;
    int32_t on_device;
    const int32_t* edge_offset;   /* [n_frames + 1] */
    const float* pose;            /* [n_frames][7] */
    const float* world_pos;       /* [ne][3] */
    const float* obs;             /* [ne][3] */
    const float* inv_sigma2;      /* [ne] */
    float fx, fy, cx, cy, bf;     /* pFrame->fx .. mbf */
    int32_t n_edges_max;          /* on_device: an upper bound of edge_offset[n_frames] (sizes the scratch); else ignored */
} orbo_pose_problems;

orb_status orbo_pose_optimization(orbx_handle* h, const orbo_pose_problems* in, double* pose_out, uint8_t* outlier_out,
                                  int32_t* inliers_out, int32_t* stats_out);

/* The correspondence walk of PoseOptimization (Optimizer.cc:104-290) for frames whose features and matches are still on
 * the device: one edge per feature that holds a map point, in feature order.  feature_match (per compact keypoint row:
 * query index or -1) is the output of orbm_search_last_frame / orbm_search_bow; query_match (per query: feature index or
 * -1) the output of orbm_search_local_points; one of the two is given, or both together with query_world_pos.  world_pos[q] = pMP->GetWorldPos() of
 * query q.  ALL pointers are device memory; no synchronisation.  Outputs feed
 * orbo_pose_optimization (on_device = 1): edge_offset_out[n_frames + 1], and per edge the feature index inside its frame
 * (to map outlier flags back to mvbOutlier), world position, observation (x, y, mvuRight or -1) and
 * mvInvLevelSigma2[octave]; each output must hold one entry per feature of the listed frames. */
typedef struct {
    int32_t n_frames;
    const int32_t* frame_image;   /* [n_frames] image index in the handle's last batch */
    const int32_t* feature_match; /* or NULL */
    const int32_t* query_offset;  /* [n_frames + 1], with query_match */
    const int32_t* query_match;   /* or NULL */
    const float* world_pos;       /* [nq][3] */
    const float* query_world_pos; /* NULL, or -- with BOTH feature_match and query_match given (TrackLocalMap: the map points the motion-model
                                     search left in the frame plus the local-map matches; a feature both hold goes to the local-map one, as
                                     ORBmatcher.cc:116-118 only lets the second search take features whose map point has no observations) --
                                     GetWorldPos() of the query_match entries; world_pos then belongs to the feature_match entries */
} orbo_edge_source;

orb_status orbo_pose_edges(orbx_handle* h, const orbo_edge_source* src, int32_t* edge_offset_out, int32_t* edge_feature_out,
                           float* world_pos_out, float* obs_out, float* inv_sigma2_out);


/* PoseOptimization for frames of the handle's last batch straight from a search's result arrays (HOST memory): the
 * correspondence walk runs on the device against the resident features.  feature_match: the feature_match_out array of
 * orbm_search_last_frame / orbm_search_bow (all compact rows of the batch); or query_offset + query_match: the match_out
 * array of orbm_search_local_points.  world_pos[q] = pMP->GetWorldPos() of query q (n_queries entries).
 * feature_outlier_out (may be NULL): pFrame->mvbOutlier per compact row, written for the listed frames only. */
typedef struct {
    int32_t n_frames;
    const int32_t* frame_image;
    const float* pose;             /* [n_frames][7] */
    const int32_t* feature_match;  /* or NULL */
    const int32_t* query_offset;   /* [n_frames + 1], with query_match */
    const int32_t* query_match;    /* or NULL */
    const float* world_pos;        /* [n_queries][3] */
    int32_t n_queries;
    float fx, fy, cx, cy, bf;
} orbo_frame_matches;

orb_status orbo_pose_optimization_frames(orbx_handle* h, const orbo_frame_matches* in, double* pose_out,
                                         uint8_t* feature_outlier_out, int32_t* inliers_out);


/* ------------------------------------------------------------------------------------------------
 * Frame::ComputeBoW / KeyFrame::ComputeBoW  (src/Frame.cc:984-997): mpORBvocabulary->transform(descriptors, mBowVec,
 * mFeatVec, 4) -- DBoW2 TemplatedVocabulary::transform, Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1260, with the
 * TF_IDF weighting and L1 scoring ORBvoc.txt is loaded with.
 *
 * orbv_create uploads the vocabulary tree the caller flattened from its DBoW2 object: node 0 is the root, the children of
 * node i are child_ids[child_offset[i] .. child_offset[i+1]) in m_nodes[i].children order, node_desc = m_nodes[i].descriptor
 * (32 bytes), node_word / node_weight = word_id / weight of the leaves (ignored for inner nodes), depth_levels = m_L.
 * orbv_transform runs every descriptor of the extractor's last batch down the tree: word_out / weight_out per compact row
 * (WordId, idf weight; weight 0 = stopped word), node_out = the NodeId at levelsup levels above the leaf (what
 * mFeatVec.addFeature receives and what orbm_search_bow takes as feature_node).  DBoW2 adds a feature to mBowVec AND to mFeatVec
 * only when its weight is > 0 (TemplatedVocabulary.h:1153-1157): a caller rebuilding mFeatVec lists feature i under node_out[i]
 * iff weight_out[i] > 0 and passes feature_node = -1 for the others.  Optionally the BowVector of every image:
 * bow_count_out[img] entries of (bow_word_out, bow_weight_out)[img][max features] in ascending word order, weights summed
 * in feature order and L1-normalised exactly like BowVector::addWeight / normalize.  on_device != 0: outputs are device
 * memory, no synchronisation. */
typedef struct orbv_vocabulary orbv_vocabulary;
orb_status orbv_create(int32_t device, int32_t n_nodes, int32_t depth_levels, const int32_t* child_offset, const int32_t* child_ids,
                       const uint8_t* node_desc, const int32_t* node_word, const double* node_weight, orbv_vocabulary** out);
void orbv_destroy(orbv_vocabulary* v);
orb_status orbv_transform(orbx_handle* h, const orbv_vocabulary* voc, int32_t levelsup, int32_t on_device, int32_t* word_out,
                          int32_t* node_out, double* weight_out, int32_t* bow_count_out, int32_t* bow_word_out, double* bow_weight_out);


/* ------------------------------------------------------------------------------------------------
 * MapPoint maintenance either side of the searches (LocalMapping.cc:300-340, 860-875), batched over map points; the
 * extractor handle lends its stream, scratch and level tables.  Observations of point i are rows
 * [obs_offset[i], obs_offset[i+1]) in the order the reference walks mObservations (std::map<KeyFrame*, ...>).
 *
 * MapPoint::ComputeDistinctiveDescriptors  src/MapPoint.cc:438-520: best_index_out[i] = position (inside the point's
 * observation list) of the descriptor with the smallest median Hamming distance to the set -- sort + vDists[0.5*(N-1)],
 * first minimum -- or -1 for a point without observations (mDescriptor is then left as it is).
 *
 * MapPoint::UpdateNormalAndDepth  src/MapPoint.cc:567-640: obs_center = pKF->GetCameraCenter() per observation, ref_center /
 * ref_level = camera centre of mpRefKF and the octave of the point's keypoint there.  normal_out = mNormalVector,
 * max_dist_out / min_dist_out = mfMaxDistance / mfMinDistance (in/out: points without observations keep their values). */
orb_status orbp_distinctive_descriptors(orbx_handle* h, int32_t n_points, const int32_t* obs_offset, const uint8_t* obs_desc,
                                        int32_t* best_index_out);
orb_status orbp_update_normal_and_depth(orbx_handle* h, int32_t n_points, const int32_t* obs_offset, const float* obs_center,
                                        const float* world_pos, const float* ref_center, const int32_t* ref_level,
                                        float* normal_out, float* max_dist_out, float* min_dist_out);

/* ------------------------------------------------------------------------------------------------
 * Optimizer::LocalInertialBA  (include/Optimizer.h:63, src/Optimizer.cc:2203-2812), single camera -- the numeric core
 * `optimizer.optimize(opt_it)`: g2o Levenberg (user lambda 1e0, or 1e-2 when bLarge) over BlockSolverX with
 * VertexPose / VertexVelocity / VertexGyroBias / VertexAccBias per keyframe, marginalised VertexSBAPointXYZ, EdgeMono /
 * EdgeStereo (Huber sqrt(5.991) / sqrt(7.815)), EdgeInertial (+ optional Huber sqrt(16.92)), EdgeGyroRW, EdgeAccRW.
 *
 * Device parity: tests/test_liba_gpu.py (same LM iterations / trials as the fp64 oracle, states to 1e-13); host emulation of the
 * same source: tests/test_liba_emul.py.  The shim builds the window (Optimizer.cc:2217-2340) and fills these arrays:
 *   state[k]   Rwb (9, row-major) twb v bg ba of keyframe k  (ImuCamPose of VertexPose + the three additive vertices)
 *   fixed[k]   1 for the N+1-th keyframe and the covisible lFixedKeyFrames (all four vertices setFixed)
 *   links      one per consecutive pair with mpImuPreintegrated: float members of IMU::Preintegrated (dR dV dP JRg JVg JVa
 *              JPg JPa, the bias b it was integrated at as bax bay baz bwx bwy bwz), dT, info = EdgeInertial's 9 x 9
 *              information (G2oTypes.cc:575-586: inverse of C.block<9,9>(0,0) symmetrised, eigenvalues < 1e-12 zeroed; x 1e-2
 *              for the oldest link i == N-1, Optimizer.cc:2467-2479), infoG / infoA = inverses of C.block<3,3>(9,9) / (12,12)
 *              (Optimizer.cc:2486-2494); robust = 1 where the reference installs the Huber kernel (i == N-1 || bRecInit)
 *   edges      as lba_problem (obs z < 0 => EdgeMono)
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t k1, k2, robust, pad;
    double dt;
    float dR[9], dV[3], dP[3], JRg[9], JVg[9], JVa[9], JPg[9], JPa[9], bias[6];
    double info[81], infoG[9], infoA[9];
} liba_link;                       /* 1080 bytes */

typedef struct {
    int32_t n_kf, n_mp, n_edges, n_links;
    const double* state;           /* [n_kf][21] */
    const uint8_t* fixed;          /* [n_kf] */
    const double* point;           /* [n_mp][3] */
    const int32_t* edge_kf;        /* [n_edges] */
    const int32_t* edge_mp;        /* [n_edges] */
    const double* obs;             /* [n_edges][3] */
    const double* inv_sigma2;      /* [n_edges] */
    const liba_link* links;        /* [n_links] */
    double Tcb[12];                /* Rcb (9, row-major) tcb (3): ImuCamPose::Rcb[0] / tcb[0] */
    double fx, fy, cx, cy, bf;
    double lambda_init;            /* 1e0 / 1e-2 (0 = g2o's automatic tau * max diagonal) */
    int32_t max_iters;             /* opt_it: 10, or 4 when bLarge */
} liba_problem;

typedef struct {
    double* state;                 /* [n_kf][21] optimised */
    double* point;                 /* [n_mp][3] */
    double* edge_chi2;             /* [n_edges] (may be NULL) */
    double* link_chi2;             /* [n_links][3] inertial, gyro RW, acc RW (may be NULL) */
    uint8_t* edge_depth_positive;  /* [n_edges] e->isDepthPositive() at the final estimate (may be NULL); Optimizer.cc:2704 */
    int32_t iterations, trials;
    double lambda, chi2, chi2_initial;
    double chi2_last_trial;        /* optimizer.activeRobustChi2() as read right after optimize() (err_end, Optimizer.cc:2685): the
                                      errors of the LAST Levenberg trial, accepted or not -- what edge_chi2 / link_chi2 hold too */
} liba_result;

typedef struct liba_handle liba_handle;
orb_status liba_create(int32_t device, liba_handle** out);
void liba_destroy(liba_handle* h);
/* independent windows, one CTA each */
orb_status liba_solve(liba_handle* h, int32_t n_problems, const liba_problem* in, liba_result* out);
/* Host helper (no device work): liba_link::info / infoG / infoA from IMU::Preintegrated::C (15 x 15 floats, row-major), as
 * EdgeInertial's constructor (G2oTypes.cc:575-586: inverse of the top-left 9 x 9 block, symmetrised, eigenvalues < 1e-12 zeroed)
 * and Optimizer.cc:2486-2494 (inverses of C.block<3,3>(9,9) and (12,12)) compute them; oldest != 0 applies the 1e-2 of
 * Optimizer.cc:2477-2478 (i == N - 1). */
orb_status liba_link_information(const float* C15x15, int32_t oldest, double* info81, double* infoG9, double* infoA9);

/* ------------------------------------------------------------------------------------------------
 * Batched sequence replay: the tracking-thread step of n_frames stereo frames, HOST buffers in, HOST buffers out.
 *
 * What Tracking does per frame -- Frame::Frame (both eyes through ORBextractor::operator(), Frame.cc:136-141, and
 * ComputeStereoMatches, Frame.cc:1102), TrackWithMotionModel (ORBmatcher::SearchByProjection(cur, last) then
 * Optimizer::PoseOptimization, Tracking.cc:3389-3443), TrackLocalMap (SearchByProjection(F, local map points) then
 * PoseOptimization, Tracking.cc:4052, 3522) -- queued for a batch of frames (one per replayed sequence) on the handle's
 * stream.  orbr_submit copies the images and the query arrays in, queues every kernel and returns without waiting;
 * orbr_collect waits for the batch's count tables, copies back exactly the rows it produced and waits once more.  Pinned
 * host memory makes the copies asynchronous; a host thread that keeps several handles in flight (submit on handles
 * k+1 .. k+H-1 before collecting handle k) overlaps uploads, kernels and downloads without further threads.
 * One step per handle may be in flight.  Images: 2 * n_frames, left eye of frame p = image 2p, right eye = image 2p + 1.
 *
 * Monocular step (orbr_step::monocular != 0): what Tracking::GrabImageMonocular -> Frame::Frame(monocular) -> Track does per frame
 * for a rectified camera.  Image f is frame f (n_frames images, n_frames <= max_batch).  Each image goes through
 * ORBextractor::operator() with vLappingArea = {0, 1000} (Frame.cc:380), so keypoints are back-filled as the reference orders them;
 * Frame::UndistortKeyPoints is an identity copy for a camera with zero distortion and is not run.  ComputeStereoMatches does not run:
 * every feature has mvuRight = mvDepth = -1, so both searches and PoseOptimization take their monocular branches and bf / b are
 * ignored.  TrackWithMotionModel passes bMono = true for a monocular sensor (Tracking.cc:3389-3443), so the last-frame search
 * never looks forward or backward: every last->direction[f] must be 0 (ORBmatcher.cc:1967-1971).  frame_image indexes
 * [0, n_frames).  The searches, PoseOptimization and the chained flow keep their meaning.  orbr_collect returns n / offsets with
 * n_frames / n_frames + 1 entries and fills uright / depth with -1.
 * ---------------------------------------------------------------------------------------------- */
/* The chained data flow of one tracked frame (Tracking.cc:3389-3522, 4010-4062) instead of two independent searches with precomputed
 * projections: the motion-model search and its PoseOptimization run first; the features whose map point came out an outlier are released
 * (Tracking.cc:3447-3470); the optimised pose goes through Sophus::SE3f (Optimizer.cc:406-410, Frame::UpdatePoseMatrices) into
 * Frame::isInFrustum for every local map point that the motion-model search did not already put into the frame (mnLastFrameSeen,
 * Tracking.cc:3997-4000); SearchByProjection(F, local map points) sees the features that still hold a map point with observations
 * (ORBmatcher.cc:116-118); the second PoseOptimization starts from the first one's pose over ALL map points the frame holds. */
typedef struct {
    const int32_t* point_offset;         /* [n_frames + 1] local map points of every frame (mvpLocalMapPoints, isBad ones removed) */
    const float* world_pos;              /* [np][3] GetWorldPos */
    const float* normal;                 /* [np][3] GetNormal */
    const float* max_dist;               /* [np] mfMaxDistance (raw) */
    const float* min_dist;               /* [np] mfMinDistance (raw) */
    const uint8_t* desc;                 /* [np][32] GetDescriptor */
    const int32_t* last_query;           /* [np] this map point's index in the frame's OWN `last` query list (0-based inside the frame), or -1 */
    float viewing_cos_limit;             /* 0.5 (Tracking.cc:4022) */
} orbr_chain;

typedef struct {
    int32_t n_frames;
    const uint8_t* images;               /* HOST: 2 * n_frames images (n_frames with monocular or depth_maps) */
    int32_t width, height, stride;       /* stride in bytes between rows */
    size_t image_stride_bytes;           /* between consecutive images */
    float bf, b;                         /* Frame::mbf, Frame::mb */
    const orbm_last_queries* last;       /* HOST arrays (on_device is ignored); NULL = no motion-model search */
    float th_last;
    int32_t check_orientation_last;      /* ORBmatcher::mbCheckOrientation */
    const orbm_local_queries* local;     /* HOST arrays; feature_claimed must be NULL; NULL = no local-map search */
    float th_local, nnratio_local;
    int32_t far_points;
    float th_far;
    int32_t pose_optimization;           /* != 0: Optimizer::PoseOptimization after each search */
    const float* pose;                   /* [n_frames][7] pFrame->GetPose() on entry of PoseOptimization (with pose_optimization) */
    const float* local_world_pos;        /* [nq_local][3] GetWorldPos() of the local-map entries (with pose_optimization) */
    const orbr_chain* chain;             /* NULL, or the chained flow: needs `last` and `pose`, `local` must be NULL; PoseOptimization runs after both
                                            searches whatever pose_optimization says; local_* results are indexed by the chain's map points */
    int32_t monocular;                   /* != 0: n_frames images, one per frame (Frame's monocular constructor), instead of 2 * n_frames stereo eyes */
    /* Camera images as they arrive (orbx_extract_batch_device_format): all five zero = grey images of width x height laid out by
       stride / image_stride_bytes above.  Otherwise `images` holds src_width x src_height images in image_format, laid out by
       src_stride / src_image_stride_bytes, resized to width x height (when the sizes differ) and converted to grey on the device;
       stride / image_stride_bytes are not read. */
    int32_t image_format;                /* orb_image_format */
    int32_t src_width, src_height;       /* 0 = width x height */
    int32_t src_stride;                  /* bytes between rows; 0 = src_width x channels */
    size_t src_image_stride_bytes;       /* bytes between images; 0 = src_stride x src_height */
    /* RGB-D step (depth_maps != NULL; all five zero = as above): what Tracking::GrabImageRGBD -> Frame::Frame(RGB-D) -> Track does per
       frame for a camera with zero distortion.  Image f is frame f (n_frames images, extracted with vLappingArea = {0, 0}), and HOST
       depth map f, of width x height, gives its mvuRight / mvDepth as orbm_stereo_rgbd_batch does, in place of ComputeStereoMatches.
       The searches (any direction), PoseOptimization and the chained flow follow unchanged.  Refused: monocular together with depth
       maps (ORB_ERR_INVALID), and camera images of another size than width x height (ORB_ERR_UNSUPPORTED: System::TrackRGBD would
       resize the depth map too, which is not built). */
    const void* depth_maps;
    int32_t depth_format;                /* orb_depth_format */
    int32_t depth_stride;                /* bytes between rows; 0 = width x element size */
    size_t depth_image_stride_bytes;     /* bytes between maps; 0 = depth_stride x height */
    float depth_factor;                  /* Tracking::mDepthMapFactor */
} orbr_step;

typedef struct {                         /* HOST result buffers; any pointer may be NULL (that result is not copied back) */
    int32_t cap_rows;                    /* capacity, in rows, of every per-row / per-edge array below */
    orbx_keypoint* keypoints;            /* compact rows of the whole batch, image after image (mvKeys) */
    uint8_t* descriptors;                /* [rows][32] (mDescriptors) */
    float* uright;                       /* [rows] mvuRight (stereo: the left-eye rows hold it; RGB-D: every row; monocular: -1) */
    float* depth;                        /* [rows] mvDepth (as uright) */
    int32_t* n;                          /* [2 n_frames] keypoints per image (n_frames in a monocular or RGB-D step) */
    int32_t* offsets;                    /* [2 n_frames + 1] first row of every image (n_frames + 1 in a monocular or RGB-D step) */
    int32_t* last_feature_match;         /* [rows] as orbm_search_last_frame */
    int32_t* last_nmatches;              /* [n_frames] */
    int32_t* local_match;                /* [nq_local] as orbm_search_local_points */
    int32_t* local_nmatches;             /* [n_frames] */
    /* PoseOptimization after the motion-model search [0] and after the local-map search [1] */
    double* pose[2];                     /* [n_frames][7] */
    int32_t* inliers[2];                 /* [n_frames] */
    int32_t* edge_offset[2];             /* [n_frames + 1] */
    int32_t* edge_feature[2];            /* [edges] feature index inside its frame */
    uint8_t* edge_outlier[2];            /* [edges] pFrame->mvbOutlier of that feature */
    /* chained flow only: what Frame::isInFrustum wrote into every local map point (0 / -1 where it was skipped or not in view) */
    uint8_t* chain_in_view;              /* [np] mbTrackInView */
    float* chain_proj_x;                 /* [np] mTrackProjX */
    float* chain_proj_y;
    float* chain_proj_xr;
    int32_t* chain_level;                /* [np] mnTrackScaleLevel */
    float* chain_view_cos;               /* [np] mTrackViewCos */
    float* chain_pose_f;                 /* [n_frames][7] the Sophus::SE3f the frame holds after the first PoseOptimization (qx qy qz qw tx ty tz) */
} orbr_results;

orb_status orbr_submit(orbx_handle* h, const orbm_camera* cam, const orbr_step* step);
orb_status orbr_collect(orbx_handle* h, const orbr_results* out, int32_t* total_rows_out);

/* Keyframe state of image `image` of the last batch (the pose the caller passes, mvKeysUn positions and octaves, mvuRight,
 * mDescriptors: what KeyFrame::KeyFrame(Frame&) keeps, KeyFrame.cc:45-90) as ONE block in device memory:
 * [int32 n][7 x f32 pose][n x (x, y) f32][n x int32 octave][n x f32 uright][n x 32 B descriptors], at most
 * orbx_keyframe_block_bytes(h) bytes.  Replicas that share a map all-gather these fixed-capacity blocks (NCCL) when a rank
 * inserts a keyframe.  d_pose7 and d_block (16-byte aligned) are device memory; no synchronisation. */
size_t orbx_keyframe_block_bytes(const orbx_handle* h);
orb_status orbx_pack_keyframe_device(orbx_handle* h, int32_t image, const float* d_pose7, uint8_t* d_block, size_t block_bytes);

#ifdef __cplusplus
}
#endif
#endif /* ORBSLAM3_B200_H */
