// tests/host/host_units.cc -- runs the nine host translation units that host_boundary.cc does not (both SearchByBoW overloads,
// SearchForInitialization, SearchForTriangulation, Fuse(pKF, vpMapPoints), the relocalisation SearchByProjection, the Sim3 searches,
// Frame::ComputeBoW, PoseOptimization, LocalInertialBA) the way their callers would, linked with the library.  Frames that must be on the
// device come from a real extraction through the drop-in ORBextractor; keyframes, map points, the vocabulary and the inertial map are
// built from raw arrays as the CPU drivers (bow_cpu.cc, fuse_cpu.cc, voc_cpu.cc, pose_cpu.cc, liba_cpu.cc) build them.
// build_units.sh links it with -Wl,--wrap= on the C ABI calls the units make: every wrapper below writes the call's exact inputs and
// outputs to the scratch directory (rec_<call><k>_<field>, k = call index) and forwards to the library, so that
// tests/test_zz_host_units_gpu.py can compare each device answer with the oracle on the recorded inputs and, separately, restate what
// the unit wrote back from that answer.
//   host_units <dir>        (unit.txt names the member to run; meta.txt holds its parameters)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "ref_skeleton_impl.h"   // also brings the reference's ORBextractor.h
#include "ORBmatcher.h"
#include "Optimizer.h"
#include "orb_b200_host.h"

using namespace ORB_SLAM3;
extern "C" void orb_b200_use_handle_for_keyframe_searches(orbx_handle* h);   // host/ORBmatcher_bow_b200.cc

static std::string g_dir;
template <typename T>
static std::vector<T> rd(const std::string& name) {
    std::ifstream f(g_dir + "/" + name, std::ios::binary);
    if (!f) { std::fprintf(stderr, "missing input %s\n", name.c_str()); std::exit(2); }
    f.seekg(0, std::ios::end);
    const size_t n = (size_t)f.tellg();
    f.seekg(0);
    std::vector<T> v(n / sizeof(T));
    f.read((char*)v.data(), (std::streamsize)(v.size() * sizeof(T)));
    return v;
}
static void wr_raw(const std::string& name, const void* p, size_t bytes) {
    std::ofstream f(g_dir + "/" + name, std::ios::binary);
    if (bytes) f.write((const char*)p, (std::streamsize)bytes);
}
template <typename T>
static void wr(const std::string& name, const std::vector<T>& v) { wr_raw(name, v.data(), v.size() * sizeof(T)); }
static std::map<std::string, double> read_meta() {
    std::map<std::string, double> m;
    std::ifstream f(g_dir + "/meta.txt");
    std::string k;
    double v;
    while (f >> k >> v) m[k] = v;
    return m;
}
static Sophus::SE3f se3_of(const float* q7) {   // qx qy qz qw tx ty tz
    return Sophus::SE3f(Eigen::Quaternionf(q7[3], q7[0], q7[1], q7[2]), Eigen::Vector3f(q7[4], q7[5], q7[6]));
}
static std::vector<cv::KeyPoint> keys_of(const std::vector<orbx_keypoint>& k) {
    std::vector<cv::KeyPoint> o(k.size());
    for (size_t i = 0; i < k.size(); ++i) { o[i].pt.x = k[i].x; o[i].pt.y = k[i].y; o[i].size = k[i].size; o[i].angle = k[i].angle; o[i].response = k[i].response; o[i].octave = k[i].octave; o[i].class_id = k[i].class_id; }
    return o;
}
static cv::Mat desc_mat(const std::vector<uint8_t>& d) {
    cv::Mat D((int)(d.size() / 32), 32, CV_8UC1);
    if (!d.empty()) std::memcpy(D.ptr(0), d.data(), d.size());
    return D;
}
static void set_desc(MapPoint& p, const uint8_t* d) { p.mock_desc.create(1, 32, CV_8UC1); std::memcpy(p.mock_desc.ptr(0), d, 32); }

// ---------------------------------------------------------------------------------------------------------------------------------
// recorders: one file per argument, named after the call and its index
// ---------------------------------------------------------------------------------------------------------------------------------
static std::map<std::string, int> g_calls;
struct Rec {
    std::string pre;
    explicit Rec(const char* tag) { const int k = g_calls[tag]++; pre = std::string("rec_") + tag + std::to_string(k) + "_"; }
    void put(const char* field, const void* p, size_t bytes) const { wr_raw(pre + field, p, p ? bytes : 0); }
    template <typename T>
    void val(const char* field, T v) const { put(field, &v, sizeof(T)); }
};
static int32_t rows_of(orbx_handle* h) { int32_t n = 0; orbx_counts(h, &n, nullptr, nullptr); return n; }

extern "C" {
orb_status __real_orbm_search_bow(orbx_handle*, const orbm_bow_queries*, float, int32_t, int32_t*, int32_t*);
orb_status __real_orbm_search_bow_keyframes(orbx_handle*, const orbm_bow_kf_queries*, float, int32_t, int32_t*, int32_t*);
orb_status __real_orbm_search_initialization(orbx_handle*, const orbm_camera*, const orbm_init_queries*, int32_t, float, int32_t, int32_t*, int32_t*);
orb_status __real_orbm_search_triangulation(orbx_handle*, const orbm_triangulation*, int32_t*, int32_t*);
orb_status __real_orbm_search_keyframe(orbx_handle*, const orbm_camera*, const orbm_kf_queries*, int32_t, float, float, int32_t, int32_t*, int32_t*);
orb_status __real_orbv_create(int32_t, int32_t, int32_t, const int32_t*, const int32_t*, const uint8_t*, const int32_t*, const double*, orbv_vocabulary**);
orb_status __real_orbv_transform(orbx_handle*, const orbv_vocabulary*, int32_t, int32_t, int32_t*, int32_t*, double*, int32_t*, int32_t*, double*);
orb_status __real_orbo_pose_optimization(orbx_handle*, const orbo_pose_problems*, double*, uint8_t*, int32_t*, int32_t*);
orb_status __real_liba_solve(liba_handle*, int32_t, const liba_problem*, liba_result*);

orb_status __wrap_orbm_search_bow(orbx_handle* h, const orbm_bow_queries* q, float nnratio, int32_t check, int32_t* fm, int32_t* nm) {
    const orb_status s = __real_orbm_search_bow(h, q, nnratio, check, fm, nm);
    Rec r("bow");
    const int nq = q->query_offset[1], N = rows_of(h);
    r.val("handle", (uint64_t)(size_t)h); r.val("status", (int32_t)s);
    const float par[5] = {nnratio, (float)check, (float)q->n_frames, (float)q->on_device, (float)q->frame_image[0]};
    r.put("par", par, sizeof(par));
    r.put("qnode", q->query_node, 4 * (size_t)nq); r.put("qangle", q->query_angle, 4 * (size_t)nq); r.put("qdesc", q->desc, 32 * (size_t)nq);
    r.put("fnode", q->feature_node, 4 * (size_t)N);
    if (s == ORB_OK) { r.put("fm", fm, 4 * (size_t)N); r.put("nm", nm, 4); }
    return s;
}
orb_status __wrap_orbm_search_bow_keyframes(orbx_handle* h, const orbm_bow_kf_queries* q, float nnratio, int32_t check, int32_t* m12, int32_t* nm) {
    const orb_status s = __real_orbm_search_bow_keyframes(h, q, nnratio, check, m12, nm);
    Rec r("bowkf");
    const int nq = q->query_offset[1], n2 = q->feat_offset[1];
    r.val("handle", (uint64_t)(size_t)h); r.val("status", (int32_t)s);
    const float par[3] = {nnratio, (float)check, (float)q->n_pairs};
    r.put("par", par, sizeof(par));
    r.put("kp2", q->kp2, sizeof(orbx_keypoint) * n2); r.put("desc2", q->desc2, 32 * (size_t)n2); r.put("node2", q->node2, 4 * (size_t)n2);
    r.put("valid2", q->valid2, n2);
    r.put("qnode", q->query_node, 4 * (size_t)nq); r.put("qangle", q->query_angle, 4 * (size_t)nq); r.put("desc1", q->desc1, 32 * (size_t)nq);
    if (s == ORB_OK) { r.put("m12", m12, 4 * (size_t)nq); r.put("nm", nm, 4); }
    return s;
}
orb_status __wrap_orbm_search_initialization(orbx_handle* h, const orbm_camera* cam, const orbm_init_queries* q, int32_t window, float nnratio, int32_t check,
                                             int32_t* m12, int32_t* nm) {
    const orb_status s = __real_orbm_search_initialization(h, cam, q, window, nnratio, check, m12, nm);
    Rec r("init");
    r.val("handle", (uint64_t)(size_t)h); r.val("status", (int32_t)s);
    r.put("cam", cam, sizeof(*cam));
    const float par[5] = {(float)window, nnratio, (float)check, (float)q->target_image, (float)q->n2};
    r.put("par", par, sizeof(par));
    r.put("kp1", q->kp1, sizeof(orbx_keypoint) * q->n1); r.put("desc1", q->desc1, 32 * (size_t)q->n1); r.put("prev", q->prev_matched, 8 * (size_t)q->n1);
    if (q->kp2) { r.put("kp2", q->kp2, sizeof(orbx_keypoint) * q->n2); r.put("desc2", q->desc2, 32 * (size_t)q->n2); }
    if (s == ORB_OK) { r.put("m12", m12, 4 * (size_t)q->n1); r.put("nm", nm, 4); }
    return s;
}
orb_status __wrap_orbm_search_triangulation(orbx_handle* h, const orbm_triangulation* t, int32_t* m12, int32_t* nm) {
    const orb_status s = __real_orbm_search_triangulation(h, t, m12, nm);
    Rec r("tri");
    const int nq = t->n_queries, n2 = t->n2;
    r.val("handle", (uint64_t)(size_t)h); r.val("status", (int32_t)s);
    r.put("kp1", t->kp1, sizeof(orbx_keypoint) * nq); r.put("desc1", t->desc1, 32 * (size_t)nq); r.put("node1", t->node1, 4 * (size_t)nq); r.put("stereo1", t->stereo1, nq);
    r.put("kp2", t->kp2, sizeof(orbx_keypoint) * n2); r.put("desc2", t->desc2, 32 * (size_t)n2); r.put("node2", t->node2, 4 * (size_t)n2);
    r.put("valid2", t->valid2, n2); r.put("stereo2", t->stereo2, n2);
    r.put("F12", t->F12, sizeof(t->F12)); r.put("ep2", t->epipole2, sizeof(t->epipole2));
    const int32_t flags[2] = {t->coarse, t->check_orientation};
    r.put("flags", flags, sizeof(flags));
    if (s == ORB_OK) { r.put("m12", m12, 4 * (size_t)nq); r.put("nm", nm, 4); }
    return s;
}
orb_status __wrap_orbm_search_keyframe(orbx_handle* h, const orbm_camera* cam, const orbm_kf_queries* q, int32_t variant, float th, float hamming_max, int32_t check,
                                       int32_t* match, int32_t* nm) {
    const orb_status s = __real_orbm_search_keyframe(h, cam, q, variant, th, hamming_max, check, match, nm);
    Rec r("kf");
    const int nq = q->query_offset[1], N = q->kp ? q->feat_offset[1] : rows_of(h);
    r.val("handle", (uint64_t)(size_t)h); r.val("status", (int32_t)s);
    r.put("cam", cam, sizeof(*cam));
    const float par[6] = {(float)variant, th, hamming_max, (float)check, (float)q->n_targets, q->kp ? -1.f : (float)q->target_image[0]};
    r.put("par", par, sizeof(par));
    if (q->kp) { r.put("kp", q->kp, sizeof(orbx_keypoint) * N); r.put("desc", q->desc, 32 * (size_t)N); r.put("uright", q->uright, 4 * (size_t)N); }
    r.put("claimed", q->feat_claimed, N);
    r.put("Tcw", q->Tcw, 28); r.put("Ow", q->Ow, 12); r.put("Sim3", q->Sim3, 32);
    r.put("xw", q->world_pos, 12 * (size_t)nq); r.put("normal", q->normal, 12 * (size_t)nq); r.put("maxd", q->max_dist, 4 * (size_t)nq);
    r.put("mind", q->min_dist, 4 * (size_t)nq); r.put("qdesc", q->desc_q, 32 * (size_t)nq); r.put("angle", q->angle, 4 * (size_t)nq);
    if (s == ORB_OK) { r.put("match", match, 4 * (size_t)nq); r.put("nm", nm, 4); }
    return s;
}
orb_status __wrap_orbv_create(int32_t dev, int32_t n, int32_t L, const int32_t* co, const int32_t* ci, const uint8_t* nd, const int32_t* nw, const double* wt,
                              orbv_vocabulary** out) {
    Rec r("vcreate");
    r.val("L", L);
    r.put("child_offset", co, 4 * ((size_t)n + 1)); r.put("child_ids", ci, 4 * (size_t)co[n]); r.put("node_desc", nd, 32 * (size_t)n);
    r.put("node_word", nw, 4 * (size_t)n); r.put("node_weight", wt, 8 * (size_t)n);
    return __real_orbv_create(dev, n, L, co, ci, nd, nw, wt, out);
}
orb_status __wrap_orbv_transform(orbx_handle* h, const orbv_vocabulary* voc, int32_t levelsup, int32_t on_device, int32_t* word, int32_t* node, double* weight,
                                 int32_t* bow_count, int32_t* bow_word, double* bow_weight) {
    const orb_status s = __real_orbv_transform(h, voc, levelsup, on_device, word, node, weight, bow_count, bow_word, bow_weight);
    Rec r("vtransform");
    const int N = rows_of(h);
    const int32_t par[2] = {levelsup, on_device};
    r.put("par", par, sizeof(par)); r.val("status", (int32_t)s);
    if (s == ORB_OK) {
        r.put("word", word, 4 * (size_t)N); r.put("node", node, 4 * (size_t)N); r.put("weight", weight, 8 * (size_t)N);
        r.put("bow_count", bow_count, 4); r.put("bow_word", bow_word, 4 * (size_t)*bow_count); r.put("bow_weight", bow_weight, 8 * (size_t)*bow_count);
    }
    return s;
}
orb_status __wrap_orbo_pose_optimization(orbx_handle* h, const orbo_pose_problems* in, double* pose_out, uint8_t* outlier, int32_t* inliers, int32_t* stats) {
    int32_t st[4] = {0, 0, 0, 0};              // rounds, LM iterations, LM trials: recorded whether or not the caller asks for them
    const orb_status s = __real_orbo_pose_optimization(h, in, pose_out, outlier, inliers, st);
    if (stats) std::memcpy(stats, st, sizeof(st));
    Rec r("pose");
    const int ne = in->edge_offset[1];
    r.val("status", (int32_t)s);
    const float cam5[5] = {in->fx, in->fy, in->cx, in->cy, in->bf};
    r.put("cam5", cam5, sizeof(cam5)); r.put("pose", in->pose, 28);
    r.put("xw", in->world_pos, 12 * (size_t)ne); r.put("obs", in->obs, 12 * (size_t)ne); r.put("inv_sigma2", in->inv_sigma2, 4 * (size_t)ne);
    if (s == ORB_OK) { r.put("pose_out", pose_out, 56); r.put("outlier", outlier, ne); r.put("inliers", inliers, 4); r.put("stats", st, sizeof(st)); }
    return s;
}
orb_status __wrap_liba_solve(liba_handle* h, int32_t n_problems, const liba_problem* in, liba_result* out) {
    const orb_status s = __real_liba_solve(h, n_problems, in, out);
    Rec r("liba");
    const liba_problem& P = in[0];
    const liba_result& R = out[0];
    r.val("status", (int32_t)s); r.val("n_problems", n_problems);
    const int32_t sizes[4] = {P.n_kf, P.n_mp, P.n_edges, P.n_links};
    r.put("sizes", sizes, sizeof(sizes));
    r.put("state", P.state, 168 * (size_t)P.n_kf); r.put("fixed", P.fixed, P.n_kf); r.put("point", P.point, 24 * (size_t)P.n_mp);
    r.put("edge_kf", P.edge_kf, 4 * (size_t)P.n_edges); r.put("edge_mp", P.edge_mp, 4 * (size_t)P.n_edges); r.put("obs", P.obs, 24 * (size_t)P.n_edges);
    r.put("inv_sigma2", P.inv_sigma2, 8 * (size_t)P.n_edges); r.put("links", P.links, sizeof(liba_link) * P.n_links);
    const double scal[9] = {P.Tcb[0], P.fx, P.fy, P.cx, P.cy, P.bf, P.lambda_init, (double)P.max_iters, 0};
    r.put("Tcb", P.Tcb, sizeof(P.Tcb)); r.put("scal", scal, sizeof(scal));
    if (s == ORB_OK) {
        r.put("state_out", R.state, 168 * (size_t)P.n_kf); r.put("point_out", R.point, 24 * (size_t)P.n_mp);
        r.put("edge_chi2", R.edge_chi2, 8 * (size_t)P.n_edges); r.put("edge_depth_positive", R.edge_depth_positive, P.n_edges);
        const double st[5] = {(double)R.iterations, (double)R.trials, R.lambda, R.chi2, R.chi2_initial};
        r.put("stats", st, sizeof(st));
    }
    return s;
}
}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------------------------
// the objects the units run on
// ---------------------------------------------------------------------------------------------------------------------------------
struct Extracted {                 // one image through the drop-in ORBextractor: the frame its extractor produced last
    std::vector<cv::KeyPoint> kps;
    cv::Mat desc;
};
static Extracted extract(ORBextractor& ex, const std::string& img, int W, int H, const char* out_tag) {
    std::vector<uint8_t> pix = rd<uint8_t>(img);
    cv::Mat m(H, W, CV_8UC1, pix.data(), (size_t)W);
    Extracted e;
    std::vector<int> lap = {0, 1000};
    ex(m, cv::Mat(), e.kps, e.desc, lap);
    std::vector<uint8_t> k((const uint8_t*)e.kps.data(), (const uint8_t*)e.kps.data() + e.kps.size() * 28), d(e.kps.size() * 32);
    for (size_t i = 0; i < e.kps.size(); ++i) std::memcpy(&d[i * 32], e.desc.ptr((int)i), 32);
    wr(std::string("out_") + out_tag + "_kps.bin", k); wr(std::string("out_") + out_tag + "_desc.u8", d);
    return e;
}
static void frame_of(Frame& F, ORBextractor* ex, const Extracted& e) {
    F.mpORBextractorLeft = ex;
    F.N = (int)e.kps.size();
    F.mvKeys = e.kps; F.mvKeysUn = e.kps; F.mDescriptors = e.desc;
    F.mvpMapPoints.assign(F.N, nullptr); F.mvbOutlier.assign(F.N, false); F.mvuRight.assign(F.N, -1.f);
}

struct MockKF {                    // as bow_cpu.cc: keyframe `tag` from <tag>.kp, <tag>_desc.u8, <tag>_node.i32, <tag>_has.u8, <tag>_bad.u8, <tag>_ur.f32, <tag>_T.f32
    std::vector<MapPoint> mps;
    KeyFrame* kf;
    MockKF(int id, const std::string& tag, const float* cam6) {
        auto k = rd<orbx_keypoint>(tag + ".kp");
        auto d = rd<uint8_t>(tag + "_desc.u8"), has = rd<uint8_t>(tag + "_has.u8"), bad = rd<uint8_t>(tag + "_bad.u8");
        auto node = rd<int>(tag + "_node.i32");
        auto ur = rd<float>(tag + "_ur.f32"), T = rd<float>(tag + "_T.f32");
        const int n = (int)k.size();
        mps.resize(n);
        kf = new KeyFrame(id, cam6[0], cam6[1], cam6[2], cam6[3], cam6[4], cam6[5], keys_of(k), ur, std::vector<float>(8, 1.f));
        kf->mock_Tcw = se3_of(T.data());
        const_cast<cv::Mat&>(kf->mDescriptors) = desc_mat(d);
        for (int i = 0; i < n; ++i) if (node[i] >= 0) kf->mFeatVec[(DBoW2::NodeId)node[i]].push_back((unsigned int)i);
        kf->mock_matches.assign(n, nullptr);
        for (int i = 0; i < n; ++i) if (has[i]) { mps[i].mock_bad = bad[i] != 0; mps[i].mock_id = i; kf->mock_matches[i] = &mps[i]; }
    }
    int index_of(MapPoint* p) const { return p ? (int)(p - mps.data()) : -1; }
};

// keyframe-side map points with geometry (Fuse, relocalisation, Sim3): objects from q_xw.f32, q_normal.f32, q_max.f32, q_min.f32, q_desc.u8, q_bad.u8, q_obs.i32
struct QueryPoints {
    std::vector<MapPoint> obj;
    std::vector<KeyFrame*> others;
    explicit QueryPoints(const std::string& tag) {
        auto xw = rd<float>(tag + "_xw.f32"), nr = rd<float>(tag + "_normal.f32"), mx = rd<float>(tag + "_max.f32"), mn = rd<float>(tag + "_min.f32");
        auto qd = rd<uint8_t>(tag + "_desc.u8"), qbad = rd<uint8_t>(tag + "_bad.u8");
        auto qobs = rd<int>(tag + "_obs.i32");
        const int n = (int)mx.size();
        obj.resize(n);
        for (int j = 0; j < n; ++j) {
            MapPoint& p = obj[j];
            p.mock_id = j; p.mnId = j;
            p.mock_pos = Eigen::Vector3f(xw[3 * j], xw[3 * j + 1], xw[3 * j + 2]); p.mock_normal = Eigen::Vector3f(nr[3 * j], nr[3 * j + 1], nr[3 * j + 2]);
            p.mock_set_distances(mn[j], mx[j]);
            set_desc(p, &qd[(size_t)j * 32]);
            p.mock_bad = qbad[j] != 0;
            for (int k = 0; k < qobs[j]; ++k) {     // stand-ins for the observers that make up Observations()
                while ((int)others.size() <= k) others.push_back((KeyFrame*)(size_t)(0x1000 + 64 * others.size()));
                p.mock_obs[others[k]] = std::make_tuple(0, -1);
            }
        }
    }
};

// the target keyframe of Fuse and the Sim3 searches: features from t.kp / t_desc.u8 / t_ur.f32, pose t_T.f32, bounds from meta;
// feature i holds point t_slot[i] of `pts` (-1: none)
static KeyFrame* target_kf(int id, const float* cam6, const std::map<std::string, double>& M, QueryPoints& pts, bool observe) {
    auto k = rd<orbx_keypoint>("t.kp");
    auto d = rd<uint8_t>("t_desc.u8");
    auto ur = rd<float>("t_ur.f32"), T = rd<float>("t_T.f32");
    auto slot = rd<int>("t_slot.i32");
    KeyFrame* K = new KeyFrame(id, cam6[0], cam6[1], cam6[2], cam6[3], cam6[4], cam6[5], keys_of(k), ur, std::vector<float>(8, 1.f));
    const_cast<int&>(K->mnMinX) = (int)M.at("minx"); const_cast<int&>(K->mnMaxX) = (int)M.at("maxx");
    const_cast<int&>(K->mnMinY) = (int)M.at("miny"); const_cast<int&>(K->mnMaxY) = (int)M.at("maxy");
    K->mock_Tcw = se3_of(T.data());
    const_cast<cv::Mat&>(K->mDescriptors) = desc_mat(d);
    K->mock_matches.assign(k.size(), nullptr);
    for (size_t i = 0; i < k.size(); ++i)
        if (slot[i] >= 0) {
            K->mock_matches[i] = &pts.obj[slot[i]];
            if (observe) pts.obj[slot[i]].mock_obs[K] = std::make_tuple((int)i, -1);
        }
    return K;
}

static std::vector<int> ids_of(const std::vector<MapPoint*>& v) {
    std::vector<int> o(v.size());
    for (size_t i = 0; i < v.size(); ++i) o[i] = v[i] ? v[i]->mock_id : -1;
    return o;
}

extern "C" void* liba_mock_camera() { static double storage[4]; return storage; }

static int run_liba(std::map<std::string, double>& M);

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: host_units <dir>\n"); return 2; }
    g_dir = argv[1];
    auto M = read_meta();
    const std::string unit = [&] { std::ifstream f(g_dir + "/unit.txt"); std::string s; f >> s; return s; }();
    const float cam6[6] = {(float)M["fx"], (float)M["fy"], (float)M["cx"], (float)M["cy"], (float)M["bf"], (float)M["b"]};
    Frame::fx = cam6[0]; Frame::fy = cam6[1]; Frame::cx = cam6[2]; Frame::cy = cam6[3];
    Frame::mnMinX = (float)M["minx"]; Frame::mnMaxX = (float)M["maxx"]; Frame::mnMinY = (float)M["miny"]; Frame::mnMaxY = (float)M["maxy"];
    const int W = (int)M["W"], H = (int)M["H"], NF = (int)M["nfeatures"];
    std::vector<std::string> errors;   // orb_b200::Error messages the units threw, in order (the process carries on)
    auto guarded = [&](const std::function<void()>& f) {
        try { f(); } catch (const orb_b200::Error& e) { errors.push_back(e.what()); }
    };
    try {
        if (unit == "liba") return run_liba(M);
        ORBextractor ex(NF, M.count("scale") ? (float)M["scale"] : 1.2f, M.count("levels") ? (int)M["levels"] : 8, 20, 7);
        std::vector<uint64_t> handles;
        Extracted E = extract(ex, "img.u8", W, H, "frame");
        handles.push_back((uint64_t)(size_t)orb_b200_handle_of(&ex));
        Frame F;
        frame_of(F, &ex, E);
        if (M.count("frame_T")) F.mTcw = se3_of(rd<float>("frame_T.f32").data());

        if (unit == "bow") {                     // ---- SearchByBoW(KF, F) ----
            auto fnode = rd<int>("frame_node.i32");
            for (int i = 0; i < F.N; ++i) if (fnode[i] >= 0) F.mFeatVec[(DBoW2::NodeId)fnode[i]].push_back((unsigned int)i);
            MockKF K(1, "k1", cam6);
            ORBmatcher matcher((float)M["nnratio"], M["checkori"] != 0);
            std::vector<MapPoint*> vp(3, nullptr);          // the function resizes it
            const int ret = matcher.SearchByBoW(K.kf, F, vp);
            std::vector<int> out(vp.size());
            for (size_t i = 0; i < vp.size(); ++i) out[i] = K.index_of(vp[i]);
            out.push_back(ret);
            wr("out_bow.i32", out);
            // a frame of a fisheye rig is refused; nothing is searched
            F.Nleft = 5;
            guarded([&] { matcher.SearchByBoW(K.kf, F, vp); });
            F.Nleft = -1;
        } else if (unit == "bowkf") {            // ---- SearchByBoW(KF, KF) and SearchForTriangulation on the keyframe-search handle ----
            MockKF K1(1, "k1", cam6), K2(2, "k2", cam6);
            auto tri1 = rd<uint8_t>("k1_trihas.u8"), tri2 = rd<uint8_t>("k2_trihas.u8");
            ORBmatcher matcher((float)M["nnratio"], M["checkori"] != 0);
            std::vector<MapPoint*> vp12;
            std::vector<std::pair<size_t, size_t> > pairs;
            // no frame search yet and no handle named: both keyframe searches refuse, and the process carries on
            guarded([&] { matcher.SearchByBoW(K1.kf, K2.kf, vp12); });
            guarded([&] { matcher.SearchForTriangulation(K1.kf, K2.kf, pairs, false); });
            ORBextractor exO(NF, (float)M["other_scale"], (int)M["other_levels"], 20, 7);   // an extractor with other level tables
            if (M["use_other"] != 0) {
                extract(exO, "img.u8", W, H, "other");
                handles.push_back((uint64_t)(size_t)orb_b200_handle_of(&exO));
                orb_b200_use_handle_for_keyframe_searches(orb_b200_handle_of(&exO));
            } else {
                orb_b200_use_handle_for_keyframe_searches(orb_b200_handle_of(&ex));
            }
            vp12.assign(2, nullptr);
            const int rb = matcher.SearchByBoW(K1.kf, K2.kf, vp12);
            std::vector<int> fb(vp12.size());
            for (size_t i = 0; i < vp12.size(); ++i) fb[i] = K2.index_of(vp12[i]);
            fb.push_back(rb);
            wr("out_bowkf.i32", fb);
            if (M.count("big_n")) {                 // a host keyframe beyond ORB_MAX_FRAME_ROWS: refused, then the same handle still searches
                MockKF KB(3, "kb", cam6);
                guarded([&] { matcher.SearchByBoW(K1.kf, KB.kf, vp12); });
                const int again = matcher.SearchByBoW(K1.kf, K2.kf, vp12);
                wr("out_after_refusal.i32", std::vector<int>{again});
            }
            for (size_t i = 0; i < tri1.size(); ++i) K1.kf->mock_matches[i] = tri1[i] ? &K1.mps[i] : nullptr;
            for (size_t i = 0; i < tri2.size(); ++i) K2.kf->mock_matches[i] = tri2[i] ? &K2.mps[i] : nullptr;
            std::vector<int> fc;
            for (int combo = 0; combo < 4; ++combo) {       // bOnlyStereo x bCoarse
                pairs.assign(2, std::make_pair((size_t)7, (size_t)7));   // the function clears it
                const int rc = matcher.SearchForTriangulation(K1.kf, K2.kf, pairs, (combo & 1) != 0, (combo & 2) != 0);
                fc.push_back((int)pairs.size());
                for (auto& p : pairs) { fc.push_back((int)p.first); fc.push_back((int)p.second); }
                fc.push_back(rc);
            }
            wr("out_tri.i32", fc);
        } else if (unit == "init") {             // ---- SearchForInitialization: F1 from arrays, F2 = the extracted frame ----
            auto k1 = rd<orbx_keypoint>("f1.kp");
            auto d1 = rd<uint8_t>("f1_desc.u8");
            auto prev0 = rd<float>("f1_prev.f32");
            Frame F1;
            F1.N = (int)k1.size(); F1.mvKeys = keys_of(k1); F1.mvKeysUn = F1.mvKeys; F1.mDescriptors = desc_mat(d1);
            if (M["uploaded"] != 0) extract(ex, "img2.u8", W, H, "resident");   // another frame is on the device now: F2 is uploaded
            std::vector<cv::Point2f> prev(k1.size());
            for (size_t i = 0; i < k1.size(); ++i) prev[i] = cv::Point2f(prev0[2 * i], prev0[2 * i + 1]);
            std::vector<int> m12(3, 5);
            ORBmatcher matcher((float)M["nnratio"], M["checkori"] != 0);
            const int ret = matcher.SearchForInitialization(F1, F, prev, m12, (int)M["window"]);
            m12.push_back(ret);
            std::vector<float> pout;
            for (auto& p : prev) { pout.push_back(p.x); pout.push_back(p.y); }
            wr("out_init.i32", m12); wr("out_init_prev.f32", pout);
        } else if (unit == "reloc") {            // ---- SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) ----
            QueryPoints P("q");
            auto rk = rd<orbx_keypoint>("r.kp");
            auto slot = rd<int>("r_slot.i32");
            auto already = rd<uint8_t>("r_already.u8"), claimed = rd<uint8_t>("frame_claimed.u8");
            KeyFrame K1(9, cam6[0], cam6[1], cam6[2], cam6[3], cam6[4], cam6[5], keys_of(rk), std::vector<float>(rk.size(), -1.f), std::vector<float>(8, 1.f));
            K1.mock_matches.assign(rk.size(), nullptr);
            std::set<MapPoint*> found;
            for (size_t i = 0; i < rk.size(); ++i)
                if (slot[i] >= 0) { K1.mock_matches[i] = &P.obj[slot[i]]; if (already[slot[i]]) found.insert(&P.obj[slot[i]]); }
            MapPoint occupied;
            occupied.mock_id = -2;
            for (int i = 0; i < F.N; ++i) if (claimed[i]) F.mvpMapPoints[i] = &occupied;
            F.mbf = cam6[4]; F.mb = cam6[5];
            ORBmatcher matcher(0.9f, M["checkori"] != 0);
            const int ret = matcher.SearchByProjection(F, &K1, found, (float)M["th"], (int)M["orbdist"]);
            std::vector<int> out = ids_of(F.mvpMapPoints);
            out.push_back(ret);
            wr("out_reloc.i32", out);
        } else if (unit == "fuse") {             // ---- Fuse(pKF, vpMapPoints, th) ----
            orb_b200_use_handle_for_keyframe_searches(orb_b200_handle_of(&ex));
            QueryPoints P("q");
            KeyFrame* K = target_kf(7, cam6, M, P, true);
            auto qslot = rd<int>("q_slot.i32");
            auto qin = rd<uint8_t>("q_in_kf.u8");
            for (size_t j = 0; j < P.obj.size(); ++j) if (qin[j]) P.obj[j].mock_obs[K] = std::make_tuple(0, -1);
            std::vector<MapPoint*> vp(qslot.size());
            for (size_t i = 0; i < qslot.size(); ++i) vp[i] = qslot[i] < 0 ? nullptr : &P.obj[qslot[i]];
            ORBmatcher matcher(0.6f, true);
            const int ret = matcher.Fuse(K, vp, (float)M["th"]);
            std::vector<int> out = g_fuse_log;
            out.push_back(ret);
            wr("out_fuse_log.i32", out); wr("out_fuse_kf.i32", ids_of(K->mock_matches));
        } else if (unit == "sim3") {             // ---- SearchByProjection(pKF, Scw, ...) both overloads, Fuse(pKF, Scw, ...) ----
            orb_b200_use_handle_for_keyframe_searches(orb_b200_handle_of(&ex));
            auto sp = rd<float>("s_params.f32");      // quaternion x y z w (unit), translation, scale, th, ratioHamming
            auto matched0 = rd<int>("s_matched.i32");  // vpMatched on entry: point id, -2 = an occupying point, -1 = NULL
            Sophus::Sim3f Scw(sp[7], Eigen::Quaternionf(sp[3], sp[0], sp[1], sp[2]), Eigen::Vector3f(sp[4], sp[5], sp[6]));
            std::vector<int> out;
            {
                QueryPoints P("q");
                KeyFrame* K = target_kf(11, cam6, M, P, false);
                MapPoint occupied;
                occupied.mock_id = -2;
                std::vector<MapPoint*> vp(P.obj.size());
                for (size_t j = 0; j < vp.size(); ++j) vp[j] = &P.obj[j];
                std::vector<MapPoint*> vpMatched(matched0.size());
                for (size_t i = 0; i < matched0.size(); ++i) vpMatched[i] = matched0[i] == -2 ? &occupied : (matched0[i] >= 0 ? &P.obj[matched0[i]] : nullptr);
                std::vector<MapPoint*> vpMatchedB = vpMatched;
                ORBmatcher m3(0.75f, true);
                const int r1 = m3.SearchByProjection(K, Scw, vp, vpMatched, (int)sp[8], sp[9]);
                out = ids_of(vpMatched);
                out.push_back(r1);
                std::vector<KeyFrame*> fromKF(vp.size()), vpMatchedKF(matched0.size(), nullptr);
                for (size_t j = 0; j < vp.size(); ++j) fromKF[j] = (KeyFrame*)(size_t)(0x100000 + 64 * j);
                const int r2 = m3.SearchByProjection(K, Scw, vp, fromKF, vpMatchedB, vpMatchedKF, (int)sp[8], sp[9]);
                std::vector<int> b = ids_of(vpMatchedB);
                out.insert(out.end(), b.begin(), b.end());
                out.push_back(r2);
                for (auto* k : vpMatchedKF) out.push_back(k ? (int)(((size_t)k - 0x100000) / 64) : -1);
            }
            wr("out_sim3_proj.i32", out);
            {
                QueryPoints P("q");
                KeyFrame* K = target_kf(12, cam6, M, P, false);
                std::vector<MapPoint*> vp(P.obj.size()), repl(P.obj.size(), nullptr);
                for (size_t j = 0; j < vp.size(); ++j) vp[j] = &P.obj[j];
                ORBmatcher m3(0.75f, true);
                g_fuse_log.clear();
                const int r3 = m3.Fuse(K, Scw, vp, sp[8], repl);
                std::vector<int> o = ids_of(repl);
                o.push_back(r3);
                wr("out_sim3_fuse.i32", o); wr("out_sim3_fuse_log.i32", g_fuse_log); wr("out_sim3_fuse_kf.i32", ids_of(K->mock_matches));
            }
        } else if (unit == "voc") {              // ---- Frame::ComputeBoW: two frames against one vocabulary object ----
            auto co = rd<int>("child_offset.i32"), ci = rd<int>("child_ids.i32"), nw = rd<int>("node_word.i32");
            auto nd = rd<uint8_t>("node_desc.u8");
            auto wt = rd<double>("node_weight.f64");
            const int n = (int)nw.size();
            std::vector<ORBVocabulary::Node> nodes(n);
            for (int i = 0; i < n; ++i) {
                nodes[i].id = (DBoW2::NodeId)i;
                for (int c = co[i]; c < co[i + 1]; ++c) { nodes[i].children.push_back((DBoW2::NodeId)ci[c]); nodes[ci[c]].parent = (DBoW2::NodeId)i; }
                if (i > 0) { nodes[i].descriptor.create(1, 32, CV_8UC1); std::memcpy(nodes[i].descriptor.ptr(0), &nd[(size_t)i * 32], 32); }
                if (co[i] == co[i + 1]) { nodes[i].word_id = (DBoW2::WordId)nw[i]; nodes[i].weight = wt[i]; }
            }
            ORBVocabulary voc;
            voc.mock_set((int)M["L"], nodes);
            std::vector<int> out_i;
            std::vector<double> out_w;
            for (int pass = 0; pass < 2; ++pass) {
                Frame G;
                if (pass == 0) G = F;
                else frame_of(G, &ex, extract(ex, "img2.u8", W, H, "second"));
                G.mpORBvocabulary = &voc;
                G.ComputeBoW();
                const size_t before = G.mBowVec.size();
                G.ComputeBoW();                       // mBowVec is filled: returns at once
                out_i.push_back((int)(G.mBowVec.size() - before));
                out_i.push_back((int)G.mBowVec.size());
                for (const auto& kv : G.mBowVec) { out_i.push_back((int)kv.first); out_w.push_back(kv.second); }
                out_i.push_back((int)G.mFeatVec.size());
                for (const auto& kv : G.mFeatVec) {
                    out_i.push_back((int)kv.first); out_i.push_back((int)kv.second.size());
                    for (unsigned int f : kv.second) out_i.push_back((int)f);
                }
            }
            wr("out_voc.i32", out_i); wr("out_voc.f64", out_w);
        } else if (unit == "pose") {             // ---- Optimizer::PoseOptimization(Frame*) on the extracted frame ----
            auto xw = rd<float>("p_xw.f32"), ur = rd<float>("p_ur.f32"), isg = rd<float>("p_inv_sigma2.f32");
            auto has = rd<uint8_t>("p_has.u8");
            F.mvuRight = ur; F.mbf = cam6[4]; F.mb = cam6[5]; F.mvInvLevelSigma2 = isg;
            std::vector<MapPoint> mps(F.N);
            F.mvbOutlier.assign(F.N, true);              // true: the function must clear the flags it owns
            for (int i = 0; i < F.N; ++i)
                if (has[i]) { mps[i].mock_pos = Eigen::Vector3f(xw[3 * i], xw[3 * i + 1], xw[3 * i + 2]); F.mvpMapPoints[i] = &mps[i]; }
            const int ret = Optimizer::PoseOptimization(&F);
            const Sophus::SE3f T = F.GetPose();
            std::vector<float> pout = {T.unit_quaternion().x(), T.unit_quaternion().y(), T.unit_quaternion().z(), T.unit_quaternion().w(),
                                       T.translation()(0), T.translation()(1), T.translation()(2)};
            std::vector<uint8_t> outl(F.N);
            for (int i = 0; i < F.N; ++i) outl[i] = F.mvbOutlier[i] ? 1 : 0;
            wr("out_pose.f32", pout); wr("out_outlier.u8", outl); wr("out_pose_ret.i32", std::vector<int>{ret, F.mock_pose_sets});
        } else {
            std::fprintf(stderr, "unknown unit %s\n", unit.c_str());
            return 2;
        }
        wr("handles.u64", handles);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "host_units: %s\n", e.what());
        return 1;
    }
    std::string all;
    for (auto& e : errors) all += e + "\n";
    wr_raw("out_errors.txt", all.data(), all.size());
    std::printf("host_units ok\n");
    return 0;
}

static void fill3x3(Eigen::Matrix3f& Mx, const float* p) { for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Mx(r, c) = p[3 * r + c]; }

// ---- Optimizer::LocalInertialBA over the mock map of liba_cpu.cc (same inputs, same outputs) ----
static int run_liba(std::map<std::string, double>& M) {
    const float cam[5] = {(float)M["fx"], (float)M["fy"], (float)M["cx"], (float)M["cy"], (float)M["bf"]};
    const int nKF = (int)M["nkf"], nMP = (int)M["nmp"];
    auto pose = rd<float>("kf_pose.f32"), vel = rd<float>("kf_vel.f32"), bias = rd<float>("kf_bias.f32");
    auto flags = rd<int>("kf_flags.i32");
    auto pre = rd<float>("kf_pre.f32"), tcb = rd<float>("tcb.f32");
    auto pts = rd<float>("point.f32"), depth = rd<float>("point_track_depth.f32");
    auto badmp = rd<uint8_t>("point_bad.u8");
    auto ekf = rd<int>("edge_kf.i32"), emp = rd<int>("edge_mp.i32");
    auto eobs = rd<float>("edge_obs.f32"), ew = rd<float>("edge_inv_sigma2.f32");
    const int nE = (int)ekf.size();
    Map map;
    map.mock_n_keyframes = (long unsigned)M["keyframes_in_map"];
    std::vector<std::vector<cv::KeyPoint>> keys(nKF);
    std::vector<std::vector<float>> ur(nKF), sig(nKF);
    std::vector<int> featOf(nE);
    for (int e = 0; e < nE; ++e) {
        const int k = ekf[e];
        cv::KeyPoint kp;
        kp.pt.x = eobs[3 * e]; kp.pt.y = eobs[3 * e + 1]; kp.octave = (int)keys[k].size();
        featOf[e] = (int)keys[k].size();
        keys[k].push_back(kp); ur[k].push_back(eobs[3 * e + 2]); sig[k].push_back(ew[e]);
    }
    std::vector<KeyFrame*> kfs(nKF);
    std::vector<IMU::Preintegrated> pres(nKF);
    KeyFrame* block = (KeyFrame*)::operator new(sizeof(KeyFrame) * nKF);   // pointer order == index order (std::map<KeyFrame*, ...> iteration)
    const Sophus::SE3f Tcb = se3_of(tcb.data());
    for (int k = 0; k < nKF; ++k) {
        kfs[k] = new (block + k) KeyFrame(100 + k, cam[0], cam[1], cam[2], cam[3], cam[4], (float)M["b"], keys[k], ur[k], sig[k]);
        KeyFrame* K = kfs[k];
        K->mock_Tcw = se3_of(&pose[7 * k]);
        K->mock_map = &map;
        K->mock_bad = flags[4 * k + 2] != 0;
        K->mock_matches.assign(keys[k].size(), nullptr);
        K->mpCamera = reinterpret_cast<GeometricCamera*>(liba_mock_camera());
        K->bImu = flags[4 * k] != 0;
        K->mImuCalib.mTcb = Tcb; K->mImuCalib.mTbc = Tcb.inverse();
        K->mock_vel = Eigen::Vector3f(vel[3 * k], vel[3 * k + 1], vel[3 * k + 2]);
        const float* b = &bias[6 * k];
        K->mock_bias = IMU::Bias(b[0], b[1], b[2], b[3], b[4], b[5]);
        if (flags[4 * k + 3]) {
            const float* p = &pre[292 * (size_t)k];
            IMU::Preintegrated& P = pres[k];
            P.dT = p[0];
            for (int r = 0; r < 15; ++r) for (int c = 0; c < 15; ++c) P.C(r, c) = p[1 + 15 * r + c];
            P.b = IMU::Bias(p[226], p[227], p[228], p[229], p[230], p[231]);
            fill3x3(P.dR, p + 232);
            P.dV = Eigen::Vector3f(p[241], p[242], p[243]);
            P.dP = Eigen::Vector3f(p[244], p[245], p[246]);
            fill3x3(P.JRg, p + 247); fill3x3(P.JVg, p + 256); fill3x3(P.JVa, p + 265); fill3x3(P.JPg, p + 274); fill3x3(P.JPa, p + 283);
            K->mpImuPreintegrated = &P;
        }
    }
    for (int k = 0; k < nKF; ++k)
        if (flags[4 * k + 1] >= 0) kfs[k]->mPrevKF = kfs[flags[4 * k + 1]];
    std::vector<MapPoint> mps(nMP);
    for (int p = 0; p < nMP; ++p) {
        mps[p].mnId = 1000 + p; mps[p].mock_pos = Eigen::Vector3f(pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]);
        mps[p].mock_map = &map; mps[p].mock_bad = badmp[p] != 0; mps[p].mTrackDepth = depth[p];
    }
    for (int e = 0; e < nE; ++e) {
        mps[emp[e]].mock_obs[kfs[ekf[e]]] = std::make_tuple(featOf[e], -1);
        kfs[ekf[e]]->mock_matches[featOf[e]] = &mps[emp[e]];
    }
    bool stop = false;
    int nFixed = -7, nOpt = -7, nMPs = -7, nEdges = -7;
    Optimizer::LocalInertialBA(kfs[(int)M["ba_kf"]], &stop, &map, nFixed, nOpt, nMPs, nEdges, M["large"] != 0, M["rec_init"] != 0);
    std::vector<float> pout((size_t)nKF * 7), vout((size_t)nKF * 3), bout((size_t)nKF * 6), xout((size_t)nMP * 3);
    std::vector<int> counters = {nFixed, nOpt, nMPs, nEdges, map.mock_change_index};
    for (int k = 0; k < nKF; ++k) {
        const Sophus::SE3f T = kfs[k]->GetPose();
        float* o = &pout[(size_t)k * 7];
        o[0] = T.unit_quaternion().x(); o[1] = T.unit_quaternion().y(); o[2] = T.unit_quaternion().z(); o[3] = T.unit_quaternion().w();
        o[4] = T.translation()(0); o[5] = T.translation()(1); o[6] = T.translation()(2);
        for (int c = 0; c < 3; ++c) vout[3 * k + c] = kfs[k]->mock_vel(c);
        const IMU::Bias b = kfs[k]->mock_bias;
        const float bb[6] = {b.bax, b.bay, b.baz, b.bwx, b.bwy, b.bwz};
        for (int c = 0; c < 6; ++c) bout[6 * k + c] = bb[c];
        counters.push_back(kfs[k]->mock_pose_sets); counters.push_back(kfs[k]->mock_vel_sets); counters.push_back(kfs[k]->mock_bias_sets);
        counters.push_back(pres[k].mock_bias_sets); counters.push_back((int)kfs[k]->mnBALocalForKF); counters.push_back((int)kfs[k]->mnBAFixedForKF);
    }
    std::vector<int> alive(nE), updates(nMP);
    for (int p = 0; p < nMP; ++p) {
        const Eigen::Vector3f X = mps[p].GetWorldPos();
        xout[3 * p] = X(0); xout[3 * p + 1] = X(1); xout[3 * p + 2] = X(2);
        updates[p] = mps[p].mock_normal_updates;
    }
    for (int e = 0; e < nE; ++e)
        alive[e] = (kfs[ekf[e]]->mock_matches[featOf[e]] == &mps[emp[e]] ? 1 : 0) + (mps[emp[e]].mock_obs.count(kfs[ekf[e]]) ? 2 : 0);
    wr("out_pose.f32", pout); wr("out_vel.f32", vout); wr("out_bias.f32", bout); wr("out_point.f32", xout);
    wr("out_counters.i32", counters); wr("out_alive.i32", alive); wr("out_updates.i32", updates);
    std::printf("host_units ok\n");
    return 0;
}
