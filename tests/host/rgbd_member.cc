// tests/host/rgbd_member.cc -- runs Frame::ComputeStereoFromRGBD (host/Frame_stereo_b200.cc) the way the reference's RGB-D Frame
// constructor does, through the reference's own class declarations over the skeletons of host/refshim, then the drop-in
// ORBmatcher::SearchByProjection(F, vpMapPoints) on that frame.  Inputs and outputs are raw arrays in a scratch directory;
// tests/test_zz_rgbd_member_gpu.py writes the inputs and compares the outputs with the oracle.
//   rgbd_member <dir>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>
#include <string>
#include <vector>

#include "ref_skeleton_impl.h"   // also brings the reference's ORBextractor.h
#include "ORBmatcher.h"
#include "orb_b200_host.h"

using namespace ORB_SLAM3;

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
template <typename T>
static void wr(const std::string& name, const std::vector<T>& v) {
    std::ofstream f(g_dir + "/" + name, std::ios::binary);
    f.write((const char*)v.data(), (std::streamsize)(v.size() * sizeof(T)));
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: rgbd_member <dir>\n"); return 2; }
    g_dir = argv[1];
    std::map<std::string, double> M;
    {
        std::ifstream f(g_dir + "/meta.txt");
        std::string k;
        double v;
        while (f >> k >> v) M[k] = v;
    }
    const int W = (int)M["W"], H = (int)M["H"], NF = (int)M["nfeatures"];
    try {
        // ---- the RGB-D Frame constructor: ExtractORB(0, imGray, 0, 0), mvKeysUn = mvKeys, ComputeStereoFromRGBD(imDepth) ----
        std::vector<uint8_t> img = rd<uint8_t>("grey.u8");
        std::vector<float> depth = rd<float>("depth.f32");        // what GrabImageRGBD's convertTo left: CV_32F metres
        ORBextractor ex(NF, 1.2f, 8, 20, 7);
        cv::Mat mImg(H, W, CV_8UC1, img.data(), (size_t)W), d;
        std::vector<cv::KeyPoint> k;
        std::vector<int> lap = {0, 0};
        ex(mImg, cv::Mat(), k, d, lap);
        Frame::fx = (float)M["fx"]; Frame::fy = (float)M["fy"]; Frame::cx = (float)M["cx"]; Frame::cy = (float)M["cy"];
        Frame::mnMinX = 0; Frame::mnMaxX = (float)W; Frame::mnMinY = 0; Frame::mnMaxY = (float)H;
        Frame F;
        F.mpORBextractorLeft = &ex;
        F.mbf = (float)M["bf"]; F.mb = F.mbf / Frame::fx;
        F.N = (int)k.size();
        F.mvKeys = k; F.mvKeysUn = k;
        F.mDescriptors = d;
        F.mvpMapPoints.assign(F.N, nullptr);
        F.mvbOutlier.assign(F.N, false);
        F.ComputeStereoFromRGBD(cv::Mat(H, W, CV_32F, depth.data(), (size_t)W * 4));
        std::vector<uint8_t> kb((const uint8_t*)k.data(), (const uint8_t*)k.data() + k.size() * 28);
        wr("out_kps.bin", kb);
        wr("out_uright.f32", F.mvuRight);
        wr("out_depth.f32", F.mvDepth);
        // ---- SearchByProjection(F, vpMapPoints, th) on that frame: its mvuRight is read from the device ----
        const int nq = (int)M["loc_n"];
        auto px = rd<float>("loc_px.f32"), py = rd<float>("loc_py.f32"), pxr = rd<float>("loc_pxr.f32"), vc = rd<float>("loc_vcos.f32"),
             dep = rd<float>("loc_depth.f32");
        auto lv = rd<int>("loc_level.i32");
        auto qd = rd<uint8_t>("loc_desc.u8");
        std::vector<MapPoint> mps(nq);
        std::vector<MapPoint*> vp(nq);
        KeyFrame dummyKF(0, 1, 1, 0, 0, 1, 1, {}, {}, {});
        for (int i = 0; i < nq; ++i) {
            MapPoint& p = mps[i];
            p.mnId = i; p.mTrackProjX = px[i]; p.mTrackProjY = py[i]; p.mTrackProjXR = pxr[i]; p.mnTrackScaleLevel = lv[i];
            p.mTrackViewCos = vc[i]; p.mTrackDepth = dep[i]; p.mbTrackInView = true;
            p.mock_desc = cv::Mat(1, 32, CV_8U);
            std::memcpy(p.mock_desc.data, &qd[(size_t)i * 32], 32);
            p.mock_obs[&dummyKF] = std::make_tuple(0, -1);
            vp[i] = &p;
        }
        ORBmatcher matcher((float)M["loc_nnratio"], true);
        const int nm = matcher.SearchByProjection(F, vp, (float)M["loc_th"], false, 50.0f);
        std::vector<int> res(F.N + 1, -1);
        for (int i = 0; i < F.N; ++i) res[i] = F.mvpMapPoints[i] ? (int)(F.mvpMapPoints[i] - mps.data()) : -1;
        res[F.N] = nm;
        wr("out_local.i32", res);
        orb_b200_release(&ex);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "error: %s\n", e.what());
        return 1;
    }
    return 0;
}
