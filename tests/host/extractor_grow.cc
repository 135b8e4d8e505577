// tests/host/extractor_grow.cc -- the drop-in ORB_SLAM3::ORBextractor (host/ORBextractor_b200.cc), created at its compile-time default
// size, fed frames of growing size through the reference's own class declarations; for every frame also Frame::ComputeStereoMatches
// (host/Frame_stereo_b200.cc) on the same extractors.  tests/test_zz_large_frames_gpu.py builds it, writes the inputs and compares the
// outputs with the oracle.
//   extractor_grow <dir>      inputs: meta.txt (n, nfeatures, fx, fy, cx, cy, bf, b, W<k>, H<k>), left<k>.u8, right<k>.u8
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>
#include <string>
#include <vector>

#include "ref_skeleton_impl.h"   // also brings the reference's ORBextractor.h
#include "orb_b200_host.h"

using namespace ORB_SLAM3;

static std::string g_dir;
static std::vector<uint8_t> rd(const std::string& name) {
    std::ifstream f(g_dir + "/" + name, std::ios::binary);
    if (!f) { std::fprintf(stderr, "missing input %s\n", name.c_str()); std::exit(2); }
    f.seekg(0, std::ios::end);
    std::vector<uint8_t> v((size_t)f.tellg());
    f.seekg(0);
    f.read((char*)v.data(), (std::streamsize)v.size());
    return v;
}
template <typename T>
static void wr(const std::string& name, const std::vector<T>& v) {
    std::ofstream f(g_dir + "/" + name, std::ios::binary);
    f.write((const char*)v.data(), (std::streamsize)(v.size() * sizeof(T)));
}

int main(int argc, char** argv) {
    if (argc < 2) { std::fprintf(stderr, "usage: extractor_grow <dir>\n"); return 2; }
    g_dir = argv[1];
    std::map<std::string, double> M;
    {
        std::ifstream f(g_dir + "/meta.txt");
        std::string k;
        double v;
        while (f >> k >> v) M[k] = v;
    }
    try {
        const int NF = (int)M["nfeatures"];
        ORBextractor exL(NF, 1.2f, 8, 20, 7), exR(NF, 1.2f, 8, 20, 7);
        for (int k = 0; k < (int)M["n"]; ++k) {
            const std::string s = std::to_string(k);
            const int W = (int)M["W" + s], H = (int)M["H" + s];
            std::vector<uint8_t> imgL = rd("left" + s + ".u8"), imgR = rd("right" + s + ".u8");
            cv::Mat mL(H, W, CV_8UC1, imgL.data(), (size_t)W), mR(H, W, CV_8UC1, imgR.data(), (size_t)W), dL, dR;
            std::vector<cv::KeyPoint> kL, kR;
            std::vector<int> lap = {0, 0};
            const int monoL = exL(mL, cv::Mat(), kL, dL, lap), monoR = exR(mR, cv::Mat(), kR, dR, lap);
            wr("out_kpsL" + s + ".bin", std::vector<uint8_t>((const uint8_t*)kL.data(), (const uint8_t*)kL.data() + kL.size() * 28));
            wr("out_kpsR" + s + ".bin", std::vector<uint8_t>((const uint8_t*)kR.data(), (const uint8_t*)kR.data() + kR.size() * 28));
            std::vector<uint8_t> d((size_t)kL.size() * 32);
            for (size_t i = 0; i < kL.size(); ++i) std::memcpy(&d[i * 32], dL.ptr((int)i), 32);
            wr("out_descL" + s + ".bin", d);
            wr("out_mono" + s + ".i32", std::vector<int>{monoL, monoR});
            // Frame::ComputeStereoMatches on the pair the extractors just produced
            Frame::fx = (float)M["fx"]; Frame::fy = (float)M["fy"]; Frame::cx = (float)M["cx"]; Frame::cy = (float)M["cy"];
            Frame::mnMinX = 0; Frame::mnMaxX = (float)W; Frame::mnMinY = 0; Frame::mnMaxY = (float)H;
            Frame F;
            F.mpORBextractorLeft = &exL; F.mpORBextractorRight = &exR;
            F.mbf = (float)M["bf"]; F.mb = (float)M["b"];
            F.N = (int)kL.size();
            F.mvKeys = kL; F.mvKeysUn = kL; F.mvKeysRight = kR;
            F.mDescriptors = dL;
            F.mvpMapPoints.assign(F.N, nullptr);
            F.mvbOutlier.assign(F.N, false);
            F.ComputeStereoMatches();
            wr("out_uright" + s + ".f32", F.mvuRight);
            wr("out_depth" + s + ".f32", F.mvDepth);
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "exception: %s\n", e.what());
        return 1;
    }
    return 0;
}
