// ORBextractor_b200.cc -- drop-in replacement for /root/reference/src/ORBextractor.cc.
//
// Compiled AGAINST THE REFERENCE'S OWN HEADER (include/ORBextractor.h, unchanged) and linked with
// liborbslam3_b200.so instead of the reference's ORBextractor.cc, it gives Tracking / Frame the same
// ORB_SLAM3::ORBextractor class: same constructor, same operator(), same getters, mvImagePyramid populated.
// All arithmetic happens on the GPU behind the C ABI (include/orbslam3_b200.h); this file only marshals.
//
//   g++ -std=c++14 -I<ORB_SLAM3>/include -I<this repo>/include $(pkg-config --cflags opencv4) \
//       -c ORBextractor_b200.cc            # then link -lorbslam3_b200 in place of ORBextractor.o
//
// The reference class has no spare member and an inline empty destructor, so the device handle lives in a
// side table keyed by `this` (three extractors per session: left, right, ini -- Tracking.cc:629-635); the table's
// destructor releases every handle at process exit, orb_b200_release() releases one earlier.
//
// The reference constructor takes no image size.  A handle starts at ORB_B200_MAX_WIDTH x ORB_B200_MAX_HEIGHT; operator() re-creates it
// for a larger image (each side grows to the larger of the two, never shrinks) and the side table then maps `this` to the new handle,
// which the stereo and matcher units look up per call.
#include <algorithm>
#include <cassert>
#include <cstring>
#include <mutex>
#include <unordered_map>

#include "ORBextractor.h"      // the reference's header
#include "orb_b200_host.h"

#ifndef ORB_B200_MAX_WIDTH
#define ORB_B200_MAX_WIDTH 1280
#endif
#ifndef ORB_B200_MAX_HEIGHT
#define ORB_B200_MAX_HEIGHT 1024
#endif
#ifndef ORB_B200_MATERIALIZE_PYRAMID
#define ORB_B200_MATERIALIZE_PYRAMID 1   // only the reference's own Frame::ComputeStereoMatches reads mvImagePyramid (Frame.cc:1249,1275);
#endif                                   // with host/Frame_stereo_b200.cc linked, build with 0 and the pyramid never leaves the device

namespace {
struct Registry {
    std::mutex mu;
    std::unordered_map<const void*, orbx_handle*> handles;
    std::unordered_map<const void*, orbx_config> configs;   // the configuration each handle was created with
    lba_handle* lba = nullptr;
    ~Registry() {
        for (auto& kv : handles) orbx_destroy(kv.second);
        if (lba) lba_destroy(lba);
    }
};
Registry& registry() {
    static Registry r;
    return r;
}
}  // namespace

extern "C" orbx_handle* orb_b200_handle_of(const void* extractor) {
    Registry& r = registry();
    std::lock_guard<std::mutex> lk(r.mu);
    auto it = r.handles.find(extractor);
    return it == r.handles.end() ? nullptr : it->second;
}

extern "C" void orb_b200_release(const void* extractor) {
    Registry& r = registry();
    std::lock_guard<std::mutex> lk(r.mu);
    auto it = r.handles.find(extractor);
    if (it == r.handles.end()) return;
    orbx_destroy(it->second);
    r.handles.erase(it);
    r.configs.erase(extractor);
}

// the handle of `extractor`, re-created first when the image is larger than it was sized for
static orbx_handle* handle_for_image(const void* extractor, int w, int h) {
    Registry& r = registry();
    std::lock_guard<std::mutex> lk(r.mu);
    orbx_handle* cur = r.handles.at(extractor);
    orbx_config cfg = r.configs.at(extractor);
    if (w <= cfg.max_width && h <= cfg.max_height) return cur;
    cfg.max_width = std::max(cfg.max_width, w);
    cfg.max_height = std::max(cfg.max_height, h);
    orbx_destroy(cur);            // first: the old and the new workspace need not fit on the device together
    r.handles.erase(extractor);
    r.configs.erase(extractor);
    orbx_handle* grown = nullptr;
    orb_b200::check(orbx_create(&cfg, &grown), "orbx_create (grow to the image size)");
    r.handles[extractor] = grown;
    r.configs[extractor] = cfg;
    return grown;
}

extern "C" lba_handle* orb_b200_lba_handle(void) {
    Registry& r = registry();
    std::lock_guard<std::mutex> lk(r.mu);
    if (!r.lba) orb_b200::check(lba_create(orb_b200::device_ordinal(), &r.lba), "lba_create");
    return r.lba;
}

namespace ORB_SLAM3 {

// ORBextractor.cc:468-571
ORBextractor::ORBextractor(int _nfeatures, float _scaleFactor, int _nlevels, int _iniThFAST, int _minThFAST)
    : nfeatures(_nfeatures), scaleFactor(_scaleFactor), nlevels(_nlevels), iniThFAST(_iniThFAST), minThFAST(_minThFAST) {
    orbx_config cfg;
    cfg.n_features = _nfeatures;
    cfg.scale_factor = _scaleFactor;
    cfg.n_levels = _nlevels;
    cfg.ini_th_fast = _iniThFAST;
    cfg.min_th_fast = _minThFAST;
    cfg.max_width = ORB_B200_MAX_WIDTH;
    cfg.max_height = ORB_B200_MAX_HEIGHT;
    cfg.max_batch = 1;
    cfg.device = orb_b200::device_ordinal();
    orbx_handle* h = nullptr;
    orb_b200::check(orbx_create(&cfg, &h), "orbx_create");
    {
        Registry& r = registry();
        std::lock_guard<std::mutex> lk(r.mu);
        auto old = r.handles.find(this);          // an extractor destroyed and another constructed at the same address
        if (old != r.handles.end()) orbx_destroy(old->second);
        r.handles[this] = h;
        r.configs[this] = cfg;
    }
    mvScaleFactor.resize(nlevels);
    mvInvScaleFactor.resize(nlevels);
    mvLevelSigma2.resize(nlevels);
    mvInvLevelSigma2.resize(nlevels);
    mnFeaturesPerLevel.resize(nlevels);
    umax.resize(16);
    orbx_get_tables(h, mvScaleFactor.data(), mvInvScaleFactor.data(), mvLevelSigma2.data(), mvInvLevelSigma2.data(),
                    mnFeaturesPerLevel.data(), umax.data());
    mvImagePyramid.resize(nlevels);
}

// ORBextractor.cc:1557-1682
int ORBextractor::operator()(cv::InputArray _image, cv::InputArray /*_mask*/, std::vector<cv::KeyPoint>& _keypoints,
                             cv::OutputArray _descriptors, std::vector<int>& vLappingArea) {
    if (_image.empty()) return -1;
    cv::Mat image = _image.getMat();
    assert(image.type() == CV_8UC1);
    orbx_handle* h = handle_for_image(this, image.cols, image.rows);
    static_assert(sizeof(cv::KeyPoint) == sizeof(orbx_keypoint), "cv::KeyPoint layout");
    const int cap = orbx_max_features(h);
    std::vector<cv::KeyPoint> kps(cap);
    int n = 0, mono = 0;
    const int lap0 = vLappingArea.size() > 0 ? vLappingArea[0] : 0, lap1 = vLappingArea.size() > 1 ? vLappingArea[1] : 0;
    // descriptors land in a scratch block first: _descriptors must be created with exactly n rows, and n is an output
    static thread_local std::vector<unsigned char> desc;
    desc.resize((size_t)cap * 32);
    orb_b200::check(orbx_extract(h, image.data, image.cols, image.rows, (int)image.step, lap0, lap1,
                                 reinterpret_cast<orbx_keypoint*>(kps.data()), desc.data(), cap, &n, &mono), "orbx_extract");
    kps.resize(n);
    _keypoints.swap(kps);
    if (n == 0) {
        _descriptors.release();
    } else {
        _descriptors.create(n, 32, CV_8U);
        cv::Mat d = _descriptors.getMat();
        if (d.isContinuous()) std::memcpy(d.ptr(0), desc.data(), (size_t)n * 32);
        else for (int i = 0; i < n; ++i) std::memcpy(d.ptr(i), &desc[(size_t)i * 32], 32);
    }
#if ORB_B200_MATERIALIZE_PYRAMID
    {   // all levels queued on the handle's stream, ONE synchronisation
        std::vector<unsigned char*> dst(nlevels);
        std::vector<int> stride(nlevels);
        for (int l = 0; l < nlevels; ++l) {
            int w = 0, hh = 0;
            orbx_level_size(h, l, &w, &hh);
            mvImagePyramid[l].create(hh, w, CV_8UC1);
            dst[l] = mvImagePyramid[l].data;
            stride[l] = (int)mvImagePyramid[l].step;
        }
        orb_b200::check(orbx_download_pyramid(h, 0, 0, dst.data(), stride.data()), "orbx_download_pyramid");
    }
#endif
    return mono;
}

}  // namespace ORB_SLAM3
