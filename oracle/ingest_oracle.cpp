// oracle/ingest_oracle.cpp -- TEST INFRASTRUCTURE (see oracle.h).
// What happens to a camera image before Frame::Frame: System::TrackStereo / TrackMonocular's cv::resize(im, newImSize, INTER_LINEAR)
// (System.cc:286-298), then Tracking::GrabImageStereo / GrabImageMonocular's cv::cvtColor to grey (Tracking.cc:1523-1601), restated
// for 8-bit images of 1, 3 or 4 interleaved channels.  Pinned against cv2 by tests/test_oracle_ingest_cpu.py.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace orb_oracle {

// cv::resize(u8, INTER_LINEAR) tap of one destination coordinate: source index and the two 11-bit coefficients (resize.cpp,
// resizeGeneric_ / HResizeLinear / VResizeLinear with VResizeLinearVec_32s8u).  Columns clamp the tap at both borders (xmin / xmax);
// rows keep the fraction and clip the two source rows when they are read.
static void tap(int d, double scale, int ssize, bool clamp, int& s, int& c0, int& c1) {
    float f = (float)((d + 0.5) * scale - 0.5);
    s = (int)std::floor(f);
    f -= (float)s;
    if (clamp && s < 0) { s = 0; f = 0.f; }
    if (clamp && s >= ssize - 1) { s = ssize - 1; f = 0.f; }
    c0 = (int)lrintf((1.f - f) * 2048.f);
    c1 = (int)lrintf(f * 2048.f);
}

// one channel of an interleaved image (pixel stride cn), resized; cv::resize with equal sizes copies
static void resize_channel(const uint8_t* src, int cn, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh) {
    if (sw == dw && sh == dh) {
        for (int y = 0; y < dh; ++y)
            for (int x = 0; x < dw; ++x) dst[(size_t)y * dw + x] = src[(size_t)y * sstride + (size_t)x * cn];
        return;
    }
    std::vector<int> xo(dw), xc0(dw), xc1(dw);
    for (int x = 0; x < dw; ++x) tap(x, (double)sw / dw, sw, true, xo[x], xc0[x], xc1[x]);
    std::vector<int> r0(dw), r1(dw);
    for (int y = 0; y < dh; ++y) {
        int sy, b0, b1;
        tap(y, (double)sh / dh, sh, false, sy, b0, b1);
        const uint8_t* a = src + (size_t)std::min(std::max(sy, 0), sh - 1) * sstride;
        const uint8_t* b = src + (size_t)std::min(std::max(sy + 1, 0), sh - 1) * sstride;
        for (int x = 0; x < dw; ++x) {
            const size_t x0 = (size_t)xo[x] * cn, x1 = (size_t)std::min(xo[x] + 1, sw - 1) * cn;
            r0[x] = a[x0] * xc0[x] + a[x1] * xc1[x];
            r1[x] = b[x0] * xc0[x] + b[x1] * xc1[x];
        }
        for (int x = 0; x < dw; ++x)
            dst[(size_t)y * dw + x] = (uint8_t)((((b0 * (r0[x] >> 4)) >> 16) + ((b1 * (r1[x] >> 4)) >> 16) + 2) >> 2);
    }
}

}  // namespace orb_oracle

using namespace orb_oracle;

extern "C" {

// cv::cvtColor(COLOR_BGR2GRAY) of one pixel: OpenCV's 15-bit fixed point (color_rgb.simd.hpp RGB2Gray<uchar>: BY15 3735, GY15 19235,
// RY15 9798, rounding 2^14)
uint8_t orc_bgr_to_gray(uint8_t b, uint8_t g, uint8_t r) { return (uint8_t)((b * 3735 + g * 19235 + r * 9798 + (1 << 14)) >> 15); }

// format: 0 grey, 1 RGB, 2 BGR, 3 RGBA, 4 BGRA (orb_image_format).  src: sw x sh pixels, rows sstride bytes apart; dst: dw x dh grey,
// tight.  Each of the first three channels is resized (when the sizes differ), then the pixel is converted; alpha is ignored.
int orc_ingest(const uint8_t* src, int format, int sw, int sh, int sstride, uint8_t* dst, int dw, int dh) {
    if (format < 0 || format > 4 || sw < 1 || sh < 1 || dw < 1 || dh < 1) return -1;
    const int cn = format == 0 ? 1 : format <= 2 ? 3 : 4;
    if (cn == 1) {
        resize_channel(src, 1, sw, sh, sstride, dst, dw, dh);
        return 0;
    }
    std::vector<uint8_t> ch[3];
    for (int c = 0; c < 3; ++c) {
        ch[c].resize((size_t)dw * dh);
        resize_channel(src + c, cn, sw, sh, sstride, ch[c].data(), dw, dh);
    }
    const bool rgb = format == 1 || format == 3;
    const std::vector<uint8_t>& B = rgb ? ch[2] : ch[0];
    const std::vector<uint8_t>& R = rgb ? ch[0] : ch[2];
    for (size_t i = 0; i < (size_t)dw * dh; ++i) dst[i] = orc_bgr_to_gray(B[i], ch[1][i], R[i]);
    return 0;
}

}  // extern "C"
