// refshim/opencv2/opencv.hpp -- a stand-in for the handful of OpenCV types that the reference's include/ORBextractor.h,
// ORBmatcher.h and the skeleton classes mention, so that the host translation units can be COMPILE-CHECKED against the
// reference's real class declarations and their marshaling RUN (tests/host/) in an image without OpenCV C++.  A real
// integration uses the real <opencv2/opencv.hpp>; nothing here is linked into liborbslam3_b200.so.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <vector>

#define CV_8U 0
#define CV_8UC1 0
#define CV_16U 2
#define CV_32F 5

namespace cv {

template <typename T>
struct Point_ {
    T x, y;
    Point_() : x(0), y(0) {}
    Point_(T x_, T y_) : x(x_), y(y_) {}
};
typedef Point_<int> Point2i;
typedef Point_<int> Point;
typedef Point_<float> Point2f;

struct KeyPoint {
    Point2f pt;
    float size, angle, response;
    int octave, class_id;
    KeyPoint() : size(0), angle(-1), response(0), octave(0), class_id(-1) {}
};

class Mat {
   public:
    int rows = 0, cols = 0;
    uint8_t* data = nullptr;
    size_t step = 0;
    Mat() {}
    Mat(int r, int c, int /*type*/) { create(r, c, 0); }
    // over external data of any element type (a CV_32F depth map: Frame::ComputeStereoFromRGBD); the owning forms are 8-bit only
    Mat(int r, int c, int type, void* ext, size_t stp) : rows(r), cols(c), data((uint8_t*)ext), step(stp), type_(type) {}
    void create(int r, int c, int /*type*/) {
        rows = r; cols = c; step = (size_t)c;
        store_.reset(new std::vector<uint8_t>((size_t)r * c));
        data = store_->data();
    }
    void release() { rows = cols = 0; data = nullptr; store_.reset(); }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    int type() const { return type_; }
    bool isContinuous() const { return step == (size_t)cols; }
    uint8_t* ptr(int r = 0) { return data + (size_t)r * step; }
    const uint8_t* ptr(int r = 0) const { return data + (size_t)r * step; }
    template <typename T> T* ptr(int r = 0) { return reinterpret_cast<T*>(data + (size_t)r * step); }
    template <typename T> const T* ptr(int r = 0) const { return reinterpret_cast<const T*>(data + (size_t)r * step); }
    Mat row(int r) const { Mat m; m.rows = 1; m.cols = cols; m.step = step; m.data = data + (size_t)r * step; m.type_ = type_; m.store_ = store_; return m; }
    Mat clone() const { Mat m; if (!empty()) { m.create(rows, cols, 0); for (int r = 0; r < rows; ++r) std::memcpy(m.ptr(r), ptr(r), (size_t)cols); } return m; }

   private:
    int type_ = CV_8UC1;
    std::shared_ptr<std::vector<uint8_t>> store_;
};

// InputArray / OutputArray reduced to "a reference to a Mat"
class _InputArray {
   public:
    _InputArray() : m_(nullptr) {}
    _InputArray(const Mat& m) : m_(const_cast<Mat*>(&m)) {}
    Mat getMat() const { return m_ ? *m_ : Mat(); }
    bool empty() const { return !m_ || m_->empty(); }

   protected:
    Mat* m_;
};
class _OutputArray : public _InputArray {
   public:
    _OutputArray() {}
    _OutputArray(Mat& m) { m_ = &m; }
    void create(int r, int c, int t) const { if (m_) m_->create(r, c, t); }
    void release() const { if (m_) m_->release(); }
};
typedef const _InputArray& InputArray;
typedef const _OutputArray& OutputArray;

}  // namespace cv
