// exporter_ref facade — TEST INFRASTRUCTURE ONLY (oracle/exporter_ref, never linked into the product).
//
// The slice of an OpenCV-*shaped* cv:: API, written from scratch, that the reference's export/Exporter.cpp and the
// headers it includes use, so that unit compiles in place (oracle/exporter_ref/build.py) in an image without OpenCV C++
// headers.  Only u8 matrices exist.  Mat bookkeeping (headers, ref-counted buffers, views, create / copyTo / clone /
// setTo) is native; every pixel operation is forwarded to the real OpenCV kernel in cv2 (facade.cpp).
#pragma once

#include <cstddef>
#include <cstdint>
#include <memory>
#include <stdexcept>

#define CV_8U 0
#define CV_CN_SHIFT 3
#define CV_MAT_DEPTH(t) ((t) & 7)
#define CV_MAT_CN(t) ((((t) >> CV_CN_SHIFT) & 511) + 1)
#define CV_MAKETYPE(depth, cn) (CV_MAT_DEPTH(depth) + (((cn) - 1) << CV_CN_SHIFT))
#define CV_8UC1 CV_MAKETYPE(CV_8U, 1)
#define CV_8UC3 CV_MAKETYPE(CV_8U, 3)

namespace cv {

typedef unsigned char uchar;

struct Size {
    int width = 0, height = 0;
    Size() = default;
    Size(int w, int h) : width(w), height(h) {}
};
inline bool operator==(const Size& a, const Size& b) { return a.width == b.width && a.height == b.height; }
inline bool operator!=(const Size& a, const Size& b) { return !(a == b); }

struct Point {
    int x = 0, y = 0;
    Point() = default;
    Point(int x_, int y_) : x(x_), y(y_) {}
};

struct Rect {
    int x = 0, y = 0, width = 0, height = 0;
    Rect() = default;
    Rect(int x_, int y_, int w, int h) : x(x_), y(y_), width(w), height(h) {}
    // intersection, as OpenCV's Rect_::operator&=: an empty result is all zeros
    Rect& operator&=(const Rect& r) {
        const int x0 = x > r.x ? x : r.x, y0 = y > r.y ? y : r.y;
        const int x1 = x + width < r.x + r.width ? x + width : r.x + r.width;
        const int y1 = y + height < r.y + r.height ? y + height : r.y + r.height;
        *this = x1 <= x0 || y1 <= y0 ? Rect() : Rect(x0, y0, x1 - x0, y1 - y0);
        return *this;
    }
};

struct Scalar {
    double val[4] = {0, 0, 0, 0};
    Scalar() = default;
    Scalar(double v0, double v1 = 0, double v2 = 0, double v3 = 0) : val{v0, v1, v2, v3} {}
    double operator[](int i) const { return val[i]; }
};

class Mat {
public:
    int flags = 0;   // the type (u8, 1..4 channels)
    int rows = 0, cols = 0;
    uchar* data = nullptr;
    size_t step = 0;   // bytes per row

    Mat() = default;
    Mat(int r, int c, int type) { create(r, c, type); }
    Mat(Size s, int type, const Scalar& v) { create(s.height, s.width, type); setTo(v); }
    Mat(const Mat& m, const Rect& roi);   // view

    int type() const { return flags; }
    int channels() const { return CV_MAT_CN(flags); }
    bool empty() const { return data == nullptr || rows == 0 || cols == 0; }
    Size size() const { return Size(cols, rows); }

    // OpenCV's create(): keeps the buffer (a view's too) when size and type already match, else allocates a fresh one
    void create(int r, int c, int type);
    template <typename T> T* ptr(int row = 0) { return reinterpret_cast<T*>(data + (size_t)row * step); }
    template <typename T> const T* ptr(int row = 0) const { return reinterpret_cast<const T*>(data + (size_t)row * step); }

    Mat clone() const;
    void copyTo(Mat& dst) const;
    void copyTo(Mat&& dst) const { copyTo(dst); }   // into a view such as canvas(roi), as OpenCV's OutputArray allows
    Mat& setTo(const Scalar& s);
    Mat operator()(const Rect& roi) const { return Mat(*this, roi); }

private:
    std::shared_ptr<uchar[]> buf_;
};

}  // namespace cv
