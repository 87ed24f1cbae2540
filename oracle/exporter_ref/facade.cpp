// exporter_ref facade — TEST INFRASTRUCTURE ONLY.  Mat bookkeeping natively, pixel operations through the `cv2` Python
// module (pybind11; the GIL is held because this code only runs inside calls made from Python into _exporter_ref).
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>

#include <cstring>
#include <vector>

#include "opencv2/core.hpp"
#include "opencv2/imgproc.hpp"

namespace py = pybind11;

namespace cv {

void Mat::create(int r, int c, int type) {
    if (data && rows == r && cols == c && flags == type) return;
    if (CV_MAT_DEPTH(type) != CV_8U) throw std::runtime_error("exporter_ref facade: u8 only");
    flags = type;
    rows = r;
    cols = c;
    step = (size_t)c * (size_t)CV_MAT_CN(type);
    const size_t n = step * (size_t)r;
    buf_ = std::shared_ptr<uchar[]>(new uchar[n ? n : 1]());
    data = buf_.get();
}

Mat::Mat(const Mat& m, const Rect& roi) : Mat(m) {
    if (roi.x < 0 || roi.y < 0 || roi.width < 0 || roi.height < 0 || roi.x + roi.width > m.cols || roi.y + roi.height > m.rows)
        throw std::runtime_error("exporter_ref facade: roi outside the matrix");
    data = m.data + (size_t)roi.y * m.step + (size_t)roi.x * m.channels();
    rows = roi.height;
    cols = roi.width;
}

void Mat::copyTo(Mat& dst) const {
    if (empty()) { dst = Mat(); return; }
    const Mat src = *this;   // keeps the source alive if dst re-allocates
    dst.create(rows, cols, flags);
    if (dst.data == src.data && dst.step == src.step) return;
    for (int y = 0; y < rows; ++y) std::memmove(dst.ptr<uchar>(y), src.ptr<uchar>(y), (size_t)cols * channels());
}

Mat Mat::clone() const {
    Mat m;
    copyTo(m);
    return m;
}

Mat& Mat::setTo(const Scalar& s) {
    const int cn = channels();
    for (int y = 0; y < rows; ++y)
        for (int x = 0; x < cols; ++x)
            for (int c = 0; c < cn; ++c) ptr<uchar>(y)[x * cn + c] = (uchar)s[c & 3];
    return *this;
}

namespace {

py::object cv2() {
    static py::object* m = new py::object(py::module_::import("cv2"));   // leaked on purpose (no dtor at exit)
    return *m;
}

// zero-copy numpy view of a Mat (the Mat outlives the call)
py::array view(const Mat& m) {
    std::vector<ssize_t> shape{m.rows, m.cols}, strides{(ssize_t)m.step, (ssize_t)m.channels()};
    if (m.channels() > 1) { shape.push_back(m.channels()); strides.push_back(1); }
    static int anchor = 0;
    static py::object* keep = new py::object(py::capsule(&anchor, [](void*) {}));
    return py::array(py::dtype::of<uint8_t>(), shape, strides, m.data, *keep);
}

// a cv2 result into dst with create() semantics: into dst's own rows (a view's too) when size and type match
void store(const py::handle& obj, Mat& dst) {
    py::array_t<uint8_t, py::array::c_style | py::array::forcecast> a(py::reinterpret_borrow<py::object>(obj));
    const int rows = (int)a.shape(0), cols = (int)a.shape(1), cn = a.ndim() == 3 ? (int)a.shape(2) : 1;
    dst.create(rows, cols, CV_MAKETYPE(CV_8U, cn));
    for (int y = 0; y < rows; ++y) std::memmove(dst.ptr<uchar>(y), a.data(y), (size_t)cols * cn);
}

}  // namespace

void cvtColor(const Mat& src, Mat& dst, int code) { store(cv2().attr("cvtColor")(view(src), code), dst); }

void resize(const Mat& src, Mat& dst, Size dsize, double fx, double fy, int interpolation) {
    store(cv2().attr("resize")(view(src), py::make_tuple(dsize.width, dsize.height), py::arg("fx") = fx, py::arg("fy") = fy,
                               py::arg("interpolation") = interpolation),
          dst);
}

void addWeighted(const Mat& a, double alpha, const Mat& b, double beta, double gamma, Mat& dst) {
    store(cv2().attr("addWeighted")(view(a), alpha, view(b), beta, gamma), dst);
}

Size getTextSize(const std::string& text, int fontFace, double fontScale, int thickness, int* baseLine) {
    py::tuple t = cv2().attr("getTextSize")(text, fontFace, fontScale, thickness);
    py::tuple sz = t[0];
    if (baseLine) *baseLine = t[1].cast<int>();
    return Size(sz[0].cast<int>(), sz[1].cast<int>());
}

void putText(Mat& img, const std::string& text, Point org, int fontFace, double fontScale, Scalar color, int thickness,
             int lineType, bool bottomLeftOrigin) {
    // cv2 draws into the array in place; the result is stored back as well, in case it had to copy
    store(cv2().attr("putText")(view(img), text, py::make_tuple(org.x, org.y), fontFace, fontScale,
                                py::make_tuple(color[0], color[1], color[2], color[3]), thickness, lineType, bottomLeftOrigin),
          img);
}

}  // namespace cv
