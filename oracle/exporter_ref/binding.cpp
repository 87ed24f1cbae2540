// _exporter_ref — TEST INFRASTRUCTURE ONLY (oracle/exporter_ref).  The reference exporter's own canvas: compose(orig,
// proc, split, overlay) with drawLabel's "Original" / "Processed" labels (export/Exporter.cpp:25-88).  Both live in an
// anonymous namespace of Exporter.cpp, so this unit compiles that file in place by including it, against the facade in
// this directory, and binds compose().
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>

#include <cstring>

#include "export/Exporter.cpp"

namespace py = pybind11;

// Exporter::run, compiled with the unit but never called here, drives the magnification chain.  That chain is pinned by
// _livim_ref (oracle/build_ref.py); this module binds only compose(), so the chain's two entry points are placeholders.
namespace livim {
std::vector<std::unique_ptr<IProcessor>> buildProcessors() { throw std::logic_error("_exporter_ref binds compose() only"); }
FrameRef runChainOnce(const std::vector<std::unique_ptr<IProcessor>>&, const FrameRef&, const ProcessorConfig&, FrameRef&) {
    throw std::logic_error("_exporter_ref binds compose() only");
}
}  // namespace livim

namespace {

livim::FrameRef frame_of(const py::array& arr_in) {
    py::array_t<uint8_t, py::array::c_style | py::array::forcecast> arr(arr_in);
    auto f = std::make_shared<livim::Frame>();
    if (arr.ndim() < 2 || arr.shape(0) == 0 || arr.shape(1) == 0) return f;   // an empty tap
    const int rows = (int)arr.shape(0), cols = (int)arr.shape(1), cn = arr.ndim() == 3 ? (int)arr.shape(2) : 1;
    f->image = cv::Mat(rows, cols, CV_MAKETYPE(CV_8U, cn));
    std::memcpy(f->image.data, arr.data(), (size_t)rows * cols * cn);
    f->width = cols;
    f->height = rows;
    f->format = cn == 1 ? livim::PixelFormat::Gray8 : livim::PixelFormat::BGR8;
    return f;
}

}  // namespace

PYBIND11_MODULE(_exporter_ref, m) {
    m.doc() = "The reference exporter's compose() (tschnz/Live-Video-Magnification src/export/Exporter.cpp), compiled in "
              "place against a facade that forwards pixel operations to cv2. Test infrastructure only.";
    m.def(
        "compose",
        [](const py::array& orig, const py::array& proc, int split, bool overlay) -> py::object {
            if (split < 0 || split > 2) throw std::invalid_argument("split");
            const cv::Mat c = livim::compose(frame_of(orig), frame_of(proc), static_cast<livim::SplitMode>(split), overlay);
            if (c.empty()) return py::none();
            py::array_t<uint8_t> out({(ssize_t)c.rows, (ssize_t)c.cols, (ssize_t)3});
            for (int y = 0; y < c.rows; ++y) std::memcpy(out.mutable_data(y), c.ptr<uint8_t>(y), (size_t)c.cols * 3);
            return std::move(out);
        },
        "compose(original, proc, split, overlay): the export canvas (HxWx3 u8), or None where the reference skips the "
        "frame (an empty Mat)",
        py::arg("original"), py::arg("proc"), py::arg("split"), py::arg("overlay"));
}
