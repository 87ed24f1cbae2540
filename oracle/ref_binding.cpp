// _livim_ref — TEST INFRASTRUCTURE ONLY (oracle/).  Python bindings over the *reference's own* hot-path classes,
// compiled unmodified from /root/reference/src (see oracle/build_ref.py) against the cvshim facade:
//   * Chain      = buildProcessors() + runChainOnce()                       (processing/ChainBuilder.cpp:11-29)
//   * Processor  = livim::MagnificationProcessor                            (processing/MagnificationProcessor.cpp)
//   * Core       = magcore::magnifyMotion / magnifyColor / magnifyRiesz with their public state structs
//                  (processing/magnification/MagnifyCore.hpp:24-40,83,163,209) so tests can read the state
//   * toParams, motionHzToBlend, calculateMaxLevels, getOptimalBufferSize, butterworth
// Used by tests/ to pin oracle/livim_oracle.py against the reference's real control flow, and by
// bench.py --impl reference / cpu_baseline as the CPU arm (kind "reference").
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <opencv2/core.hpp>

#include "core/Frame.hpp"
#include "processing/ChainBuilder.hpp"
#include "processing/GrayscaleProcessor.hpp"
#include "processing/IProcessor.hpp"
#include "processing/PreprocessProcessor.hpp"
#include "processing/MagnificationParamsUi.hpp"
#include "processing/MagnificationProcessor.hpp"
#include "processing/magnification/MagnifyCore.hpp"
#include "processing/magnification/SpatialFilter.hpp"
#include "processing/magnification/TemporalFilter.hpp"

namespace py = pybind11;
using namespace livim;

namespace cv { void cvshim_selfcheck(); }
void mc_dl_open(const std::string& path);   // oracle/mc_dl.cpp

// the reference-side adapter of the product, compiled here against the REAL reference headers
#include "MagnificationProcessorB200.hpp"

static cv::Mat mat_from_u8(const py::array& arr_in) {
    py::array_t<uint8_t, py::array::c_style | py::array::forcecast> arr(arr_in);
    if (arr.ndim() != 2 && arr.ndim() != 3) throw std::invalid_argument("frame must be HxW or HxWxC uint8");
    const int rows = (int)arr.shape(0), cols = (int)arr.shape(1), cn = arr.ndim() == 3 ? (int)arr.shape(2) : 1;
    if (rows == 0 || cols == 0) return cv::Mat();
    cv::Mat m(rows, cols, CV_MAKETYPE(CV_8U, cn));
    std::memcpy(m.data, arr.data(), (size_t)rows * cols * cn);
    return m;
}

static py::object mat_to_np(const cv::Mat& m) {
    if (m.empty()) return py::none();
    const int cn = m.channels();
    std::vector<ssize_t> shape{m.rows, m.cols};
    if (cn > 1) shape.push_back(cn);
    py::dtype dt = m.depth() == CV_8U ? py::dtype::of<uint8_t>() : m.depth() == CV_32F ? py::dtype::of<float>() : py::dtype::of<double>();
    py::array out(dt, shape);
    const size_t rowbytes = (size_t)m.cols * m.elemSize();
    for (int y = 0; y < m.rows; ++y) std::memcpy(static_cast<uint8_t*>(out.mutable_data()) + (size_t)y * rowbytes, m.ptr<uint8_t>(y), rowbytes);
    return out;
}

static MutableFrameRef frame_from_np(const py::array& a, std::uint64_t seq) {
    auto f = std::make_shared<Frame>();
    f->image = mat_from_u8(a);
    f->width = f->image.cols;
    f->height = f->image.rows;
    f->format = f->image.channels() == 1 ? PixelFormat::Gray8 : PixelFormat::BGR8;
    f->seq = seq;
    f->ptsUs = (std::int64_t)seq * 1000;
    return f;
}

struct RefChain {
    std::vector<std::unique_ptr<IProcessor>> chain = buildProcessors();
    std::uint64_t seq = 0;
    // -> (processed image, original-tap image, processed_is_input, original_is_input, format is gray)
    py::tuple process(const py::array& frame, const ProcessorConfig& cfg) {
        FrameRef in = frame_from_np(frame, seq++);
        FrameRef original;
        FrameRef out = runChainOnce(chain, in, cfg, original);
        if (out->seq != in->seq || out->ptsUs != in->ptsUs) throw std::runtime_error("frame metadata not preserved");
        return py::make_tuple(mat_to_np(out->image), mat_to_np(original->image), out.get() == in.get(), original.get() == in.get(),
                              out->format == PixelFormat::Gray8);
    }
    void reset() { for (auto& p : chain) p->reset(); }
};

// The drop-in itself: the reference's chain exactly as buildProcessors() assembles it (ChainBuilder.cpp:11-17) with
// the single substitution INTEGRATION.md describes at ChainBuilder.cpp:15 — MagnificationProcessorB200 (the adapter
// over the C ABI) in place of MagnificationProcessor — driven by the reference's own runChainOnce().  The two
// front stages are the reference's compiled code.  Needs an H100: the adapter's constructor throws without one.
struct DropInChain {
    std::vector<std::unique_ptr<IProcessor>> chain;
    std::uint64_t seq = 0;
    explicit DropInChain(int device) {
        chain.push_back(std::make_unique<PreprocessProcessor>());
        chain.push_back(std::make_unique<GrayscaleProcessor>());
        chain.push_back(std::make_unique<MagnificationProcessorB200>(device));
    }
    py::tuple process(const py::array& frame, const ProcessorConfig& cfg) {
        FrameRef in = frame_from_np(frame, seq++);
        FrameRef original;
        FrameRef out = runChainOnce(chain, in, cfg, original);
        if (out->seq != in->seq || out->ptsUs != in->ptsUs) throw std::runtime_error("frame metadata not preserved");
        if (out.get() != in.get() && out->image.data == in->image.data) throw std::runtime_error("output aliases the input buffer");
        return py::make_tuple(mat_to_np(out->image), mat_to_np(original->image), out.get() == in.get(), original.get() == in.get(),
                              out->format == PixelFormat::Gray8);
    }
    void reset() { for (auto& p : chain) p->reset(); }
};

struct RefProcessor {
    MagnificationProcessor proc;
    std::uint64_t seq = 0;
    // -> (produced, image); produced == false means the reference returned the *same* FrameRef it was given
    py::tuple process(const py::array& frame, const ProcessorConfig& cfg) {
        FrameRef in = frame_from_np(frame, seq++);
        FrameRef out = proc.process(in, cfg);
        const bool produced = out.get() != in.get();
        if (produced && out->image.data == in->image.data) throw std::runtime_error("output aliases the input buffer");
        return py::make_tuple(produced, mat_to_np(out->image));
    }
    void reset() { proc.reset(); }
};

struct RefCore {
    magcore::MotionState motion;
    magcore::ColorState color;
    magcore::RieszState riesz;

    py::tuple run(int mode, const py::array& frame, const MagnificationParams& p, int levels) {
        cv::Mat in = mat_from_u8(frame), out;
        PixelFormat fmt = PixelFormat::BGR8;
        const int channels = in.channels();
        bool produced = false;
        switch (mode) {
        case 0: produced = magcore::magnifyMotion(in, p, levels, channels, motion, out, fmt); break;
        case 1: produced = magcore::magnifyRiesz(in, p, levels, channels, riesz, out, fmt); break;
        case 2: produced = magcore::magnifyColor(in, p, levels, channels, color, out, fmt); break;
        default: throw std::invalid_argument("mode");
        }
        return py::make_tuple(produced, produced ? mat_to_np(out) : py::object(py::none()));
    }
    py::tuple motion_state() const {
        py::list hi, lo;
        for (const auto& m : motion.lowpassHi) hi.append(mat_to_np(m));
        for (const auto& m : motion.lowpassLo) lo.append(mat_to_np(m));
        return py::make_tuple(hi, lo);
    }
    py::object color_window() const { return mat_to_np(color.window); }
    py::list riesz_levels(bool old) const {
        py::list out;
        const auto& pyr = old ? riesz.old : riesz.cur;
        if (!pyr) return out;
        for (const auto& l : pyr->pyrLevels) {
            py::dict d;
            d["lowpass"] = mat_to_np(l.itsLowpass);
            d["rx"] = mat_to_np(real(l.itsRiesz));
            d["ry"] = mat_to_np(imag(l.itsRiesz));
            d["amplitude"] = mat_to_np(l.itsAmplitude);
            d["amplitude_blurred"] = mat_to_np(l.itsAmplitudeBlurred);
            d["phase_diff_cos"] = mat_to_np(cos(l.itsPhaseDiff));
            d["phase_diff_sin"] = mat_to_np(sin(l.itsPhaseDiff));
            d["lowpass_iir_cos"] = mat_to_np(cos(l.itsLowpassIIR));
            d["lowpass_iir_sin"] = mat_to_np(sin(l.itsLowpassIIR));
            d["highpass_iir_cos"] = mat_to_np(cos(l.itsHighpassIIR));
            d["highpass_iir_sin"] = mat_to_np(sin(l.itsHighpassIIR));
            out.append(d);
        }
        return out;
    }
    py::tuple riesz_coefficients() const {
        if (!riesz.lo) return py::make_tuple(py::none(), py::none(), py::none(), py::none());
        return py::make_tuple(riesz.lo->itsA, riesz.lo->itsB, riesz.hi->itsA, riesz.hi->itsB);
    }
    void reset() { motion.reset(); color.reset(); riesz.reset(); }
};

PYBIND11_MODULE(_livim_ref, m) {
    m.doc() = "The reference's own hot path (tschnz/Live-Video-Magnification src/processing), compiled in place against "
              "the cvshim facade that forwards pixel operations to cv2. Test infrastructure only.";
    cv::cvshim_selfcheck();

    py::enum_<MagnificationMode>(m, "MagnificationMode")
        .value("Laplace", MagnificationMode::Laplace).value("Phase", MagnificationMode::Phase)
        .value("Color", MagnificationMode::Color).value("None_", MagnificationMode::None);

    py::class_<MagnificationParams>(m, "MagnificationParams")
        .def(py::init<>())
        .def_readwrite("mode", &MagnificationParams::mode)
        .def_readwrite("amplification", &MagnificationParams::amplification)
        .def_readwrite("coWavelength", &MagnificationParams::coWavelength)
        .def_readwrite("coLow", &MagnificationParams::coLow)
        .def_readwrite("coHigh", &MagnificationParams::coHigh)
        .def_readwrite("chromAttenuation", &MagnificationParams::chromAttenuation)
        .def_readwrite("levels", &MagnificationParams::levels)
        .def_readwrite("framerate", &MagnificationParams::framerate);

    py::class_<PreprocessParams>(m, "PreprocessParams")
        .def(py::init<>())
        .def_readwrite("downscale", &PreprocessParams::downscale)
        .def_readwrite("roiEnabled", &PreprocessParams::roiEnabled)
        .def_readwrite("roiX", &PreprocessParams::roiX)
        .def_readwrite("roiY", &PreprocessParams::roiY)
        .def_readwrite("roiW", &PreprocessParams::roiW)
        .def_readwrite("roiH", &PreprocessParams::roiH);

    py::class_<ProcessorConfig>(m, "ProcessorConfig")
        .def(py::init<>())
        .def_readwrite("grayscale", &ProcessorConfig::grayscale)
        .def_readwrite("preprocess", &ProcessorConfig::preprocess)
        .def_readwrite("magnification", &ProcessorConfig::magnification);

    py::class_<MagUiValues>(m, "MagUiValues")
        .def(py::init<>())
        .def_readwrite("mode", &MagUiValues::mode)
        .def_readwrite("amplification", &MagUiValues::amplification)
        .def_readwrite("wavelength", &MagUiValues::wavelength)
        .def_readwrite("low", &MagUiValues::low)
        .def_readwrite("high", &MagUiValues::high)
        .def_readwrite("chroma", &MagUiValues::chroma)
        .def_readwrite("levels", &MagUiValues::levels)
        .def_readwrite("captureFps", &MagUiValues::captureFps);

    m.def("toParams", &toParams);
    m.def("toUi", &toUi);
    m.def("defaultsFor", &defaultsFor);
    m.def("motionHzToBlend", &motionHzToBlend);
    m.def("calculateMaxLevels", [](int w, int h) { return calculateMaxLevels(cv::Size(w, h)); });
    m.def("getOptimalBufferSize", &getOptimalBufferSize);
    m.def("butterworth", [](unsigned n, double wn) {
        std::vector<double> a, b;
        butterworth(n, wn, a, b);
        return py::make_tuple(a, b);
    });

    m.def("set_magcore_library", &mc_dl_open, "path of libmagcore_b200.so for DropInChain (resolved lazily with dlopen)");
    py::class_<DropInChain>(m, "DropInChain").def(py::init<int>()).def("process", &DropInChain::process).def("reset", &DropInChain::reset);
    py::class_<RefChain>(m, "Chain").def(py::init<>()).def("process", &RefChain::process).def("reset", &RefChain::reset);
    py::class_<RefProcessor>(m, "Processor").def(py::init<>()).def("process", &RefProcessor::process).def("reset", &RefProcessor::reset);
    py::class_<RefCore>(m, "Core")
        .def(py::init<>())
        .def("run", &RefCore::run)
        .def("motion_state", &RefCore::motion_state)
        .def("color_window", &RefCore::color_window)
        .def("riesz_levels", &RefCore::riesz_levels)
        .def("riesz_coefficients", &RefCore::riesz_coefficients)
        .def("reset", &RefCore::reset);
}
