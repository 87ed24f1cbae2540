// Reference-side adapter: a livim::IProcessor that forwards the magnification stage to the H100 core
// through the C ABI (include/magcore_b200.h).  It is the ONLY file the reference application needs:
//
//     // src/processing/ChainBuilder.cpp:15
//     procs.push_back(std::make_unique<MagnificationProcessorB200>());   // was MagnificationProcessor
//
// Contract mirrored from reference src/processing/MagnificationProcessor.cpp:17-67:
//   * identity / passthrough (mode None, empty or too-small image, Color warm-up, Riesz first frame or
//     gray input) returns the *same* FrameRef;
//   * otherwise a fresh Frame copying the metadata, whose image never aliases the input (:63-66);
//   * a core failure throws std::runtime_error so ProcessingChain's firewall (ProcessingChain.cpp:50-62)
//     counts it, calls reset() on every stage and shows the input frame;
//   * one instance is driven by one thread in frame order; instances are independent (no globals).
#pragma once

#include <memory>
#include <stdexcept>
#include <string>

#include "magcore_b200.h"
#include "processing/IProcessor.hpp"

namespace livim {

class MagnificationProcessorB200 : public IProcessor {
public:
    explicit MagnificationProcessorB200(int cudaDevice = 0) {
        if (mc_create(cudaDevice, &h_) != MC_OK)
            throw std::runtime_error(std::string("magcore_b200: ") + mc_last_error(nullptr));
    }
    ~MagnificationProcessorB200() override { mc_destroy(h_); }
    MagnificationProcessorB200(const MagnificationProcessorB200&) = delete;
    MagnificationProcessorB200& operator=(const MagnificationProcessorB200&) = delete;

    void reset() override {
        if (mc_reset(h_) != MC_OK) throw std::runtime_error(std::string("magcore_b200: ") + mc_last_error(h_));
    }

    FrameRef process(const FrameRef& in, const ProcessorConfig& cfg) override {
        const MagnificationParams& m = cfg.magnification;
        mc_params p;
        mc_params_default(&p);
        p.mode = static_cast<int32_t>(m.mode);  // same enumerator order (IProcessor.hpp:10)
        p.levels = m.levels;
        p.amplification = m.amplification;
        p.coWavelength = m.coWavelength;
        p.coLow = m.coLow;
        p.coHigh = m.coHigh;
        p.chromAttenuation = m.chromAttenuation;
        p.framerate = m.framerate;
        p.pre_downscale = cfg.preprocess.downscale;
        p.pre_roiEnabled = cfg.preprocess.roiEnabled ? 1 : 0;
        p.pre_roiX = cfg.preprocess.roiX;
        p.pre_roiY = cfg.preprocess.roiY;
        p.pre_roiW = cfg.preprocess.roiW;
        p.pre_roiH = cfg.preprocess.roiH;

        const cv::Mat& src = in->image;
        int produced = 0;
        if (src.empty()) {
            check(mc_process(h_, nullptr, 0, 0, 3, 0, &p, nullptr, 0, &produced));
            return in;
        }
        cv::Mat dst(src.rows, src.cols, src.type());  // fresh buffer; never aliases in->image
        check(mc_process(h_, src.data, src.cols, src.rows, src.channels(), static_cast<size_t>(src.step), &p,
                         dst.data, static_cast<size_t>(dst.step), &produced));
        if (!produced) return in;  // warm-up / unsupported input / identity: emit the input unchanged
        auto out = std::make_shared<Frame>(*in);
        out->image = std::move(dst);
        out->format = src.channels() >= 3 ? PixelFormat::BGR8 : PixelFormat::Gray8;
        return out;
    }

private:
    void check(mc_status st) const {
        if (st != MC_OK) throw std::runtime_error(std::string("magcore_b200: ") + mc_last_error(h_));
    }
    mc_handle* h_ = nullptr;
};

}  // namespace livim
