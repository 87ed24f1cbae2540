// TEST INFRASTRUCTURE ONLY.  The product's NV12 per-pixel functions (csrc/mc_math.cuh: nv12_to_bgr_px, bgr_to_ycc_px)
// compiled for the CPU, so tests/test_nv12_host.py can compare them with cv2 on every input without a GPU.  Built by
// that test into a temporary directory; never loaded by the product.
#include <cstdint>

#include <cuda_runtime.h>

#include "mc_math.cuh"

using namespace mc;

extern "C" {
// n pixels (y[i], u[i], v[i]) -> BGR
void nc_nv12_to_bgr(const uint8_t* y, const uint8_t* u, const uint8_t* v, int n, uint8_t* bgr) {
    for (int i = 0; i < n; ++i) nv12_to_bgr_px(y[i], u[i], v[i], bgr[3 * i], bgr[3 * i + 1], bgr[3 * i + 2]);
}
// n BGR pixels -> (Y, Cb, Cr)
void nc_bgr_to_ycc(const uint8_t* bgr, int n, uint8_t* ycc) {
    for (int i = 0; i < n; ++i) bgr_to_ycc_px(bgr[3 * i], bgr[3 * i + 1], bgr[3 * i + 2], ycc[3 * i], ycc[3 * i + 1], ycc[3 * i + 2]);
}
}
