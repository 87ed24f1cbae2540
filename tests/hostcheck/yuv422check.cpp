// TEST INFRASTRUCTURE ONLY.  The product's packed 4:2:2 per-pixel function (csrc/mc_math.cuh: yuv422_to_bgr_px) compiled
// for the CPU, so tests/test_yuv422_host.py can compare it with cv2 on every input without a GPU.  Built by that test
// into a temporary directory; never loaded by the product.
#include <cstddef>
#include <cstdint>

#include <cuda_runtime.h>

#include "mc_math.cuh"

using namespace mc;

extern "C" {
// h rows of w pixels (w even) of a packed YUYV (uyvy = 0) or UYVY frame, `pitch` bytes per row -> tight BGR
void yc_yuv422_to_bgr(const uint8_t* src, size_t pitch, int w, int h, int uyvy, uint8_t* bgr) {
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const uint8_t* q = src + (size_t)y * pitch + (size_t)2 * (x & ~1);
            const uint32_t grp = (uint32_t)q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | (uint32_t)q[3] << 24;
            uint8_t* o = bgr + 3 * ((size_t)y * w + x);
            yuv422_to_bgr_px(grp, x & 1, uyvy != 0, o[0], o[1], o[2]);
        }
}
}
