// Host-side constant tables and scalar design code (no CUDA calls here).
#include <algorithm>
#include <cmath>
#include <complex>
#include <cstring>

#include <vector_types.h>

#include "mc_internal.h"

// lab_lut_s16.bin is linked in with `ld -r -b binary` (see __graft_entry__.build): the int16
// [b][g][r][3] table OpenCV's float BGR2Lab interpolates (tools/extract_lab_lut.py, SURVEY.md A.3).
extern "C" const unsigned char _binary_lab_lut_s16_bin_start[];
extern "C" const unsigned char _binary_lab_lut_s16_bin_end[];

namespace mc {

void build_lab_lut_cells(std::vector<LabLutCell>& out) {
    const int n = kLabLutDim;
    const size_t bytes = (size_t)(_binary_lab_lut_s16_bin_end - _binary_lab_lut_s16_bin_start);
    if (bytes != (size_t)n * n * n * 3 * sizeof(int16_t)) {
        out.clear();
        return;
    }
    std::vector<int16_t> raw((size_t)n * n * n * 3);
    std::memcpy(raw.data(), _binary_lab_lut_s16_bin_start, bytes);
    out.assign((size_t)kLabLutCells, LabLutCell{});
    for (int b = 0; b <= n; ++b)          // slab n repeats slab n-1 (only ever read with weight 0)
        for (int g = 0; g < n; ++g)
            for (int r = 0; r < n; ++r) {
                const int bb = std::min(b, n - 1), g1 = std::min(g + 1, n - 1), r1 = std::min(r + 1, n - 1);
                LabLutCell& c = out[((size_t)b * n + g) * n + r];
                const int gs[2] = {g, g1}, rs[2] = {r, r1};
                for (int ig = 0; ig < 2; ++ig)
                    for (int ch = 0; ch < 3; ++ch)
                        for (int ir = 0; ir < 2; ++ir)
                            c.v[6 * ig + 2 * ch + ir] = raw[((((size_t)bb * n + gs[ig]) * n + rs[ir]) * 3) + ch];
            }
}

void build_lab_lut_packs(const std::vector<LabLutCell>& cells, std::vector<LabLutPack>& out) {
    out.assign(cells.size(), LabLutPack{});
    for (size_t i = 0; i < cells.size(); ++i) {
        const int16_t* c = cells[i].v;   // {L00,L01, a00,a01, b00,b01, L10,L11, a10,a11, b10,b11}
        const int v[3] = {c[0], c[2] - kPackA0, c[4] - kPackB0};
        int dr[3], dg[3], e[3];
        for (int ch = 0; ch < 3; ++ch) {
            dr[ch] = c[2 * ch + 1] - c[2 * ch];
            dg[ch] = c[6 + 2 * ch] - c[2 * ch];
            e[ch] = c[6 + 2 * ch + 1] - c[6 + 2 * ch];
        }
        dg[1] = -dg[1];
        // {value, bit width} of every field in the order of the layout (mc_math.cuh)
        const int f[12][2] = {{v[0], 15}, {dr[0], 9}, {dr[2], 8}, {v[1], 14}, {dr[1], 9}, {dg[1], 9},
                              {v[2], 14}, {dg[2], 9}, {e[1], 9}, {dg[0], 10}, {e[0], 9}, {e[2], 8}};
        for (int k = 0; k < 12; ++k)
            if (f[k][0] < 0 || f[k][0] >= (1 << f[k][1])) {
                out.clear();
                return;
            }
        LabLutPack& p = out[i];
        p.w[0] = (uint32_t)f[0][0] | (uint32_t)f[1][0] << 15 | (uint32_t)f[2][0] << 24;
        p.w[1] = (uint32_t)f[3][0] | (uint32_t)f[4][0] << 14 | (uint32_t)f[5][0] << 23;
        p.w[2] = (uint32_t)f[6][0] | (uint32_t)f[7][0] << 14 | (uint32_t)f[8][0] << 23;
        p.w[3] = (uint32_t)f[9][0] | (uint32_t)f[10][0] << 10 | (uint32_t)f[11][0] << 19;
    }
}

// OpenCV's sRGBInvGammaTab: natural cubic spline (splineBuild) through the inverse sRGB transfer
// function sampled at i/1024; f32 arithmetic as OpenCV's softfloat build does it.
void build_inv_gamma_spline(std::vector<float4>& out) {
    const int n = kGammaTabSize;
    std::vector<float> f(n + 1), tab((size_t)n * 4, 0.0f);
    for (int i = 0; i <= n; ++i) {
        const double x = (double)((float)i / (float)n);
        f[i] = (float)(x <= 0.0031308 ? x * 12.92 : std::pow(x, 1.0 / 2.4) * 1.055 - 0.055);
    }
    float cn = 0.0f;
    for (int i = 1; i < n; ++i) {
        const float t = (f[i + 1] - f[i] * 2.0f + f[i - 1]) * 3.0f;
        const float l = 1.0f / (4.0f - tab[(size_t)(i - 1) * 4]);
        tab[(size_t)i * 4] = l;
        tab[(size_t)i * 4 + 1] = (t - tab[(size_t)(i - 1) * 4 + 1]) * l;
    }
    for (int j = 0; j < n; ++j) {
        const int i = n - j - 1;
        const float c = tab[(size_t)i * 4 + 1] - tab[(size_t)i * 4] * cn;
        const float b = f[i + 1] - f[i] - (cn + c * 2.0f) / 3.0f;
        const float d = (cn - c) / 3.0f;
        tab[(size_t)i * 4] = f[i];
        tab[(size_t)i * 4 + 1] = b;
        tab[(size_t)i * 4 + 2] = c;
        tab[(size_t)i * 4 + 3] = d;
        cn = c;
    }
    out.resize(n);
    for (int i = 0; i < n; ++i) out[i] = float4{tab[(size_t)i * 4], tab[(size_t)i * 4 + 1], tab[(size_t)i * 4 + 2], tab[(size_t)i * 4 + 3]};
}

void build_lab_inv_coeffs(LabInvCoeffs& out) {
    // XYZ -> linear sRGB (D65), columns scaled by the white point; rows ordered B, G, R.
    static const double m[9] = {3.240479, -1.53715, -0.498535, -0.969256, 1.875991, 0.041556, 0.055648, -0.204043, 1.057311};
    static const double wp[3] = {0.950456, 1.0, 1.088754};
    for (int row = 0; row < 3; ++row) {
        const int src_row = 2 - row;  // B row first
        for (int i = 0; i < 3; ++i) out.c[row * 3 + i] = (float)(m[src_row * 3 + i] * wp[i]);
    }
}

int calculate_max_levels(int w, int h) {
    int n = 0;
    while (w > 5 && h > 5) {
        w = (1 + w) / 2;
        h = (1 + h) / 2;
        ++n;
    }
    return n;
}

int optimal_buffer_size(int fps) {
    unsigned v = (unsigned)std::max(2 * fps, 16);
    unsigned p = 1;
    while (p < v) p <<= 1;
    return (int)p;
}

// Order-N digital Butterworth low-pass, cutoff wn (fraction of Nyquist): analog prototype poles on
// the unit circle, frequency-scaled by the pre-warped cutoff, mapped with the bilinear transform
// (fs = 2).  Same design the reference reaches through its transfer-function route; equals
// scipy.signal.butter(N, wn) to rounding.
void butterworth(unsigned order, double wn, std::vector<double>& a, std::vector<double>& b) {
    typedef std::complex<double> cd;
    const double pi = 3.14159265358979323846;
    const double fs = 2.0;
    const double w0 = 2.0 * fs * std::tan(pi * wn / fs);
    std::vector<cd> den(1, cd(1.0, 0.0));  // prod (z - pz_k)
    cd gain_den(1.0, 0.0);
    for (unsigned k = 1; k <= order; ++k) {
        const cd p = w0 * std::exp(cd(0.0, pi * (2.0 * k + order - 1.0) / (2.0 * order)));
        const cd pz = (2.0 * fs + p) / (2.0 * fs - p);
        gain_den *= (2.0 * fs - p);
        std::vector<cd> nd(den.size() + 1, cd(0.0, 0.0));
        for (size_t i = 0; i < den.size(); ++i) {
            nd[i] += den[i];
            nd[i + 1] -= den[i] * pz;
        }
        den.swap(nd);
    }
    const double gain = std::real(std::pow(cd(w0, 0.0), (double)order) / gain_den);
    a.assign(order + 1, 0.0);
    b.assign(order + 1, 0.0);
    double binom = 1.0;
    for (unsigned i = 0; i <= order; ++i) {
        a[i] = std::real(den[i]);
        b[i] = gain * binom;  // zeros at z = -1: (z + 1)^N
        binom = binom * (double)(order - i) / (double)(i + 1);
    }
}

void motion_gains(double amplification, double coWavelength, int levels, int w, int h, std::vector<float>& gains) {
    // MagnifyCore.hpp:114-134 — kept in the reference's mixed float/double arithmetic so the gains
    // are bit-identical.
    gains.assign((size_t)levels + 1, 0.0f);
    const float delta = static_cast<float>(coWavelength / (8.0 * (1.0 + amplification)));
    const float boost = 2.0f;
    float lambda = static_cast<float>(std::sqrt(double(w * w + h * h)) / 3.0);
    for (int lv = levels; lv >= 0; --lv) {
        const float cur = static_cast<float>((lambda / (delta * 8.0) - 1.0) * boost);
        gains[(size_t)lv] = (lv == levels || lv == 0) ? 0.0f : std::min(static_cast<float>(amplification), cur);
        lambda = static_cast<float>(lambda / 2.0);
    }
}

// OpenCV computeResizeAreaTab (imgproc/resize.cpp): taps of the general INTER_AREA path along one axis,
// grouped by destination index; ofs[d] .. ofs[d+1] index d's taps.
void build_area_tab(int ssize, int dsize, double scale, std::vector<AreaTap>& tab, std::vector<int>& ofs) {
    tab.clear();
    ofs.assign((size_t)dsize + 1, 0);
    for (int dx = 0; dx < dsize; ++dx) {
        ofs[(size_t)dx] = (int)tab.size();
        const double fsx1 = dx * scale, fsx2 = fsx1 + scale;
        const double cell = std::min(scale, ssize - fsx1);
        int sx1 = (int)std::ceil(fsx1), sx2 = (int)std::floor(fsx2);
        sx2 = std::min(sx2, ssize - 1);
        sx1 = std::min(sx1, sx2);
        if (sx1 - fsx1 > 1e-3) tab.push_back(AreaTap{dx, sx1 - 1, (float)((sx1 - fsx1) / cell)});
        for (int sx = sx1; sx < sx2; ++sx) tab.push_back(AreaTap{dx, sx, (float)(1.0 / cell)});
        if (fsx2 - sx2 > 1e-3) tab.push_back(AreaTap{dx, sx2, (float)(std::min(std::min(fsx2 - sx2, 1.), cell) / cell)});
    }
    ofs[(size_t)dsize] = (int)tab.size();
}

// PreprocessProcessor.cpp:20-33: normalised ROI -> pixel rectangle clamped inside the frame (>= 1 px).
void preprocess_roi(int cols, int rows, bool enabled, float rx, float ry, float rw, float rh, int& x, int& y, int& w, int& h) {
    x = 0; y = 0; w = cols; h = rows;
    if (!enabled) return;
    x = (int)std::lround((double)rx * cols);
    y = (int)std::lround((double)ry * rows);
    w = (int)std::lround((double)rw * cols);
    h = (int)std::lround((double)rh * rows);
    x = std::min(std::max(x, 0), cols - 1);
    y = std::min(std::max(y, 0), rows - 1);
    w = std::min(std::max(w, 1), cols - x);
    h = std::min(std::max(h, 1), rows - y);
}

void gaussian_kernel_13_3(float taps[13]) {
    // cv::getGaussianKernel(13, 3.0, CV_32F): exp(-x^2/(2 sigma^2)) normalised in double, then narrowed.
    double t[13], sum = 0.0;
    for (int i = 0; i < 13; ++i) {
        const double x = i - 6.0;
        t[i] = std::exp(-0.5 / 9.0 * x * x);
        sum += t[i];
    }
    for (int i = 0; i < 13; ++i) taps[i] = (float)(t[i] * (1.0 / sum));
}

}  // namespace mc
