// ssim_common.cuh -- the SSIM arithmetic shared by the training loss (loss.cu) and the evaluation metrics (metrics.cu):
// the 11-tap Gaussian window and the per-pixel SSIM expression.  The metrics evaluate S from the five raw moments in
// double (ssim_terms); the training loss evaluates it in float from the moments of x, y and d = x - y
// (ssim_diff_terms), which keeps its value and gradient free of the cancellation in sigma_xy near x == y.
#pragma once
#include <cmath>
#include <cuda_runtime.h>

namespace fdgs {

constexpr int SSIM_R = 5;   // filter radius: window_size 11 (reference: utils/loss_utils.py:39)

struct GaussWin {
    float g[2 * SSIM_R + 1];
};

inline GaussWin make_window() {
    // reference: utils/loss_utils.py:24-26 gaussian(11, 1.5): float32 exp values normalised by their float32 sum
    GaussWin w;
    float v[2 * SSIM_R + 1];
    float s = 0.f;
    for (int i = 0; i <= 2 * SSIM_R; ++i) {
        v[i] = (float)exp(-(double)((i - SSIM_R) * (i - SSIM_R)) / (2.0 * 1.5 * 1.5));
        s += v[i];
    }
    for (int i = 0; i <= 2 * SSIM_R; ++i) w.g[i] = v[i] / s;
    return w;
}

// The terms of the SSIM map at one pixel from the windowed moments mu_x, mu_y, E[xx], E[yy], E[xy]
// (reference: utils/loss_utils.py:50-60): S = A1 A2 / (B1 B2), inv = 1 / (B1 B2).  T = float in the training loss,
// double in the evaluation metrics.
template <typename T>
struct SsimTerms {
    T A1, A2, B1, B2, inv, S;
};

template <typename T>
__device__ __forceinline__ SsimTerms<T> ssim_terms(T m1, T m2, T e11, T e22, T e12) {
    const T C1 = T(0.01) * T(0.01), C2 = T(0.03) * T(0.03);
    const T m11 = m1 * m1, m22 = m2 * m2, m12 = m1 * m2;
    const T s11 = e11 - m11, s22 = e22 - m22, s12 = e12 - m12;
    SsimTerms<T> t;
    t.A1 = T(2) * m12 + C1;
    t.A2 = T(2) * s12 + C2;
    t.B1 = m11 + m22 + C1;
    t.B2 = s11 + s22 + C2;
    t.inv = T(1) / (t.B1 * t.B2);
    t.S = t.A1 * t.A2 * t.inv;
    return t;
}

// The same S from the means mu_x, mu_y, their difference mu_d, the variances sigma_xx, sigma_yy and E[dd], d = x - y:
//   A1 = B1 - mu_d^2,  A2 = B2 - sigma_dd  (2 sigma_xy = sigma_xx + sigma_yy - sigma_dd),  S = P Q,
//   P = A1 / B1 = 1 - mu_d^2 / B1,  Q = A2 / B2 = 1 - sigma_dd / B2.
// Near x == y, sigma_dd is formed from the small d itself instead of as the difference of sigma_xx + sigma_yy and
// 2 sigma_xy (each ~E[x^2], so their fp32 rounding would be ~1e-5 of B2 >= C2), and the partial derivatives of S are
// all O(d): the gradient has no terms of order 1/B2 that cancel.  The caller passes mu_d and the variances so that it
// can form them from moments about a shift.
template <typename T>
struct SsimDiffTerms {
    T sdd, B1, B2, P, Q, S;
};

template <typename T>
__device__ __forceinline__ SsimDiffTerms<T> ssim_diff_terms(T m1, T m2, T md, T s11, T s22, T edd) {
    const T C1 = T(0.01) * T(0.01), C2 = T(0.03) * T(0.03);
    SsimDiffTerms<T> t;
    t.sdd = edd - md * md;
    t.B1 = m1 * m1 + m2 * m2 + C1;
    t.B2 = s11 + s22 + C2;
    t.P = T(1) - md * md / t.B1;
    t.Q = T(1) - t.sdd / t.B2;
    t.S = t.P * t.Q;
    return t;
}

}  // namespace fdgs
