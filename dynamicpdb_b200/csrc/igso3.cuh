// IGSO(3) series and sigma(t) lookup shared by the score epilogue (K9, csrc/epilogue.cu: fp32 angle) and the forward
// diffusion (csrc/diffuse.cu: fp64 angle).  Reference: src/data/so3_diffuser.py:9-49 (igso3_expansion), :71-117 (score),
// :183-199 (discrete_sigma, sigma_idx, logarithmic sigma(t)).
#pragma once
#include "common.cuh"

namespace dfold {

// np.digitize(sigma(t), discrete_sigma) - 1, clamped to [0, G): the grid index of the logarithmic schedule's sigma(t)
__device__ __forceinline__ int sigma_index(double t, const double* grid, int G, double e_max, double e_min) {
    const double s = log(t * e_max + (1.0 - t) * e_min);
    // number of grid points <= s, minus one (np.digitize(..) - 1), clamped
    int lo = 0, hi = G;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (grid[mid] <= s) lo = mid + 1; else hi = mid;
    }
    int idx = lo - 1;
    idx = idx < 0 ? 0 : (idx >= G ? G - 1 : idx);
    return idx;
}

// Precision-generic helpers: the float forms are the round-to-nearest intrinsics K9 has always used (no contraction).
__device__ __forceinline__ float rn_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double rn_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float rn_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double rn_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float t_sin(float a) { return sinf(a); }
__device__ __forceinline__ double t_sin(double a) { return sin(a); }
__device__ __forceinline__ float t_cos(float a) { return cosf(a); }
__device__ __forceinline__ double t_cos(double a) { return cos(a); }
__device__ __forceinline__ void t_sincos(float a, float* s, float* c) { sincosf(a, s, c); }
__device__ __forceinline__ void t_sincos(double a, double* s, double* c) { sincos(a, s, c); }

// exponent -l(l+1) sigma^2 / 2 of term l (s2h = sigma^2 / 2); exp() of it is exactly 0 below -746, and the exponent
// decreases with l, so a sum over l may stop at the first such term
constexpr double kIgso3ExpCut = -746.0;
__device__ __forceinline__ double igso3_exponent(int l, double s2h) { return -(double)l * (double)(l + 1) * s2h; }
__device__ __forceinline__ double igso3_decay(int l, double ex) { return (double)(2 * l + 1) * exp(ex); }

// the omega-only factors of the series: lo = sin(omega/2), dlo = cos(omega/2)/2, lo^2
template <typename T>
struct Igso3Angle { T omega, lo, dlo, lo2; };

template <typename T>
__device__ __forceinline__ Igso3Angle<T> igso3_angle(T omega) {
    Igso3Angle<T> a;
    a.omega = omega;
    const T half_om = omega / T(2);
    a.lo = t_sin(half_om);
    a.dlo = T(0.5) * t_cos(half_om);
    a.lo2 = rn_mul(a.lo, a.lo);
    return a;
}

// Adds term l (weight decay = (2l+1) exp(-l(l+1) sigma^2/2)) of the expansion, of its omega-derivative and (kSecond) of
// its second derivative.  The trigonometry runs in T (fp32 for K9, as the reference's fp32 rotation vector makes it;
// fp64 for the forward marginal); weights and sums are fp64.
template <typename T, bool kSecond>
__device__ __forceinline__ void igso3_term(const Igso3Angle<T>& a, int l, double decay, double& s, double& ds, double& d2s) {
    const T h = (T)l + T(0.5);
    const T arg = rn_mul(a.omega, h);
    T sh, ch;
    t_sincos(arg, &sh, &ch);
    const T dhi = rn_mul(h, ch);
    const T num = rn_sub(rn_mul(a.lo, dhi), rn_mul(sh, a.dlo));
    s += decay * (double)sh / (double)a.lo;
    ds += decay * (double)num / (double)a.lo2;
    if (kSecond) {
        const double dlo_d = (double)a.dlo, lo_d = (double)a.lo, hi_d = (double)sh;
        const double d2hi = -(double)h * (double)h * hi_d, d2lo = -0.25 * lo_d;
        d2s += decay * ((lo_d * d2hi - hi_d * d2lo) / (lo_d * lo_d) - 2.0 * dlo_d * (double)num / (lo_d * lo_d * lo_d));
    }
}

// IGSO(3) series at angle omega over l < L, split across the 32 lanes of a warp (lane takes l = lane, lane + 32, ...) and
// combined by warp_sum_d: S = expansion, dS = d/domega, d2S = d2/domega2 (kSecond).
template <typename T, bool kSecond>
__device__ __forceinline__ void igso3_series(T omega, double sigma, int L, int lane, double& S, double& dS, double& d2S) {
    const Igso3Angle<T> a = igso3_angle(omega);
    const double s2h = sigma * sigma * 0.5;
    double s = 0.0, ds = 0.0, d2s = 0.0;
    for (int l = lane; l < L; l += 32) {
        const double ex = igso3_exponent(l, s2h);
        if (ex < kIgso3ExpCut) break;                             // exp() is exactly 0 from here on
        igso3_term<T, kSecond>(a, l, igso3_decay(l, ex), s, ds, d2s);
    }
    S = warp_sum_d(s);
    dS = warp_sum_d(ds);
    d2S = kSecond ? warp_sum_d(d2s) : 0.0;
}

}  // namespace dfold
