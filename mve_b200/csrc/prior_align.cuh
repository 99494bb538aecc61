// Scale alignment of a relative prior (b200mvs_set_view_prior_relative, include/b200mvs.h): the observation of a feature
// in the view's map, the robust fit of s and t to the observations, and the per-pixel apply that turns the map into depth
// in MVE's convention.  The rules are __host__ __device__: the kernels below call them, and tests/emu compiles the same
// functions with g++ (B200MVS_HOST_EMU) to check them against tests/prior_align_reference.py.
#pragma once
#if defined(B200MVS_HOST_EMU)
#include "simt_emu.h"      // tests/emu: runs this very file on the CPU (test infrastructure)
#else
#include <cuda_runtime.h>
#endif
#include <cmath>
#include <cstring>
#include <stdint.h>

namespace b200mvs {

enum PriorKind { PRIOR_DISPARITY = 0, PRIOR_DEPTH = 1, PRIOR_DEPTH_SCALE = 2 };
constexpr unsigned ALIGN_MIN_OBS = 16;     // observations and inliers a fit needs
constexpr int ALIGN_ROUNDS = 3;
constexpr double ALIGN_MAD_SIGMA = 1.4826, ALIGN_CUT = 3.0;

// Why a fit failed (AlignFit::status)
enum AlignStatus { ALIGN_OK = 0, ALIGN_FEW_OBS, ALIGN_FLAT, ALIGN_FEW_INLIERS, ALIGN_SINGULAR, ALIGN_BAD_SCALE };

// The view's camera as the rules read it: world-to-camera R, t and the level-0 calibration, widened to double, and the
// registered image size W0 x H0
struct AlignCam {
    double R[9], t[3];
    double ax, ay, cx, cy;
    int W0, H0;
};

struct AlignFit {
    double s, t, med_rel;
    unsigned n_obs, n_in;
    int status;
    int pad;
};

// Products, quotients and sums rounded one at a time: the device never contracts them into an FMA, so a float64
// restatement evaluated left to right gives the same bits.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ double a_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double a_add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double a_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double a_div(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double a_sqrt(double a) { return __dsqrt_rn(a); }
#else
inline double a_mul(double a, double b) { return a * b; }
inline double a_add(double a, double b) { return a + b; }
inline double a_sub(double a, double b) { return a - b; }
inline double a_div(double a, double b) { return a / b; }
inline double a_sqrt(double a) { return std::sqrt(a); }
#endif

// finite and > 0 (NaN fails the comparison)
__host__ __device__ __forceinline__ bool pos_finite(double v) { return v > 0.0 && v <= 1.7976931348623157e308; }

// The prior pixel (px, py) of feature X in a w x h map and its z; false when X is not in front of the camera or the
// pixel is outside the map
__host__ __device__ inline bool align_pixel(const AlignCam& c, float X0, float X1, float X2, int w, int h, int* px, int* py,
                                            double* z)
{
    const double x0 = X0, x1 = X1, x2 = X2;
    double xc[3];
    for (int r = 0; r < 3; ++r)
        xc[r] = a_add(a_add(a_add(a_mul(c.R[3 * r], x0), a_mul(c.R[3 * r + 1], x1)), a_mul(c.R[3 * r + 2], x2)), c.t[r]);
    if (!(xc[2] > 0.0)) return false;
    const double u = a_add(a_div(a_mul(c.ax, xc[0]), xc[2]), c.cx);
    const double v = a_add(a_div(a_mul(c.ay, xc[1]), xc[2]), c.cy);
    const double fx = a_div(a_mul(u, (double)w), (double)c.W0), fy = a_div(a_mul(v, (double)h), (double)c.H0);
    if (!(fx >= 0.0 && fx < (double)w && fy >= 0.0 && fy < (double)h)) return false;
    *px = (int)fx;             // floor: fx >= 0
    *py = (int)fy;
    *z = xc[2];
    return true;
}

// The observation (d, y) of a feature at depth z whose prior pixel holds `value`; false when the value is not finite or
// not > 0
__host__ __device__ inline bool align_observation(int kind, double z, float value, double* d, double* y)
{
    const double dv = value;
    if (!pos_finite(dv)) return false;
    *d = dv;
    *y = kind == PRIOR_DISPARITY ? a_div(1.0, z) : z;
    return true;
}

// s d + t, the fitted value of the target
__host__ __device__ __forceinline__ double align_model(double s, double t, double d) { return a_add(a_mul(s, d), t); }
// the residual y - (s d + t)
__host__ __device__ __forceinline__ double align_residual(double s, double t, double d, double y)
{
    return a_sub(y, align_model(s, t, d));
}
// the inlier bound of a round: 3 sigma with sigma = 1.4826 med(|r|)
__host__ __device__ __forceinline__ double align_cut(double med_abs_r) { return a_mul(ALIGN_CUT, a_mul(ALIGN_MAD_SIGMA, med_abs_r)); }
// |z_fit - z| / z of an observation under s and t
__host__ __device__ inline double align_rel_err(int kind, double s, double t, double d, double y)
{
    const double q = align_model(s, t, d);
    const double zf = kind == PRIOR_DISPARITY ? a_div(1.0, q) : q, z = kind == PRIOR_DISPARITY ? a_div(1.0, y) : y;
    return a_div(fabs(a_sub(zf, z)), z);
}

// The start of the two affine kinds from med(d), med(y), MAD(d) and MAD(y); false when MAD(d) = 0
__host__ __device__ inline bool align_start_affine(double med_d, double med_y, double mad_d, double mad_y, double* s, double* t)
{
    if (mad_d == 0.0) return false;
    *s = a_div(mad_y, mad_d);
    *t = a_sub(med_y, a_mul(*s, med_d));
    return true;
}
// The least-squares refit of DEPTH_SCALE from sum(d y) and sum(d^2); false when sum(d^2) = 0
__host__ __device__ inline bool align_refit_scale(double sdy, double sdd, double* s, double* t)
{
    if (sdd == 0.0) return false;
    *s = a_div(sdy, sdd);
    *t = 0.0;
    return true;
}
// The centred least-squares refit of the affine kinds from the inliers' means dm, ym and the centred sums
// sum((d - dm)(y - ym)) and sum((d - dm)^2); false when the latter is 0
__host__ __device__ inline bool align_refit_affine(double dm, double ym, double sxy, double sxx, double* s, double* t)
{
    if (sxx == 0.0) return false;
    *s = a_div(sxy, sxx);
    *t = a_sub(ym, a_mul(*s, dm));
    return true;
}
// Whether a fit may be installed: s > 0, s and t finite
__host__ __device__ inline bool align_accept(double s, double t)
{
    return pos_finite(s) && fabs(t) <= 1.7976931348623157e308;
}

// The depth of prior pixel (px, py) of a w x h map holding `value`, under the fit s, t: 0 where the value or z is not
// finite and > 0
__host__ __device__ inline float align_apply(const AlignCam& c, int kind, double s, double t, float value, int px, int py,
                                             int w, int h)
{
    const double dv = value;
    if (!pos_finite(dv)) return 0.f;
    const double q = align_model(s, t, dv);
    const double z = kind == PRIOR_DISPARITY ? a_div(1.0, q) : q;
    if (!pos_finite(z)) return 0.f;
    const double a = a_div(a_sub(a_div(a_mul(a_add((double)px, 0.5), (double)c.W0), (double)w), c.cx), c.ax);
    const double b = a_div(a_sub(a_div(a_mul(a_add((double)py, 0.5), (double)c.H0), (double)h), c.cy), c.ay);
    return (float)a_mul(z, a_sqrt(a_add(a_add(a_mul(a, a), a_mul(b, b)), 1.0)));
}

// Key of a non-negative double for exact selection: its bit pattern orders as the value does.  ALIGN_SKIP sorts after
// every value, NaN included, so an observation left out of a selection never becomes its k-th element.
constexpr unsigned long long ALIGN_SKIP = ~0ull;
__host__ __device__ __forceinline__ unsigned long long align_key(double v)
{
    unsigned long long k;
    memcpy(&k, &v, sizeof(k));
    return k;
}
__host__ __device__ __forceinline__ double align_unkey(unsigned long long k)
{
    double v;
    memcpy(&v, &k, sizeof(v));
    return v;
}

// The fit of the observations (d[i], y[i]), i in [0, m); d[i] = 0 marks a slot without an observation.  Ops runs the three
// collective steps over [0, m): select(m, k, key) gives the element of rank k of the keys key(i) (ALIGN_SKIP left out),
// sum2(m, f) the two sums of f(i) = (a, b), and count(m, pred) the number of i with pred(i).  Every caller of a given Ops
// gets the same result, so the control flow below is uniform.
#if defined(__CUDACC__)
#pragma nv_exec_check_disable
#endif
template <typename Ops, typename Arr>
__host__ __device__ AlignFit align_fit(Ops& ops, const Arr& d, const Arr& y, unsigned m, int kind)
{
    AlignFit f = {0.0, 0.0, 0.0, 0u, 0u, ALIGN_OK, 0};
    const unsigned n = ops.count(m, [&](unsigned i) { return d[i] > 0.0; });
    f.n_obs = n;
    if (n < ALIGN_MIN_OBS) { f.status = ALIGN_FEW_OBS; return f; }
    const unsigned mid = (n - 1) / 2;
    auto med = [&](auto&& value) {            // lower median of value(i) over the observations
        return ops.select(m, mid, [&](unsigned i) { return d[i] > 0.0 ? align_key(value(i)) : ALIGN_SKIP; });
    };
    double s, t;
    if (kind == PRIOR_DEPTH_SCALE) {
        s = med([&](unsigned i) { return a_div(y[i], d[i]); });
        t = 0.0;
    } else {
        const double md = med([&](unsigned i) { return d[i]; }), my = med([&](unsigned i) { return y[i]; });
        const double mad_d = med([&](unsigned i) { return fabs(a_sub(d[i], md)); });
        const double mad_y = med([&](unsigned i) { return fabs(a_sub(y[i], my)); });
        if (!align_start_affine(md, my, mad_d, mad_y, &s, &t)) { f.status = ALIGN_FLAT; return f; }
    }
    // the inliers of s, t: |r| <= 3 sigma with sigma from every observation's |r|
    auto inlier_cut = [&]() { return align_cut(med([&](unsigned i) { return fabs(align_residual(s, t, d[i], y[i])); })); };
    auto inlier = [&](unsigned i, double cut) { return d[i] > 0.0 && fabs(align_residual(s, t, d[i], y[i])) <= cut; };
    for (int round = 0; round < ALIGN_ROUNDS; ++round) {
        const double cut = inlier_cut();
        const unsigned n_in = ops.count(m, [&](unsigned i) { return inlier(i, cut); });
        if (n_in < ALIGN_MIN_OBS) { f.status = ALIGN_FEW_INLIERS; return f; }
        bool ok;
        if (kind == PRIOR_DEPTH_SCALE) {
            double sdy, sdd;
            ops.sum2(m, [&](unsigned i, double* a, double* b) {
                const bool in = inlier(i, cut);
                *a = in ? a_mul(d[i], y[i]) : 0.0;
                *b = in ? a_mul(d[i], d[i]) : 0.0;
            }, &sdy, &sdd);
            ok = align_refit_scale(sdy, sdd, &s, &t);
        } else {
            double sd, sy, sxy, sxx;
            ops.sum2(m, [&](unsigned i, double* a, double* b) {
                const bool in = inlier(i, cut);
                *a = in ? d[i] : 0.0;
                *b = in ? y[i] : 0.0;
            }, &sd, &sy);
            const double dm = a_div(sd, (double)n_in), ym = a_div(sy, (double)n_in);
            ops.sum2(m, [&](unsigned i, double* a, double* b) {
                const bool in = inlier(i, cut);
                const double dd = a_sub(d[i], dm);
                *a = in ? a_mul(dd, a_sub(y[i], ym)) : 0.0;
                *b = in ? a_mul(dd, dd) : 0.0;
            }, &sxy, &sxx);
            ok = align_refit_affine(dm, ym, sxy, sxx, &s, &t);
        }
        if (!ok) { f.status = ALIGN_SINGULAR; return f; }
    }
    const double cut = inlier_cut();
    const unsigned n_in = ops.count(m, [&](unsigned i) { return inlier(i, cut); });
    if (n_in < ALIGN_MIN_OBS) { f.status = ALIGN_FEW_INLIERS; return f; }
    if (!align_accept(s, t)) { f.status = ALIGN_BAD_SCALE; return f; }
    f.med_rel = ops.select(m, (n_in - 1) / 2,
                           [&](unsigned i) { return inlier(i, cut) ? align_key(align_rel_err(kind, s, t, d[i], y[i])) : ALIGN_SKIP; });
    f.s = s; f.t = t; f.n_in = n_in;
    return f;
}

#if !defined(B200MVS_HOST_EMU)

constexpr int ALIGN_FIT_TPB = 512;

// align_fit's collective steps for one CTA of ALIGN_FIT_TPB threads.  select is a radix select on the keys' bytes, most
// significant first, with a 256-bin histogram per pass; the sums add each thread's strided share in a fixed order and
// then a fixed tree, so a fit is deterministic.
struct CtaOps {
    unsigned* hist;            // 256 bins
    double* red;               // 2 x ALIGN_FIT_TPB
    unsigned long long* bcast; // the selected prefix and the remaining rank
    unsigned* cnt;

    template <typename K> __device__ double select(unsigned m, unsigned k, K&& key)
    {
        const unsigned tid = threadIdx.x, lane = tid & 31;
        unsigned long long prefix = 0;
        unsigned rank = k;
        for (int shift = 56; shift >= 0; shift -= 8) {
            const unsigned long long hi = shift == 56 ? 0ull : ~0ull << (shift + 8);
            for (unsigned b = tid; b < 256; b += blockDim.x) hist[b] = 0;
            __syncthreads();
            for (unsigned i = tid; i < m; i += blockDim.x) {
                const unsigned long long q = key(i);
                if ((q & hi) == prefix) atomicAdd(&hist[(q >> shift) & 0xFF], 1u);
            }
            __syncthreads();
            if (tid < 32) {            // warp 0: the bin holding rank `rank`, from a scan of 8 bins per lane
                unsigned c[8], own = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) { c[j] = hist[lane * 8 + j]; own += c[j]; }
                unsigned incl = own;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                    if (lane >= (unsigned)o) incl += v;
                }
                unsigned below = incl - own;
                if (rank >= below && rank < incl) {
                    for (int j = 0; j < 8; ++j) {
                        if (rank < below + c[j]) {
                            bcast[0] = prefix | ((unsigned long long)(lane * 8 + j) << shift);
                            bcast[1] = rank - below;
                            break;
                        }
                        below += c[j];
                    }
                }
            }
            __syncthreads();
            prefix = bcast[0];
            rank = (unsigned)bcast[1];
            __syncthreads();
        }
        return align_unkey(prefix);
    }

    template <typename F> __device__ void sum2(unsigned m, F&& f, double* A, double* B)
    {
        const unsigned tid = threadIdx.x;
        double a = 0.0, b = 0.0;
        for (unsigned i = tid; i < m; i += blockDim.x) {
            double x, z;
            f(i, &x, &z);
            a = a_add(a, x);
            b = a_add(b, z);
        }
        red[tid] = a;
        red[ALIGN_FIT_TPB + tid] = b;
        __syncthreads();
        for (unsigned h = ALIGN_FIT_TPB / 2; h > 0; h >>= 1) {
            if (tid < h) {
                red[tid] = a_add(red[tid], red[tid + h]);
                red[ALIGN_FIT_TPB + tid] = a_add(red[ALIGN_FIT_TPB + tid], red[ALIGN_FIT_TPB + tid + h]);
            }
            __syncthreads();
        }
        *A = red[0];
        *B = red[ALIGN_FIT_TPB];
        __syncthreads();
    }

    template <typename P> __device__ unsigned count(unsigned m, P&& pred)
    {
        const unsigned tid = threadIdx.x;
        if (tid == 0) *cnt = 0;
        __syncthreads();
        unsigned c = 0;
        for (unsigned i = tid; i < m; i += blockDim.x) c += pred(i) ? 1u : 0u;
        if (c) atomicAdd(cnt, c);
        __syncthreads();
        const unsigned n = *cnt;
        __syncthreads();
        return n;
    }
};

// One thread per feature of the view: pos[i] is its position (the view's features in the order of the context's
// inverted index).  obs[i] receives its observation (d, y), or (0, 0) when it has none.
__global__ void k_align_observe(const float* __restrict__ pos, unsigned m, const AlignCam cam, const float* __restrict__ values,
                                int w, int h, size_t pitch, int kind, double2* __restrict__ obs)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    int px, py;
    double z, d = 0.0, y = 0.0;
    if (align_pixel(cam, __ldg(pos + 3 * i), __ldg(pos + 3 * i + 1), __ldg(pos + 3 * i + 2), w, h, &px, &py, &z)) {
        const float v = __ldg(reinterpret_cast<const float*>(reinterpret_cast<const char*>(values) + (size_t)py * pitch) + px);
        if (!align_observation(kind, z, v, &d, &y)) d = y = 0.0;
    }
    obs[i] = make_double2(d, y);
}

// One CTA of ALIGN_FIT_TPB threads fits the m observations: obs as (d, y) pairs, split into d[] and y[] views by stride
__global__ void __launch_bounds__(ALIGN_FIT_TPB) k_align_fit(const double2* __restrict__ obs, unsigned m, int kind,
                                                             AlignFit* __restrict__ out)
{
    __shared__ unsigned hist[256];
    __shared__ double red[2 * ALIGN_FIT_TPB];
    __shared__ unsigned long long bcast[2];
    __shared__ unsigned cnt;
    CtaOps ops = {hist, red, bcast, &cnt};
    const double* o = reinterpret_cast<const double*>(obs);
    struct Strided { const double* p; __device__ double operator[](unsigned i) const { return p[2 * i]; } };
    // align_fit reads d[i] and y[i]: the pairs' two members
    const AlignFit f = align_fit(ops, Strided{o}, Strided{o + 1}, m, kind);
    if (threadIdx.x == 0) *out = f;
}

// The apply over a w x h map: src rows `src_pitch` bytes apart, dst packed (dst may be src with src_pitch = 4 w).  Runs
// only after a fit that may be installed.
__global__ void k_align_apply(const float* src, size_t src_pitch, float* dst, int w, int h, const AlignCam cam, int kind,
                              const AlignFit* __restrict__ fit)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h || fit->status != ALIGN_OK) return;
    const float v = *(reinterpret_cast<const float*>(reinterpret_cast<const char*>(src) + (size_t)y * src_pitch) + x);
    dst[(size_t)y * w + x] = align_apply(cam, kind, fit->s, fit->t, v, x, y, w, h);
}

#endif

} // namespace b200mvs
