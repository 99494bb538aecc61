// sfmrecon's radial undistortion of a view's `original` photo (sfmrecon.cc:425-437): mve::image::image_undistort_k2k4<uint8_t>
// (image_tools.h:1731-1769) with Image::linear_at(float, float, T*) (image.h:438-460) and the four-value unsigned char
// math::interpolate (functions.h:141-147), one output pixel per call, bit for bit as the reference build computes it.
// The source may be packed or pitched HWC, or planar CHW (Src): only where a texel is read from depends on the layout.
// That build (-O3 -march=x86-64-v3 -funsafe-math-optimizations) does not evaluate the source as written; its instantiation
// (tests/undistort_reference.py restates it) does, per image:
//     fwidth2 = w * 0.5, fheight2 = h * 0.5, inv_fnorm = 1 / max(w, h), inv_f2 = 1 / (flen * flen)       (double)
// per pixel:
//     fx = (x + (0.5 - fwidth2)) * inv_fnorm,  fy = (y + (0.5 - fheight2)) * inv_fnorm
//     rd = inv_f2 * fma(fx, fx, fy * fy),      rd_factor = fma(fma(k4, rd, k2), rd, 1)
//     ix = float(fma(fnorm * fx, rd_factor, fwidth2 - 0.5)),  iy = float(fma(rd_factor, fy * fnorm, fheight2 - 0.5))
//     left 0 when ix < -0.5f, double(ix) > w - 0.5, iy < -0.5f or double(iy) > h - 0.5
// and linear_at, with x, y clamped to [0, w - 1] x [0, h - 1] (min first, NaN takes the bound) and t = trunc:
//     w1 = x - t(x), w0 = t(x) + (1 - x), w3 = y - t(y), w2 = (t(y) + 1) - y                           (float)
//     v = int(fma(fma(v00, w0, v01 * w1), w2, fma(v10, w0, v11 * w1) * w3) + 0.5f)
// Every operation is pinned (__dmul_rn, __fma_rn, __double2float_rn, __fmaf_rn, ...), so nvcc neither contracts nor
// reorders it.  The same file compiles as host code with B200MVS_HOST_EMU (tests/emu/undistort_emu.cc); the host build
// must not contract either (-ffp-contract=off).
#pragma once
#if !defined(B200MVS_HOST_EMU)
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <cmath>

namespace b200mvs_undistort {

#if defined(B200MVS_HOST_EMU)
#define UNDIST_FN inline
inline double dadd(double a, double b) { return a + b; }
inline double dmul(double a, double b) { return a * b; }
inline double dfma(double a, double b, double c) { return std::fma(a, b, c); }
inline float d2f(double a) { return (float)a; }
inline float fadd(float a, float b) { return a + b; }
inline float fsub(float a, float b) { return a - b; }
inline float fmul(float a, float b) { return a * b; }
inline float ffma(float a, float b, float c) { return std::fma(a, b, c); }
inline float ftrunc(float a) { return std::trunc(a); }
inline int f2i_rz(float a) { return (int)a; }
inline uint8_t load_u8(const uint8_t* p) { return *p; }
#else
#define UNDIST_FN __device__ __forceinline__
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dfma(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ float d2f(double a) { return __double2float_rn(a); }
__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float ftrunc(float a) { return truncf(a); }
__device__ __forceinline__ int f2i_rz(float a) { return __float2int_rz(a); }
__device__ __forceinline__ uint8_t load_u8(const uint8_t* p) { return __ldg(p); }
#endif

// The per-image constants, computed once on the host (single IEEE double operations, as the reference's loop preamble)
struct Params {
    double ox, oy;          // 0.5 - fwidth2, 0.5 - fheight2
    double cx, cy;          // fwidth2 - 0.5, fheight2 - 0.5
    double xmax, ymax;      // w - 0.5, h - 0.5
    double fnorm, inv_fnorm, inv_f2, k2, k4;
    float wm1, hm1;         // float(w - 1), float(h - 1): linear_at's clamp
    int w, h, ch;           // image size and channels (1..4)
};

// Where the source image lies: texel (x, y), channel c at base + y * row + x * ch + c when interleaved (HWC; packed when
// row = w * ch), at base + c * plane + y * row + x when planar (CHW).  The layout is a template parameter of the readers,
// so the packed path computes its addresses as before and no texel read branches on it.
struct Src {
    const uint8_t* base;
    int64_t row;            // bytes between rows
    int64_t plane;          // bytes between channel planes (planar only)
};
template <bool Planar> UNDIST_FN const uint8_t* texel(const Src& s, int ch, int x, int y)
{
    return s.base + (int64_t)y * s.row + (int64_t)x * (Planar ? 1 : ch);
}
template <bool Planar> UNDIST_FN int64_t channel_offset(const Src& s, int c) { return Planar ? c * s.plane : c; }

// k2 == k4 == 0 is the reference's duplicate(): the caller imports the image unchanged instead
inline bool active(float k2, float k4) { return k2 != 0.0f || k4 != 0.0f; }

// sfmrecon passes CameraInfo's float flen, dist[0] and dist[1] (camera.h:161-162); they widen to double exactly
inline Params make_params(int w, int h, int ch, float flen, float k2, float k4)
{
    Params P;
    const double fw2 = (double)w * 0.5, fh2 = (double)h * 0.5;
    P.ox = 0.5 - fw2; P.oy = 0.5 - fh2;
    P.cx = fw2 - 0.5; P.cy = fh2 - 0.5;
    P.xmax = (double)w - 0.5; P.ymax = (double)h - 0.5;
    P.fnorm = (double)(w > h ? w : h);
    P.inv_fnorm = 1.0 / P.fnorm;
    const double f2 = (double)flen * (double)flen;
    P.inv_f2 = 1.0 / f2;
    P.k2 = (double)k2; P.k4 = (double)k4;
    P.wm1 = (float)(w - 1); P.hm1 = (float)(h - 1);
    P.w = w; P.h = h; P.ch = ch;
    return P;
}

// The channels of output pixel (x, y) of image_undistort_k2k4, channel c in bits 8c..8c+7 (0 where the reference leaves
// the pixel 0, and above channel ch - 1), read from the w x h x ch source image `src`
template <bool Planar> UNDIST_FN uint32_t undistort_px(const Params& P, const Src& src, int x, int y)
{
    const double fx = dmul(dadd((double)x, P.ox), P.inv_fnorm);
    const double fy = dmul(dadd((double)y, P.oy), P.inv_fnorm);
    const double rd = dmul(P.inv_f2, dfma(fx, fx, dmul(fy, fy)));
    const double rf = dfma(dfma(P.k4, rd, P.k2), rd, 1.0);
    float ix = d2f(dfma(dmul(P.fnorm, fx), rf, P.cx));
    float iy = d2f(dfma(rf, dmul(fy, P.fnorm), P.cy));
    if (ix < -0.5f || (double)ix > P.xmax || iy < -0.5f || (double)iy > P.ymax) return 0u;
    // linear_at: clamp (min, then max), truncation, float weights
    ix = ix < P.wm1 ? ix : P.wm1;
    iy = iy < P.hm1 ? iy : P.hm1;
    ix = ix > 0.0f ? ix : 0.0f;
    iy = iy > 0.0f ? iy : 0.0f;
    const float tx = ftrunc(ix), ty = ftrunc(iy);
    const int x0 = (int)tx, y0 = (int)ty;
    const int x1 = x0 + 1 < P.w - 1 ? x0 + 1 : P.w - 1;
    const int y1 = y0 + 1 < P.h - 1 ? y0 + 1 : P.h - 1;
    const float w1 = fsub(ix, tx), w0 = fadd(tx, fsub(1.0f, ix));
    const float w3 = fsub(iy, ty), w2 = fsub(fadd(ty, 1.0f), iy);
    const uint8_t* p00 = texel<Planar>(src, P.ch, x0, y0);
    const uint8_t* p01 = texel<Planar>(src, P.ch, x1, y0);
    const uint8_t* p10 = texel<Planar>(src, P.ch, x0, y1);
    const uint8_t* p11 = texel<Planar>(src, P.ch, x1, y1);
    uint32_t out = 0u;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c >= P.ch) break;
        const int64_t o = channel_offset<Planar>(src, c);
        const float top = ffma((float)load_u8(p00 + o), w0, fmul((float)load_u8(p01 + o), w1));
        const float bot = ffma((float)load_u8(p10 + o), w0, fmul((float)load_u8(p11 + o), w1));
        out |= (uint32_t)(f2i_rz(fadd(ffma(top, w2, fmul(bot, w3)), 0.5f)) & 0xFF) << (8 * c);
    }
    return out;
}

// The same from a packed h x w x ch image
UNDIST_FN uint32_t undistort_px(const Params& P, const uint8_t* src, int x, int y)
{
    return undistort_px<false>(P, Src{src, (int64_t)P.w * P.ch, 0}, x, y);
}

} // namespace b200mvs_undistort
