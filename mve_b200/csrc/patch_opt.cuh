// Definitions shared by the two device implementations of one mvs::PatchOptimization
// (libs/dmrecon/patch_optimization.cc:21-364 with PatchSampler patch_sampler.cc:19-393, LocalViewSelection
// local_view_selection.cc:19-160 and mvs_tools.cc:98-199; SURVEY.md Appendix A is the line-by-line behavioural spec):
//   patch_warp.cuh    one WARP per patch   - lowest latency, used for small frontier rounds
//   patch_thread.cuh  one THREAD per patch - highest throughput, used for large frontier rounds
// Both expose begin() / step() / finish(): the kernels drive them with a flat loop in which a lane (warp) that finishes a
// patch fetches the next one at once and meets the others again at the single pass() call site inside step().
// Data layout: the four bilinear taps of a sample come from ONE 16-byte load of a "quad" texel (the 2x2 neighbourhood of
// every pixel is stored contiguously, DESIGN.md "Data layout"); sRGB code values are linearised through a copy of the
// 256-entry table that is replicated per lane in shared memory (no bank conflicts, mvs_tools.cc:21-95).
#pragma once
#if defined(B200MVS_HOST_EMU)
#include "simt_emu.h"      // tests/emu: runs this very file on the CPU, 32 host threads per warp (test infrastructure)
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <cstddef>

namespace b200mvs {

constexpr int MAX_LEVELS = 12;
constexpr int MAX_GLOBAL = 32;
constexpr int MAX_LOCAL = 4;
constexpr unsigned FULL = 0xffffffffu;
constexpr int NS = 25;
constexpr int CENTER = 12;   // patch_sampler.cc:73,96
constexpr int LUT_REP = 32;  // replicas of the sRGB table in shared memory that are used (one per lane)
constexpr int LUT_STRIDE = 64; // floats per table value: a value's replicas start every 256 bytes (lut_k)

struct alignas(16) LevelParams {   // ImagePyramidLevel (image_pyramid.h:28-59): K = [ax 0 cx; 0 ay cy; 0 0 1]
    float ax, ay, cx, cy;
    int w, h;
    int pitch;                // in texels (uchar4), also the pitch of the quad image (uint4)
    int pad;
    const uchar4* img;        // RGBX8, row pitch 16-byte aligned
    const uint4* quad;        // quad[y * pitch + x] = {img(x,y), img(x+1,y), img(x,y+1), img(x+1,y+1)} (clamped at the border)
};
static_assert(sizeof(LevelParams) == 48, "LevelParams layout");

struct alignas(16) ViewParams {    // SingleView (single_view.h:28-133)
    float campos[3];
    float inv_ax0;            // source_level.invproj[0] (single_view.h:154-157)
    float w2c[12];            // rows 0..2 of worldToCam
    float rot[9];
    int nlevels;
    int valid;
    int pad;
    LevelParams lv[MAX_LEVELS];
};
static_assert(offsetof(ViewParams, lv) % 16 == 0, "ViewParams layout");

struct DevSettings {
    float min_ncc, min_parallax, accept_ncc, min_refine_diff;
    unsigned max_iterations, nr_recon_neighbors;
    int scale, use_color_scale;
};

struct JobParams {            // one reference view being reconstructed (DMRecon members, dmrecon.h:50-62)
    int ref_view, W, H, n_global;
    int gview[MAX_GLOBAL];    // global view ids by slot, ascending (neighViews)
    float ki0, ki2, ki4, ki5; // target_level.invproj entries [0],[2],[4],[5]
    const uchar4* ref_img;    // level `scale` of the reference view
    int ref_pitch;
    int tiles_x;              // 16x16-pixel tiles per row of the reference level (frontier sort)
    float* depth; float* conf; float* dz; float* normal;
    unsigned* slots;          // 4 x uint8 global slots per pixel (0xFF = none)
    unsigned long long* sel;  // per-pixel selection key of the current frontier round
    long long tile_base;      // first tile bin of this job
};

struct PatchIn  { int x, y; float depth, dzI, dzJ; unsigned slots; };   // slots: 4 x uint8, 0xFF padded, ascending
struct PatchOut { float conf, depth, dzI, dzJ, nx, ny, nz; unsigned slots; int iterations; int flags; };
// flags: bit0 converged, bit1 opti_success

// Hot-path approximations (each <= 2 ulp): MUFU reciprocal / reciprocal square root instead of the IEEE division and
// square root sequences.  The reference itself is built with -funsafe-math-optimizations (Makefile.inc:5), i.e. without
// IEEE guarantees for these operations; the effect on parity is measured by tests/test_gpu_parity.py.  Everything that
// decides integers on the host (global view selection, seeds, pyramid) stays IEEE.
// Pinned roundings: a fused multiply-add, a product and a sum that the compiler neither contracts nor splits.  Where the
// per-sample code of PatchT is written with them, its values do not depend on how the loop around it is arranged (the
// compiler contracts a * b + c only when both halves land in the same basic block).  The host emulation does not fuse
// anywhere (g++ in ISO mode, no FMA), so there they are the plain expressions.
#if defined(B200MVS_HOST_EMU)
__device__ __forceinline__ float rcp_fast(float x) { return 1.f / x; }
__device__ __forceinline__ float rsqrt_fast(float x) { return 1.f / sqrtf(x); }
__device__ __forceinline__ float fma_rn(float a, float b, float c) { return a * b + c; }
__device__ __forceinline__ float mul_rn(float a, float b) { return a * b; }
__device__ __forceinline__ float add_rn(float a, float b) { return a + b; }
__device__ __forceinline__ float sub_rn(float a, float b) { return a - b; }
#else
__device__ __forceinline__ float rcp_fast(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rsqrt_fast(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }
#endif

// sRGB code value (byte K of `w`) -> linear, through the lane-replicated table in shared memory (mvs_tools.cc:21-95).  Replica r of
// value v lives at byte offset v * 256 + r * 4: with the values 256 bytes apart the offset is (byte << 8) | lane4, and that is
// ONE instruction - a byte permute that drops byte K of the texel word next to the lane's own byte (lane4 < 128, the upper
// bytes of that register are zero).  A stride of 128 bytes (no unused half) needs a shift and an and-or per look-up: 15
// instructions more per sample.
template <int K> __device__ __forceinline__ float lut_k(const float* table, unsigned lane4, unsigned w)
{
    static_assert(LUT_REP == 32 && LUT_STRIDE == 64, "offset arithmetic assumes 32 lanes and 256-byte rows");
#if defined(B200MVS_HOST_EMU)
    const unsigned off = (((w >> (8 * K)) & 0xFFu) << 8) | lane4;
#else
    const unsigned off = __byte_perm(w, lane4, 0x6504u | ((unsigned)K << 4));      // {lane4.b0, w.bK, 0, 0}
#endif
    return *reinterpret_cast<const float*>(reinterpret_cast<const char*>(table) + off);
}

// mvs_tools.h:56-69
__device__ __forceinline__ float plx_weight(float p)
{
    if (p < 0.f || p > 180.f) return 0.f;
    const float sigma = (p <= 20.f) ? 5.f : 15.f;
    const float dlt = p - 20.f;
    return expf(-(dlt * dlt) / (2.f * sigma * sigma));
}
__device__ __forceinline__ float clamp1(float v) { return v < -1.f ? -1.f : (v > 1.f ? 1.f : v); }
__device__ __forceinline__ float deg_acos(float dp) { return acosf(dp) * 180.f / 3.141592653589793f; }

} // namespace b200mvs
