// Definitions shared by the two device implementations of one mvs::PatchOptimization
// (libs/dmrecon/patch_optimization.cc:21-364 with PatchSampler patch_sampler.cc:19-393, LocalViewSelection
// local_view_selection.cc:19-160 and mvs_tools.cc:98-199; SURVEY.md Appendix A is the line-by-line behavioural spec):
//   patch_warp.cuh    one WARP per patch   - lowest latency, used for small frontier rounds
//   patch_thread.cuh  one THREAD per patch - highest throughput, used for large frontier rounds
// Both expose begin() / step() / finish(): the kernels drive them with a flat loop in which a lane (warp) that finishes a
// patch fetches the next one at once and meets the others again at the single pass() call site inside step().
// Both keep the state of doAutoOptimization in PatchState and share its state machine (PatchState::auto_step) and every
// step that does not depend on how samples map to lanes; what does - the sample sets, the reductions, the storage of the
// selected set, the candidate scoring - is all an implementation supplies (see PatchState).
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

// ---- steps of one PatchOptimization that do not depend on the mapping ----

// Level of view V for a patch with master footprint 1 / inv_mfp and footprint nfp in V (patch_sampler.cc:76-91),
// clampLevel with minLevel = 0 (single_view.h:113-123).
__device__ __forceinline__ int level_of(const ViewParams* V, float nfp, float inv_mfp)
{
    float ratio = nfp * inv_mfp;
    int l = 0;
    while (ratio < 0.5f) { ++l; ratio *= 2.f; }
    const int nl = __ldg(&V->nlevels);
    if (l > nl - 1) l = nl - 1;
    return l;
}

// What a pass hands to the Gauss-Newton step of the same auto_step() call: the optimizeDepthOnly sums and the solution of
// the normal equations of optimizeDepthAndNormal.
struct PassOut { float num, den, nX0, nX1, nX2; };

// viewDir / epipolar plane / footprint of view V at patchPoints[12] = cp, with rd the reference view's direction
// (local_view_selection.cc:93-131)
__device__ __forceinline__ void view_geometry(const ViewParams* V, float cpx, float cpy, float cpz, float rdx, float rdy, float rdz,
                                              float& vdx, float& vdy, float& vdz, float& epx, float& epy, float& epz, float& nfp)
{
    vdx = cpx - __ldg(&V->campos[0]); vdy = cpy - __ldg(&V->campos[1]); vdz = cpz - __ldg(&V->campos[2]);
    const float nn = sqrtf(vdx * vdx + vdy * vdy + vdz * vdz);
    vdx /= nn; vdy /= nn; vdz /= nn;
    epx = vdy * rdz - vdz * rdy; epy = vdz * rdx - vdx * rdz; epz = vdx * rdy - vdy * rdx;
    const float en = sqrtf(epx * epx + epy * epy + epz * epz);
    epx /= en; epy /= en; epz /= en;
    const float z = __ldg(&V->w2c[8]) * cpx + __ldg(&V->w2c[9]) * cpy + __ldg(&V->w2c[10]) * cpz + __ldg(&V->w2c[11]);
    nfp = z * __ldg(&V->inv_ax0);
}

// The parallax and epipolar terms of a candidate (viewDir vd, epipolar plane ep) against one selected view (viewDir s,
// epipolar plane e) applied to its score (local_view_selection.cc:108-131).
__device__ __forceinline__ void lvs_weigh(float& score, float vdx, float vdy, float vdz, float epx, float epy, float epz,
                                          float sx, float sy, float sz, float ex, float ey, float ez, float min_parallax)
{
    float dp = clamp1(sx * vdx + sy * vdy + sz * vdz);
    score *= plx_weight(deg_acos(dp));
    dp = clamp1(epx * ex + epy * ey + epz * ez);
    float angle = fabsf(deg_acos(dp));
    if (angle > 90.f) angle = 180.f - angle;
    angle = fmaxf(angle, 1.f);
    if (angle < min_parallax) score *= angle / min_parallax;
}

// computeConfidence (patch_optimization.cc:114-142) + getPatchNormal (patch_sampler.cc:243-256) from the patch tangents
// a = patchPoints[14] - patchPoints[10] and b = patchPoints[2] - patchPoints[22], the centre ray cr and the mean NCC.
__device__ __forceinline__ void confidence(PatchOut& out, float ax_, float ay_, float az_, float bx_, float by_, float bz_,
                                           float crx, float cry, float crz, float mean, float accept_ncc)
{
    const float score = (mean - accept_ncc) / (1.f - accept_ncc);
    float nx = ay_ * bz_ - az_ * by_, ny = az_ * bx_ - ax_ * bz_, nz = ax_ * by_ - ay_ * bx_;
    const float nn = sqrtf(nx * nx + ny * ny + nz * nz);
    nx /= nn; ny /= nn; nz /= nn;
    out.nx = nx; out.ny = ny; out.nz = nz;
    const float dotP = -(nx * crx + ny * cry + nz * crz);
    out.conf = (dotP < 0.2f) ? 0.f : score;
}

// ---- the state of one PatchOptimization and the state machine of doAutoOptimization ----
// An implementation P derives from PatchState and supplies what depends on how the samples map to lanes:
//   pass(candidates, cs_pending, want_ncc, want_normal, cand, PassOut&)   the one pass at the current state: sample sets
//        over the selected views (or, with `candidates`, over the available global views, only their NCC: first half of
//        LocalViewSelection::performVS, local_view_selection.cc:73-85); clears and sets the COL / DER bits, and with
//        want_ncc the DF bits, when it overwrites the NCCs
//   lvs_greedy(cand)      second half of performVS (local_view_selection.cc:86-147); sets F_LVS_OK when the set is full
//   compute_points()      patch_sampler.cc:274-295, clears F_REF_OK when a sample lies behind the camera
//   sel_erase_mask(mask)  removes selected view k for every bit k of mask
//   low_ncc_mask()        bit k: selected view k has an NCC below acceptNCC
// In PatchW every lane holds the same PatchState.
struct PatchState {
    float depth, dzI, dzJ;
    unsigned avail;            // LocalViewSelection::available over global slots
    int iter;
    unsigned n_sets;           // sample sets drawn (statistics)
    // Everything small lives in ONE word (`pk`): in PatchT the state of a patch stays live across the whole sample loop, and
    // every register it occupies there is a register the loop spills.
    //   bits 0-9   flags F_*          bits 10-12 stage        bits 13-15 nsel (size of the selected set)
    //   bits 16-19 p_col_ok           bits 20-23 p_der_ok     (per selected view: colour / derivative samples valid in the last pass)
    //   bits 24-27 |NCC - oldNCC| > minRefineDiff per selected view, taken when the last pass overwrote the NCC (the
    //              reference keeps a copy, oldNCC, for this one comparison: patch_optimization.cc:196-199,217-225)
    unsigned pk;

    enum Stage { LVS_CTOR, CTOR, FIRST, PRE, POST, LVS_REPL, REPL, DONE };
    enum : unsigned {
        F_REF_OK = 1u << 0,        // sampler->success[refViewNr]
        F_OPTI = 1u << 1, F_CONVERGED = 1u << 2, F_LVS_OK = 1u << 3, F_VIEW_REMOVED = 1u << 4, F_WAS_NORMAL = 1u << 5,
        F_NORMAL = 1u << 6, F_SINGULAR = 1u << 7, F_HAS_NORMAL = 1u << 8, F_HAS_NCC = 1u << 9
    };
    static constexpr int SH_STAGE = 10, SH_NSEL = 13, SH_COL = 16, SH_DER = 20, SH_DF = 24;
    __device__ __forceinline__ bool is(unsigned f) const { return (pk & f) != 0u; }
    __device__ __forceinline__ void put(unsigned f, bool v) { pk = v ? (pk | f) : (pk & ~f); }
    __device__ __forceinline__ int stage() const { return (int)((pk >> SH_STAGE) & 7u); }
    __device__ __forceinline__ void set_stage(int v) { pk = (pk & ~(7u << SH_STAGE)) | ((unsigned)v << SH_STAGE); }
    __device__ __forceinline__ int nsel() const { return (int)((pk >> SH_NSEL) & 7u); }
    __device__ __forceinline__ void set_nsel(int v) { pk = (pk & ~(7u << SH_NSEL)) | ((unsigned)v << SH_NSEL); }
    __device__ __forceinline__ bool all_der_ok() const { return ((pk >> SH_DER) & 0xFu) == ((1u << nsel()) - 1u); }

    // start of the PatchOptimization ctor: opti = true, detATA == 0 until a solve says otherwise, everything else clear
    __device__ __forceinline__ void reset(const PatchIn& in)
    {
        depth = in.depth; dzI = in.dzI; dzJ = in.dzJ;
        iter = 0;
        pk = F_OPTI | F_SINGULAR | ((unsigned)DONE << SH_STAGE);
        avail = 0u;
    }
    __device__ __forceinline__ void finish_state(PatchOut& out) const
    {
        out.depth = depth; out.dzI = dzI; out.dzJ = dzJ;
        out.iterations = iter;
        out.flags = (is(F_CONVERGED) ? 1 : 0) | (is(F_OPTI) ? 2 : 0);
        out.conf = 0.f; out.nx = out.ny = out.nz = 0.f;
    }

    // computeColorScale of one view (patch_optimization.cc:88-110) from the per-channel sums ab = sum((m - cs n) n) and
    // aa = sum(n n): updates the scales cc, clears F_OPTI when a channel fails.
    __device__ __forceinline__ void colour_scale_step(float (&cc)[3], const float (&ab)[3], const float (&aa)[3])
    {
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
            if ((double)fabsf(aa[ch]) > 1e-6) {
                cc[ch] += ab[ch] * rcp_fast(aa[ch]);
                if ((double)cc[ch] > 1e3) pk &= ~F_OPTI;
            } else
                pk &= ~F_OPTI;
        }
    }

    // PatchSampler::update (patch_sampler.cc:259-271)
    template <class P> static __device__ __forceinline__ void update(P& p)
    {
        p.pk |= F_REF_OK;
        p.compute_points();
    }

    // optimizeDepthOnly (patch_optimization.cc:265-299) from the sums of the last pass.  Returns true when the state moved.
    template <class P> static __device__ __forceinline__ bool depth_step(P& p, const PassOut& po)
    {
        if (!p.all_der_ok()) { p.pk &= ~F_OPTI; return false; }
        if (po.den > 0.f) {
            p.depth += po.num / po.den;
            update(p);
            p.put(F_OPTI, p.is(F_REF_OK));
            return true;
        }
        return false;
    }

    // optimizeDepthAndNormal (patch_optimization.cc:302-364) from the solution prepared by the last pass.
    template <class P> static __device__ __forceinline__ bool normal_step(P& p, const PassOut& po)
    {
        if (!p.all_der_ok()) { p.pk &= ~F_OPTI; return false; }
        if (p.is(F_SINGULAR)) { p.pk &= ~F_OPTI; return false; }
        p.dzI += po.nX1; p.dzJ += po.nX2; p.depth += po.nX0;
        update(p);
        p.put(F_OPTI, p.is(F_REF_OK));
        return true;
    }

    // The rest of the ctor (performVS, computeColorScale) and PatchOptimization::doAutoOptimization
    // (patch_optimization.cc:66-77,170-242) as a state machine around the single pass() call site: one call = one pass
    // plus everything up to the next one.  Returns true when the optimisation is over.
    template <class P> static __device__ __forceinline__ bool auto_step(P& p)
    {
        const int stage = p.stage();
        if (stage == DONE) return true;
        // arguments of the one pass() call, by stage
        const bool a_cand = (stage == LVS_CTOR) | (stage == LVS_REPL);
        const bool a_cs = (stage == CTOR) | (stage == REPL) | ((stage == POST) & p.is(F_WAS_NORMAL));   // computeColorScale of :77, :230, :198
        const bool a_ncc = (stage == PRE) | (stage == POST) | (stage == REPL) | ((stage == FIRST) & (p.iter == 4));
        const bool a_normal = (stage == REPL) | ((stage == FIRST) & (p.iter == 4)) | ((stage == PRE) & p.is(F_NORMAL)) |
                              ((stage == POST) & ((p.iter + 1) % 5 == 4));
        float cand[MAX_GLOBAL];      // candidates' NCCs for PatchT (local memory, touched on the rare view-selection passes only)
        PassOut po = {0.f, 0.f, 0.f, 0.f, 0.f};
        p.pass(a_cand, a_cs, a_ncc, a_normal, cand, po);
        if (stage == LVS_CTOR || stage == LVS_REPL) {
            p.lvs_greedy(cand);
            if (!p.is(F_LVS_OK)) { if (stage == LVS_CTOR) p.pk &= ~F_OPTI; p.set_stage(DONE); return true; }
            p.set_stage((stage == LVS_CTOR) ? CTOR : REPL);
            return false;
        }
        if (!p.is(F_OPTI)) { p.set_stage(DONE); return true; }     // a colour scale failed: every caller of computeColorScale gives up here
        if (stage == POST) {
            // `abs(ncc - oldNCC) > minRefineDiff` per view was taken when the pass overwrote the NCC
            const int n = p.nsel();
            const unsigned dfb = (p.pk >> SH_DF) & ((1u << n) - 1u);
            const unsigned tbr = ((p.iter == 14) ? dfb : 0u) | p.low_ncc_mask();
            if (tbr) {
                p.pk |= F_VIEW_REMOVED;
                p.sel_erase_mask(tbr);        // LocalViewSelection::replaceViews (local_view_selection.cc:150-160)
                p.pk &= ~F_LVS_OK;
                p.set_stage(LVS_REPL);
                return false;
            }
            if (dfb == 0u) { p.pk |= F_CONVERGED; p.set_stage(DONE); return true; }
            ++p.iter;
        } else if (stage == REPL) {
            ++p.iter;
        }
        // first four iterations only refine depth (:177-180)
        while (p.iter < 4 && p.is(F_OPTI)) {
            const bool moved = depth_step(p, po);
            ++p.iter;
            if (moved && p.is(F_OPTI)) { p.set_stage(FIRST); return false; }
        }
        if (!p.is(F_OPTI)) { p.set_stage(DONE); return true; }
        // head of the main loop (:184-203)
        if (!((unsigned)p.iter < p.st->max_iterations && p.is(F_LVS_OK))) { p.set_stage(DONE); return true; }
        const bool normal = (p.iter % 5 == 4) || p.is(F_VIEW_REMOVED);
        p.put(F_NORMAL, normal);
        if (!p.is(F_HAS_NCC) || (normal && !p.is(F_HAS_NORMAL))) { p.set_stage(PRE); return false; }   // only after a depth step with denom <= 0
        // (oldNCC = ncc here in the reference: the comparison is taken when the next pass overwrites the NCC)
        p.pk &= ~F_OPTI;
        if (normal) { normal_step(p, po); p.pk &= ~F_VIEW_REMOVED; p.pk |= F_WAS_NORMAL; }
        else { depth_step(p, po); p.pk &= ~F_WAS_NORMAL; }
        if (!p.is(F_OPTI)) { p.set_stage(DONE); return true; }
        p.set_stage(POST);
        return false;
    }
};

} // namespace b200mvs
