// The host phase of DMRecon::start: analyzeFeatures + GlobalViewSelection (dmrecon.cc:179-208,
// global_view_selection.cc:17-101) and the seed list of processFeatures (dmrecon.cc:258-292).  It has two routes, the
// host planner (b200mvs.cu global_view_selection / collect_seeds) and the device planner below, one reference view per
// CTA.  Their results are an integer selection and a seed list, so they must agree bit for bit.  This file holds the
// planner's arithmetic for both routes:
//   * both read the same input (PlanInput) and call the same __host__ __device__ helpers and per-feature steps.  Every
//     float operation is the reference's, in the reference's order, as an IEEE single operation that the compiler neither
//     contracts nor reorders (dot3 = ((0 + a0 b0) + a1 b1) + a2 b2, true division and square root, the one double division
//     of the resolution ratio).  The device spells them as round-to-nearest intrinsics; on the host the plain operators
//     are the same operations as long as the host compiler is given no FMA or fast-math flags;
//   * the parallax factor needs acos, which no device function reproduces bit for bit for the host's libm.  It depends on
//     the float dot product alone, so the host tabulates it for every float in [dot_skip, 1] with its own plx_factor
//     (fill_table) and the device looks it up;
//   * the device planner's greedy loop is its own: a candidate's benefit is a sequential sum over its entries in featInd
//     order, one thread per candidate, and an entry's score multiplies the factors of the selected views in ascending
//     view id (the std::set order), not in selection order.
// The device planner's per-view work is written as phases: each runs over `tid` in [0, nt) with no barrier inside, and
// the caller puts a barrier between two phases.  The kernel runs a phase with one CTA's threads; tests/emu runs it with a
// loop over tid.
#pragma once
#if defined(B200MVS_HOST_EMU)
#include "simt_emu.h"      // tests/emu: runs this very file on the CPU (test infrastructure)
#else
#include <cuda_runtime.h>
#endif
#include <stdint.h>
#include <cmath>
#include <cstring>
#include <algorithm>

namespace b200mvs_plan {

constexpr int MAX_SEL = 32;                       // globalVSMax <= 32 (check_settings)
constexpr uint64_t TABLE_CAP = 1ull << 22;        // factor table entries; above: plan on host threads
constexpr int SEED_CHUNK = 64;                    // features per thread of the ordered seed compaction

// PLAN_FN: the device planner's code (device, or the CPU under tests/emu); PLAN_HD: the code both planners call
#if defined(B200MVS_HOST_EMU)
#define PLAN_FN inline
inline void atomic_or(unsigned* p, unsigned v) { __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
inline void atomic_add(int* p, int v) { __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
inline unsigned f2u(float f) { return __float_as_uint(f); }
#else
#define PLAN_FN __device__ __forceinline__
__device__ __forceinline__ void atomic_or(unsigned* p, unsigned v) { atomicOr(p, v); }
__device__ __forceinline__ void atomic_add(int* p, int v) { atomicAdd(p, v); }
__device__ __forceinline__ unsigned f2u(float f) { return __float_as_uint(f); }
#endif
#define PLAN_HD __host__ __device__ __forceinline__

// ---- the rounding primitives: one IEEE operation each, round to nearest ----
#if defined(__CUDA_ARCH__)
PLAN_HD float fadd(float a, float b) { return __fadd_rn(a, b); }
PLAN_HD float fmul(float a, float b) { return __fmul_rn(a, b); }
PLAN_HD float fdiv(float a, float b) { return __fdiv_rn(a, b); }
PLAN_HD float fsqrt(float a) { return __fsqrt_rn(a); }
PLAN_HD double ddiv(double a, double b) { return __ddiv_rn(a, b); }
PLAN_HD float ffloor(float a) { return floorf(a); }
PLAN_HD float fceil(float a) { return ceilf(a); }
#else
PLAN_HD float fadd(float a, float b) { return a + b; }
PLAN_HD float fmul(float a, float b) { return a * b; }
PLAN_HD float fdiv(float a, float b) { return a / b; }
PLAN_HD float fsqrt(float a) { return std::sqrt(a); }
PLAN_HD double ddiv(double a, double b) { return a / b; }
PLAN_HD float ffloor(float a) { return std::floor(a); }
PLAN_HD float fceil(float a) { return std::ceil(a); }
#endif

// ---- the host's parallax factor (global_view_selection.cc:80-81 / :93-97); the host planner and PlanTable call it ----
// dot_skip: below it the parallax is certainly above minParallax, so the factor is 1 without an acos
inline float host_dot_skip(float min_parallax)
{
    return (float)std::cos(((double)min_parallax + 0.05) * 3.14159265358979323846 / 180.0);
}
inline float host_plx_factor(float dt, float dot_skip, float min_parallax)
{
    if (dt < dot_skip) return 1.f;
    const float dp = std::max(std::min(dt, 1.f), -1.f);
    const float plx = std::acos(dp) * 180.f / 3.141592653589793f;
    if (plx < min_parallax) { const float q = plx / 10.f; return q * q; }
    return 1.f;
}
// Entries of the factor table: one per float bit pattern in [dot_skip, 1]; 0 when the device cannot plan (dot_skip <= 0
// or more than TABLE_CAP entries)
inline uint64_t table_entries(float dot_skip)
{
    if (!(dot_skip > 0.f) || dot_skip > 1.f) return 0;
    uint32_t lo, hi;
    const float one = 1.f;
    std::memcpy(&lo, &dot_skip, 4);
    std::memcpy(&hi, &one, 4);
    const uint64_t n = (uint64_t)(hi - lo) + 1;
    return n <= TABLE_CAP ? n : 0;
}
// table[i] = host_plx_factor(float with bits bits(dot_skip) + i)
inline void fill_table(float* table, uint64_t n, float dot_skip, float min_parallax)
{
    uint32_t lo;
    std::memcpy(&lo, &dot_skip, 4);
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t b = lo + (uint32_t)i;
        float dt;
        std::memcpy(&dt, &b, 4);
        table[i] = host_plx_factor(dt, dot_skip, min_parallax);
    }
}
// the device's factor: host_plx_factor through the table (dt > 1 clamps to 1 as the host's min does, NaN gives 1)
PLAN_FN float plx_lookup(float dt, float dot_skip, const float* table)
{
    if (!(dt >= dot_skip)) return 1.f;
    const float c = dt < 1.f ? dt : 1.f;
    return table[f2u(c) - f2u(dot_skip)];
}

// ---- inputs ----
struct PlanView {                 // what planning reads of a view (HostView)
    float campos[3];
    float w2c[12];
    float proj0[9];               // level 0: the frustum test
    float inv0;                   // level 0 invproj[0]: the footprint of a candidate
    float proj_s[9];              // level `scale` of a reference view: the seed's pixel
    float inv_s;                  // level `scale` invproj[0]: the footprint of the reference view
    int w0, h0;
    int valid;
    int pad;
};

struct PlanInput {                // one planning call: host arrays for the host planner, their copies for every CTA of a launch
    const PlanView* views;
    const float* feat_pos;        // 3 per feature
    const int* feat_off;          // CSR feature -> refs (as registered, duplicates and bad ids included)
    const int* feat_refs;
    const int* vf_off;            // CSR view -> ascending ids of the features that reference it
    const int* vf_ids;
    const float* table;           // the device planner's factor table (the host planner computes the factor)
    int nv, nf;
    float dot_skip;
    float aabb_min[3], aabb_max[3];
    int gvs_max;
};

struct SeedOut { int x, y; float depth; };

// Where one reference view's workspace and results live: offsets in 4-byte words from the job's base
struct JobLayout {
    uint64_t foff, ecand, edir, ebase, escore, eperm, clist, coff, benefit, state, wanted, ccount, words;
};
__host__ __device__ inline JobLayout job_layout(int F, uint64_t E, int nv, int nf)
{
    JobLayout L;
    uint64_t o = 0;
    L.foff = o;    o += (uint64_t)F + 1;
    L.ecand = o;   o += E;
    L.edir = o;    o += 3 * E;
    L.ebase = o;   o += E;
    L.escore = o;  o += E;
    L.eperm = o;   o += E;
    L.clist = o;   o += E;
    L.coff = o;    o += (uint64_t)nv + 1;
    L.benefit = o; o += (uint64_t)nv;
    L.state = o;   o += (uint64_t)nv;
    L.wanted = o;  o += ((uint64_t)nf + 31) / 32;
    L.ccount = o;  o += ((uint64_t)nf + SEED_CHUNK - 1) / SEED_CHUNK + 1;
    L.words = o;
    return L;
}
// results of one reference view: [0] n_sel, [1] n_seeds, [2] entries, [3] the view selected last (-1: none),
// [4..4+MAX_SEL) the selection, ascending, then the seeds
constexpr int OUT_SEL = 4;
constexpr int OUT_HEAD = OUT_SEL + MAX_SEL;
__host__ __device__ inline uint64_t out_words(uint64_t seed_cap) { return OUT_HEAD + 3 * seed_cap; }

struct PlanJob {                  // one reference view of a launch
    int ref;
    int F;                        // features that reference it
    uint64_t E;                   // bound on its (candidate, feature) entries: the refs of those features
    uint64_t ws;                  // word offset of its workspace (JobLayout) in the launch's workspace
    uint64_t out;                 // word offset of its results in the launch's output
    uint64_t seed_cap;
};

enum { ST_AVAIL = 1, ST_SELECTED = 2 };

// ---- the reference float arithmetic (libs/math conventions, SURVEY.md §8a) ----
PLAN_HD float dot3(const float* a, const float* b)
{
    return fadd(fadd(fadd(0.0f, fmul(a[0], b[0])), fmul(a[1], b[1])), fmul(a[2], b[2]));
}
PLAN_HD void world_to_cam(const PlanView& v, const float* p, float* o)
{
    for (int i = 0; i < 3; ++i) o[i] = fadd(dot3(v.w2c + 4 * i, p), v.w2c[4 * i + 3]);
}
PLAN_HD void mat3_mul(const float* m, const float* x, float* o) { for (int i = 0; i < 3; ++i) o[i] = dot3(m + 3 * i, x); }
// SingleView::pointInFrustum (single_view.cc:109-121)
PLAN_HD bool point_in_frustum(const PlanView& v, const float* wp)
{
    float cp[3], sp[3];
    world_to_cam(v, wp, cp);
    if (cp[2] <= 0.0f) return false;
    mat3_mul(v.proj0, cp, sp);
    const float x = fadd(fdiv(sp[0], sp[2]), -0.5f);
    const float y = fadd(fdiv(sp[1], sp[2]), -0.5f);
    return x >= 0 && x <= (float)(v.w0 - 1) && y >= 0 && y <= (float)(v.h0 - 1);
}
PLAN_HD bool in_aabb(const PlanInput& in, const float* p)
{
    for (int i = 0; i < 3; ++i) if (p[i] < in.aabb_min[i] || p[i] > in.aabb_max[i]) return false;
    return true;
}
PLAN_HD void unit_dir(const PlanView& v, const float* p, float* d)
{
    d[0] = fadd(p[0], -v.campos[0]); d[1] = fadd(p[1], -v.campos[1]); d[2] = fadd(p[2], -v.campos[2]);
    const float n = fsqrt(dot3(d, d));
    d[0] = fdiv(d[0], n); d[1] = fdiv(d[1], n); d[2] = fdiv(d[2], n);
}
PLAN_HD float foot_print(const PlanView& v, float inv, const float* p)
{
    float c[3];
    world_to_cam(v, p, c);
    return fmul(c[2], inv);
}
PLAN_HD float round_mve(float x) { return x > 0.0f ? ffloor(fadd(x, 0.5f)) : fceil(fadd(x, -0.5f)); }

// ---- the per-feature steps of both planners ----
// the reference view sees feature position p and p lies in the box: the features a plan is made of (dmrecon.cc:191-196,
// :278-284)
PLAN_HD bool seen_in_box(const PlanInput& in, const PlanView& rv, const float* p)
{
    return point_in_frustum(rv, p) && in_aabb(in, p);
}
// the resolution term of a candidate's score on a feature (global_view_selection.cc:80-87): the reference view's footprint
// mfp over the candidate's, 1 between 1 and 2, 2 / ratio above 2
PLAN_HD float footprint_ratio(const PlanView& tv, const float* p, float mfp)
{
    const float nfp = foot_print(tv, tv.inv0, p);
    float ratio = fdiv(mfp, nfp);
    if (ratio > 2.) ratio = (float)ddiv(2., (double)ratio);
    else if (ratio > 1.) ratio = 1.;
    return ratio;
}
// the seed of a feature at p that the reference view rv sees: its pixel at level `scale` by round_mve, depth = distance to
// the camera centre (dmrecon.cc:289-292)
PLAN_HD void seed_of(const PlanView& rv, const float* p, SeedOut& s)
{
    float cp[3], sp[3];
    world_to_cam(rv, p, cp);
    mat3_mul(rv.proj_s, cp, sp);
    const float px = fadd(fdiv(sp[0], sp[2]), -0.5f), py = fadd(fdiv(sp[1], sp[2]), -0.5f);
    const float dv[3] = {fadd(p[0], -rv.campos[0]), fadd(p[1], -rv.campos[1]), fadd(p[2], -rv.campos[2])};
    s.x = (int)round_mve(px);
    s.y = (int)round_mve(py);
    s.depth = fsqrt(dot3(dv, dv));
}

// One reference view: the phases in order, with a barrier between two.  `ws` and `out` point at the job's words.
struct PlanBlock {
    const PlanInput* in;
    const PlanJob* job;
    uint32_t* ws;
    uint32_t* out;
    JobLayout L;

    PLAN_FN void bind(const PlanInput* in_, const PlanJob* job_, uint32_t* ws_base, uint32_t* out_base)
    {
        in = in_; job = job_;
        ws = ws_base + job->ws;
        out = out_base + job->out;
        L = job_layout(job->F, job->E, in->nv, in->nf);
    }
    PLAN_FN int* I(uint64_t o) const { return reinterpret_cast<int*>(ws + o); }
    PLAN_FN float* Fp(uint64_t o) const { return reinterpret_cast<float*>(ws + o); }
    PLAN_FN int feat_of(int t) const { return in->vf_ids[in->vf_off[job->ref] + t]; }
    PLAN_FN bool candidate_ok(int vid) const
    {
        return vid >= 0 && vid < in->nv && vid != job->ref && in->views[vid].valid;
    }

    // A: entries per local feature t (the features of the reference view, ascending) into foff[t + 1]; candidate state
    PLAN_FN void count_entries(int tid, int nt)
    {
        int* foff = I(L.foff);
        const PlanView& rv = in->views[job->ref];
        for (int t = tid; t < job->F; t += nt) {
            const int fi = feat_of(t);
            const float* p = in->feat_pos + 3 * (size_t)fi;
            int c = 0;
            if (seen_in_box(*in, rv, p))
                for (int r = in->feat_off[fi]; r < in->feat_off[fi + 1]; ++r) {
                    const int vid = in->feat_refs[r];
                    if (candidate_ok(vid) && point_in_frustum(in->views[vid], p)) ++c;
                }
            foff[t + 1] = c;
        }
        int* state = I(L.state);
        int* coff = I(L.coff);
        for (int v = tid; v < in->nv; v += nt) { state[v] = candidate_ok(v) ? ST_AVAIL : 0; coff[v] = 0; }
        if (tid == 0) { foff[0] = 0; coff[in->nv] = 0; }
    }
    // B (one thread): feature offsets
    PLAN_FN void scan_features(int tid)
    {
        if (tid != 0) return;
        int* foff = I(L.foff);
        for (int t = 0; t < job->F; ++t) foff[t + 1] += foff[t];
        out[2] = (uint32_t)foff[job->F];
    }
    // C: the feature-major entries - candidate, unit direction, base score (:78-87) - and each candidate's count
    PLAN_FN void write_entries(int tid, int nt)
    {
        const int* foff = I(L.foff);
        int* ecand = I(L.ecand);
        float* edir = Fp(L.edir);
        float* ebase = Fp(L.ebase);
        float* escore = Fp(L.escore);
        int* coff = I(L.coff);
        const PlanView& rv = in->views[job->ref];
        const float scale_inv = rv.inv_s;
        for (int t = tid; t < job->F; t += nt) {
            int e = foff[t];
            if (foff[t + 1] == e) continue;
            const int fi = feat_of(t);
            const float* p = in->feat_pos + 3 * (size_t)fi;
            float dr[3];
            unit_dir(rv, p, dr);
            const float mfp = foot_print(rv, scale_inv, p);
            for (int r = in->feat_off[fi]; r < in->feat_off[fi + 1]; ++r) {
                const int vid = in->feat_refs[r];
                if (!candidate_ok(vid)) continue;
                const PlanView& tv = in->views[vid];
                if (!point_in_frustum(tv, p)) continue;
                float d[3];
                unit_dir(tv, p, d);
                float score = fmul(1.f, plx_lookup(dot3(dr, d), in->dot_skip, in->table));
                score = fmul(score, footprint_ratio(tv, p, mfp));
                ecand[e] = vid;
                edir[3 * (size_t)e] = d[0]; edir[3 * (size_t)e + 1] = d[1]; edir[3 * (size_t)e + 2] = d[2];
                ebase[e] = score;
                escore[e] = score;
                atomic_add(&coff[vid + 1], 1);
                ++e;
            }
        }
    }
    // D (one thread): candidate offsets
    PLAN_FN void scan_candidates(int tid)
    {
        if (tid != 0) return;
        int* coff = I(L.coff);
        for (int v = 0; v < in->nv; ++v) coff[v + 1] += coff[v];
    }
    // E: each candidate's entries in featInd order (= ascending entry index); each feature's entries by ascending
    // candidate (stable), the order its selected views multiply in
    PLAN_FN void order_entries(int tid, int nt)
    {
        const int* foff = I(L.foff);
        const int* ecand = I(L.ecand);
        const int* coff = I(L.coff);
        int* clist = I(L.clist);
        int* eperm = I(L.eperm);
        const int E = foff[job->F];
        for (int v = tid; v < in->nv; v += nt) {
            if (coff[v + 1] == coff[v]) continue;
            int k = coff[v];
            for (int e = 0; e < E; ++e) if (ecand[e] == v) clist[k++] = e;
        }
        for (int t = tid; t < job->F; t += nt)
            for (int e = foff[t]; e < foff[t + 1]; ++e) {
                int x = e;
                for (; x > foff[t] && ecand[eperm[x - 1]] > ecand[e]; --x) eperm[x] = eperm[x - 1];
                eperm[x] = e;
            }
    }
    // F: benefitFromView of every available candidate: its scores summed in featInd order
    PLAN_FN void benefits(int tid, int nt)
    {
        const int* coff = I(L.coff);
        const int* clist = I(L.clist);
        const int* state = I(L.state);
        const float* escore = Fp(L.escore);
        float* benefit = Fp(L.benefit);
        for (int v = tid; v < in->nv; v += nt) {
            if (!(state[v] & ST_AVAIL)) continue;
            float b = 0.f;
            for (int k = coff[v]; k < coff[v + 1]; ++k) b = fadd(b, escore[clist[k]]);
            benefit[v] = b;
        }
    }
    // G (one thread): the best candidate (strictly larger benefit, ascending id, as the host loop does) into out[3], or -1;
    // the selection is kept ascending
    PLAN_FN void select(int tid)
    {
        if (tid != 0) return;
        int* state = I(L.state);
        const float* benefit = Fp(L.benefit);
        const int n_sel = (int)out[0];
        float max_b = 0.f;
        int max_v = -1;
        if (n_sel < in->gvs_max)
            for (int v = 0; v < in->nv; ++v)
                if ((state[v] & ST_AVAIL) && benefit[v] > max_b) { max_b = benefit[v]; max_v = v; }
        out[3] = (uint32_t)max_v;
        if (max_v < 0) return;
        int x = n_sel;
        for (; x > 0 && (int)out[OUT_SEL + x - 1] > max_v; --x) out[OUT_SEL + x] = out[OUT_SEL + x - 1];
        out[OUT_SEL + x] = (uint32_t)max_v;
        out[0] = (uint32_t)(n_sel + 1);
        state[max_v] = ST_SELECTED;
    }
    // H: rescore the entries of every feature the view selected last sees: base times the factors of the selected views
    // that see the feature, in ascending view id; a view with two refs of a feature counts once (seesFeature)
    PLAN_FN void rescore(int tid, int nt, int s)
    {
        const int* foff = I(L.foff);
        const int* ecand = I(L.ecand);
        const int* eperm = I(L.eperm);
        const int* state = I(L.state);
        const float* edir = Fp(L.edir);
        const float* ebase = Fp(L.ebase);
        float* escore = Fp(L.escore);
        for (int t = tid; t < job->F; t += nt) {
            int selq[MAX_SEL];                      // an entry of each selected view that sees the feature, ascending view
            int ns = 0, prev = -1;
            bool sees = false;
            for (int x = foff[t]; x < foff[t + 1]; ++x) {
                const int q = eperm[x];
                const int v = ecand[q];
                if (v == prev || !(state[v] & ST_SELECTED)) continue;
                prev = v;
                selq[ns++] = q;
                sees |= v == s;
            }
            if (!sees) continue;
            for (int e = foff[t]; e < foff[t + 1]; ++e) {
                if (!(state[ecand[e]] & ST_AVAIL)) continue;
                float score = ebase[e];
                for (int i = 0; i < ns; ++i) {
                    const float f = plx_lookup(dot3(&edir[3 * (size_t)selq[i]], &edir[3 * (size_t)e]), in->dot_skip, in->table);
                    if (f != 1.f) score = fmul(score, f);
                }
                escore[e] = score;
            }
        }
    }
    // I: the features seen by the reference view or a selected view (dmrecon.cc:260-276)
    PLAN_FN void clear_wanted(int tid, int nt)
    {
        unsigned* w = reinterpret_cast<unsigned*>(ws + L.wanted);
        for (int i = tid; i < (in->nf + 31) / 32; i += nt) w[i] = 0;
    }
    PLAN_FN void mark_wanted(int tid, int nt)
    {
        unsigned* w = reinterpret_cast<unsigned*>(ws + L.wanted);
        const int n_sel = (int)out[0];
        for (int k = -1; k < n_sel; ++k) {
            const int v = k < 0 ? job->ref : (int)out[OUT_SEL + k];
            for (int i = in->vf_off[v] + tid; i < in->vf_off[v + 1]; i += nt) {
                const int fi = in->vf_ids[i];
                atomic_or(&w[fi >> 5], 1u << (fi & 31));
            }
        }
    }
    PLAN_FN bool seeds_from(int fi, SeedOut* s) const
    {
        const unsigned* w = reinterpret_cast<const unsigned*>(ws + L.wanted);
        if (!((w[fi >> 5] >> (fi & 31)) & 1u)) return false;
        const PlanView& rv = in->views[job->ref];
        const float* p = in->feat_pos + 3 * (size_t)fi;
        if (!seen_in_box(*in, rv, p)) return false;
        if (s) seed_of(rv, p, *s);
        return true;
    }
    // J: seeds per chunk of SEED_CHUNK features
    PLAN_FN void count_seeds(int tid, int nt)
    {
        int* cc = I(L.ccount);
        const int nch = (in->nf + SEED_CHUNK - 1) / SEED_CHUNK;
        for (int c = tid; c < nch; c += nt) {
            int n = 0;
            for (int fi = c * SEED_CHUNK; fi < in->nf && fi < (c + 1) * SEED_CHUNK; ++fi) n += seeds_from(fi, nullptr);
            cc[c + 1] = n;
        }
        if (tid == 0) cc[0] = 0;
    }
    // K (one thread): chunk offsets
    PLAN_FN void scan_seeds(int tid)
    {
        if (tid != 0) return;
        int* cc = I(L.ccount);
        const int nch = (in->nf + SEED_CHUNK - 1) / SEED_CHUNK;
        for (int c = 0; c < nch; ++c) cc[c + 1] += cc[c];
        out[1] = (uint32_t)cc[nch];
    }
    // L: the seeds in feature order
    PLAN_FN void write_seeds(int tid, int nt)
    {
        const int* cc = I(L.ccount);
        SeedOut* so = reinterpret_cast<SeedOut*>(out + OUT_HEAD);
        const int nch = (in->nf + SEED_CHUNK - 1) / SEED_CHUNK;
        for (int c = tid; c < nch; c += nt) {
            int k = cc[c];
            for (int fi = c * SEED_CHUNK; fi < in->nf && fi < (c + 1) * SEED_CHUNK; ++fi)
                if (seeds_from(fi, &so[k])) ++k;
        }
    }
};

// The whole plan of one reference view; `sync` is the barrier between two phases.  out[0] (the selection size) is
// zeroed by the caller before the launch.
template <typename Sync> PLAN_FN void plan_view(PlanBlock& B, int tid, int nt, Sync sync)
{
    B.count_entries(tid, nt);       sync();
    B.scan_features(tid);           sync();
    B.write_entries(tid, nt);       sync();
    B.scan_candidates(tid);         sync();
    B.order_entries(tid, nt);       sync();
    for (;;) {
        B.benefits(tid, nt);        sync();
        B.select(tid);              sync();
        const int s = (int)B.out[3];                // every thread reads the same word between two barriers
        if (s < 0) break;
        B.rescore(tid, nt, s);      sync();
    }
    B.clear_wanted(tid, nt);        sync();
    B.mark_wanted(tid, nt);         sync();
    B.count_seeds(tid, nt);         sync();
    B.scan_seeds(tid);              sync();
    B.write_seeds(tid, nt);
}

} // namespace b200mvs_plan
