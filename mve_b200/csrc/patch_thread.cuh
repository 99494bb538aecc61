// Device-side patch optimisation, THROUGHPUT variant: one THREAD per patch (32 patches per warp).
//
// Same function as PatchW in patch_warp.cuh - one mvs::PatchOptimization of the reference
// (libs/dmrecon/patch_optimization.cc:21-364 with PatchSampler patch_sampler.cc:19-393, LocalViewSelection
// local_view_selection.cc:19-160 and mvs_tools.cc:98-199) - organised for large frontier rounds, where there are far more
// queue entries than lanes on the chip:
//   * a lane walks the 25 samples of its own patch in a loop (pipelined two samples deep), so no lane idles on a 25-of-32
//     mapping, nothing is reduced across lanes (no shuffles at all) and everything that is uniform per patch - view
//     constants, level choice, colour scales, the state machine - is paid once per 32 patches instead of once per patch;
//   * nothing per-sample survives an iteration of the sample loop: the sums the reference forms in separate passes over
//     stored samples are accumulated in ONE sweep, in forms that do not need the means or the updated colour scale first.
//     Every lane accumulates the same 18 per-channel sums, whatever its state asks for (the lanes of a warp are at
//     different states: per-state sums would make the warp pay for all of them), with y = n - p around the pivot
//     p = meanX * masterMeanCol (the neighbour colours scatter around it, so the variance is formed without cancellation):
//       sum(y), sum(y^2), sum(m y), sum(d m), sum(d n), sum(d d)
//     and derives after the sweep what it asked for:
//       NCC (patch_sampler.cc:143-162)      devXY = sum_ch(sum(m y) - meanX sum(y)), sqrDevY = sum_ch(sum(y^2) - sum(y)^2 / 25)
//       colour scale (patch_optimization.cc:88-110)   ab = sum(m n) - cs sum(n n) with sum(m n) = sum(m y) + 25 p meanX and
//                                           sum(n n) = sum(y^2) + p (2 sum(y) + 25 p)
//       Gauss-Newton, depth only (:283-288) sum_ch cs (sum(d m) - cs sum(d n)) / sum_ch cs^2 sum(d d), with the current
//                                           scale or the one just updated;
//     only the normal equations (:324-343, read by one state in five) are summed per sample, channels first (by every
//     lane, without a branch - nearly every warp holds a lane that reads them): with q = sum_ch (cs d)^2
//     and s = sum_ch cs d (m - cs n) a sample adds (1, di, dj)^T (1, di, dj) q and (1, di, dj) s, whose (1, 1) / first
//     entries are the depth-only denominator / numerator above.  Only a view replacement (colour scale AND normal step at
//     one state, rare) sweeps a view twice;
//   * geometry per sample is evaluated in the neighbour's camera frame directly: with u = R^T K^-1 (x, y, 1) the patch point
//     is C + t u / |u| and its image W (C + t u/|u|) + T = (W C + T) + (t / |u|) (W u); W C + T and W u0, W ua, W ub (u is
//     affine in the pixel offsets) are formed once per view and sweep - 12 FMAs per sample for BOTH projections of
//     patch_sampler.cc:94-133 instead of two full point transforms.  Same values up to rounding order (<= 2 ulp on pixel
//     coordinates; measured against the oracle in tests/test_gpu_parity.py and on the CPU in
//     tests/test_device_code_emulated.py).
// The state and its state machine (stages, iteration counting, view replacement) are PatchState's (patch_opt.cuh).
#pragma once
#include "patch_opt.cuh"
#if defined(B200MVS_HOST_EMU)
#include <cassert>
#endif

#ifndef OPT_TPB
#define OPT_TPB 384          // threads per CTA of the patch-optimisation kernels (b200mvs.cu): one CTA per SM shares ONE 64 KB table
#endif

namespace b200mvs {

// Pixel offsets (di, dj) of sample k in the 5x5 window, row-major: the sample loop reads them as constants instead of
// deriving them from k with a division and two int-to-float conversions.
struct alignas(8) SampleOffset { float di, dj; };
#if !defined(B200MVS_HOST_EMU)
__constant__
#endif
static const SampleOffset k_sample_offset[NS] = {
    {-2.f, -2.f}, {-1.f, -2.f}, {0.f, -2.f}, {1.f, -2.f}, {2.f, -2.f},
    {-2.f, -1.f}, {-1.f, -1.f}, {0.f, -1.f}, {1.f, -1.f}, {2.f, -1.f},
    {-2.f,  0.f}, {-1.f,  0.f}, {0.f,  0.f}, {1.f,  0.f}, {2.f,  0.f},
    {-2.f,  1.f}, {-1.f,  1.f}, {0.f,  1.f}, {1.f,  1.f}, {2.f,  1.f},
    {-2.f,  2.f}, {-1.f,  2.f}, {0.f,  2.f}, {1.f,  2.f}, {2.f,  2.f}};

struct PatchT : PatchState {
    // ---- constants of the thread ----
    const DevSettings* st;
    const ViewParams* views;
#if defined(B200MVS_HOST_EMU)
    const float* lut_tab;      // lane-replicated srgb2lin table (lut_k); on the device: table() / lane_offset()
    unsigned lane4;            // 4 * (lane of this thread)
    unsigned mt_k[NS];         // master texels of the patch; on the device: mt_tab()
#endif
    // ---- constants of the patch ----
    const JobParams* job;
    unsigned xy;               // x | y << 16 of the patch centre
    float u0x, u0y, u0z;       // R^T K^-1 (x + .5, y + .5, 1): un-normalised ray of the centre pixel
    float uax, uay, uaz;       // R^T K^-1 (1, 0, 0): change of the ray per pixel in x
    float ubx, uby, ubz;       // R^T K^-1 (0, 1, 0): ... in y
    float c0x, c0y, c0z;       // camera centre of the reference view
    float mx0, mx1, mx2;       // meanX per channel (patch_sampler.cc:333-339)
    float crx, cry, crz;       // masterViewDirs[12]
    float cpx, cpy, cpz;       // patchPoints[12]
    float mfp, inv_mfp;        // footPrintScaled(patchPoints[12]) and its reciprocal
    float mm, inv_mm, sqrDevX; // masterMeanCol, its reciprocal, sqrDevX
    unsigned selp;             // the selected set: 4 x uint8 global slots, ascending, 0xFF = none
    // ---- per selected view (index = position in the ascending selected set) ----
    float cs[MAX_LOCAL][3];    // colorScale
    float ncc[MAX_LOCAL];      // NCC at the state of the last pass

    __device__ __forceinline__ int sel(int k) const { return (int)((selp >> (8 * k)) & 0xFFu); }
    __device__ __forceinline__ int px() const { return (int)(xy & 0xFFFFu); }
    __device__ __forceinline__ int py() const { return (int)(xy >> 16); }

    // ---- register arrays with a dynamic index ----
    template <typename T> static __device__ __forceinline__ T get4(const T (&a)[MAX_LOCAL], int k)
    {
        return k == 0 ? a[0] : (k == 1 ? a[1] : (k == 2 ? a[2] : a[3]));
    }
    template <typename T> static __device__ __forceinline__ void set4(T (&a)[MAX_LOCAL], int k, T v)
    {
#pragma unroll
        for (int i = 0; i < MAX_LOCAL; ++i) if (i == k) a[i] = v;
    }

    // The table is the first thing in the kernels' dynamic shared memory (b200mvs.cu, OPT_SMEM_BYTES).  Read through the
    // member - the object itself lives in shared memory - the compiler would no longer know which address space it points
    // to and emit generic loads for the 15 look-ups of every sample.
    __device__ __forceinline__ unsigned lane_offset() const
    {
#if defined(B200MVS_HOST_EMU)
        return lane4;
#else
        return (threadIdx.x & 31u) << 2;
#endif
    }
    __device__ __forceinline__ const float* table() const
    {
#if defined(B200MVS_HOST_EMU)
        return lut_tab;
#else
        extern __shared__ float b200mvs_dyn_smem[];
        return b200mvs_dyn_smem;
#endif
    }

    // The master texels of the patch, word k = sample k, constant for a whole optimisation: read from the reference image
    // once by init_sampler, then from shared memory by every sweep (a global gather of 32 unrelated patches per sample
    // before).  On the device the table follows the PatchT records of the CTA in the dynamic shared memory (b200mvs.cu,
    // OPT_SMEM_BYTES), word-major - word k of thread t at [k * OPT_TPB + t] - so a warp reading word k touches 32 banks,
    // and word k is a constant offset from the thread's own base.  Reached from the start of the shared memory, like
    // table(), so that the sample loop reads it with shared-memory loads.
#if defined(B200MVS_HOST_EMU)
    static constexpr unsigned MT_STRIDE = 1u;
#else
    static constexpr unsigned MT_STRIDE = OPT_TPB;
#endif
    static constexpr size_t MT_BYTES = sizeof(unsigned) * NS * OPT_TPB;      // the tables of a CTA
    __device__ __forceinline__ unsigned* mt_tab()
    {
#if defined(B200MVS_HOST_EMU)
        return mt_k;
#else
        extern __shared__ float b200mvs_dyn_smem[];
        return reinterpret_cast<unsigned*>(b200mvs_dyn_smem + (256 * LUT_STRIDE + OPT_TPB * (sizeof(PatchT) / sizeof(float)))) + threadIdx.x;
#endif
    }

    // un-normalised ray of the sample with pixel offsets (di, dj), its reciprocal length and the sample's depth parameter
    __device__ __forceinline__ void sample_ray(float di, float dj, float& ux, float& uy, float& uz, float& inv) const
    {
        ux = u0x + di * uax + dj * ubx;
        uy = u0y + di * uay + dj * uby;
        uz = u0z + di * uaz + dj * ubz;
        inv = rsqrt_fast(ux * ux + uy * uy + uz * uz);
    }

    // patch_sampler.cc:274-295 (+ the centre point / master footprint used by every sample set)
    __device__ __forceinline__ void compute_points()
    {
        bool bad = false;
#pragma unroll 5
        for (int k = 0; k < NS; ++k) {
            const float t = depth + (float)(k % 5 - 2) * dzI + (float)(k / 5 - 2) * dzJ;
            bad |= t <= 0.f;
        }
        if (bad) pk &= ~F_REF_OK;
        cpx = c0x + depth * crx;
        cpy = c0y + depth * cry;
        cpz = c0z + depth * crz;
        const ViewParams* rv = &views[job->ref_view];
        const float z = __ldg(&rv->w2c[8]) * cpx + __ldg(&rv->w2c[9]) * cpy + __ldg(&rv->w2c[10]) * cpz + __ldg(&rv->w2c[11]);
        mfp = z * job->ki0;     // single_view.h:160-164
        inv_mfp = rcp_fast(mfp);
    }

    // PatchSampler ctor (patch_sampler.cc:19-62) + computeMasterSamples (:298-345)
    __device__ __forceinline__ void init_sampler(int x, int y)
    {
        const float* const lut_tab = table();
        const unsigned lane4 = lane_offset();
        pk &= ~F_REF_OK; mm = 0.f; inv_mm = 0.f; sqrDevX = 0.f;
        mx0 = mx1 = mx2 = 0.f;
        crx = cry = crz = cpx = cpy = cpz = mfp = inv_mfp = 0.f;
        if (x - 2 < 0 || y - 2 < 0 || x + 2 > job->W - 1 || y + 2 > job->H - 1) return;
        {
            // viewRayScaled (single_view.cc:99-106, depthmap.cc:149-156): K^-1 has the sparsity of camera.cc:180-200
            const ViewParams* rv = &views[job->ref_view];
            const float r0 = __ldg(&rv->rot[0]), r1 = __ldg(&rv->rot[1]), r2 = __ldg(&rv->rot[2]), r3 = __ldg(&rv->rot[3]), r4 = __ldg(&rv->rot[4]);
            const float r5 = __ldg(&rv->rot[5]), r6 = __ldg(&rv->rot[6]), r7 = __ldg(&rv->rot[7]), r8 = __ldg(&rv->rot[8]);
            const float vx = job->ki0 * ((float)x + 0.5f) + job->ki2, vy = job->ki4 * ((float)y + 0.5f) + job->ki5;
            u0x = r0 * vx + r3 * vy + r6; u0y = r1 * vx + r4 * vy + r7; u0z = r2 * vx + r5 * vy + r8;
            uax = r0 * job->ki0; uay = r1 * job->ki0; uaz = r2 * job->ki0;
            ubx = r3 * job->ki4; uby = r4 * job->ki4; ubz = r5 * job->ki4;
            c0x = __ldg(&rv->campos[0]); c0y = __ldg(&rv->campos[1]); c0z = __ldg(&rv->campos[2]);
            const float inv = rsqrt_fast(u0x * u0x + u0y * u0y + u0z * u0z);
            crx = u0x * inv; cry = u0y * inv; crz = u0z * inv;
        }
        pk |= F_REF_OK;
        // master colours: mean, then the per-channel means and deviations of the normalised colours.  The first walk over
        // the master patch stores its texels in mt_tab(), the second reads them from there.
        unsigned* const mt = mt_tab();
        const uchar4* row = job->ref_img + (size_t)(y - 2) * job->ref_pitch + (x - 2);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f;
#pragma unroll 1
        for (int j = 0; j < 5; ++j) {
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                const unsigned t = reinterpret_cast<const unsigned*>(row)[i];
                s0 += lut_k<0>(lut_tab, lane4, t); s1 += lut_k<1>(lut_tab, lane4, t); s2 += lut_k<2>(lut_tab, lane4, t);
                mt[(5 * j + i) * MT_STRIDE] = t;
            }
            row += job->ref_pitch;
        }
        mm = (s0 + s1 + s2) / (3.f * NS);
        if (mm < 0.01f || mm > 0.99f) { pk &= ~F_REF_OK; return; }
        inv_mm = 1.f / mm;
        mx0 = (s0 * inv_mm) / (float)NS; mx1 = (s1 * inv_mm) / (float)NS; mx2 = (s2 * inv_mm) / (float)NS;
        float dev = 0.f;
#pragma unroll 1
        for (int j = 0; j < 5; ++j) {
#pragma unroll
            for (int i = 0; i < 5; ++i) {
                const unsigned t = mt[(5 * j + i) * MT_STRIDE];
                const float e0 = lut_k<0>(lut_tab, lane4, t) * inv_mm - mx0, e1 = lut_k<1>(lut_tab, lane4, t) * inv_mm - mx1, e2 = lut_k<2>(lut_tab, lane4, t) * inv_mm - mx2;
                dev += e0 * e0 + e1 * e1 + e2 * e2;
            }
        }
        sqrDevX = dev;
        compute_points();
    }

    // ---- one sweep of pass() over the 25 samples of a view ----
    // What a staged sample hands to its processing: the quad texel of the neighbour, the master texel, the bilinear weights
    // and the derivative step in pixels.
    struct Staged {
        uint4 Q;
        unsigned mt;
        float fx, fy, gx, gy;
    };
    // The constants of a sweep (registers), its sums and the code of one sample.  Every floating-point operation of a sample
    // is pinned (fma_rn / mul_rn / add_rn / sub_rn) in the contraction that the compiler chose for the rolled loop of the
    // earlier version of this file, so the values stay bit for bit the same wherever unrolling and peeling place the code.
    struct Sweep {
        const float* lut;
        unsigned lane4;
        float inv_mm;
        float u0x, u0y, u0z, uax, uay, uaz, ubx, uby, ubz, depth, dzI, dzJ;     // the patch (PatchT members)
        const unsigned* mt;        // its master texels (PatchT::mt_tab), MT_STRIDE words per sample
        float A0x, A0y, A0z, W0x, W0y, W0z, Wax, Way, Waz, Wbx, Wby, Wbz;       // the view: W C + T, W u0, W ua, W ub
        float Lax, Lay, Lcx, Lcy, wm1, hm1, step, dd;                           // its level, derivative step and scale
        const uint4* quad;
        unsigned qpitch;
        float pv0, pv1, pv2;       // NCC pivots
        float c0, c1, c2;          // colour scales (normal equations)
        // Every lane accumulates the same sums, whatever it derives from them after the sweep (the lanes of a warp are at
        // different states, and sums a lane would skip are still paid by the warp as divergent or predicated code).  That
        // includes the normal equations: nearly every warp holds a lane that forms them, so a per-lane branch around them
        // saved nothing and only split the loop body; a lane that does not form them never reads them.
        // Per channel, with y = n - p around the NCC pivot p = meanX * masterMeanCol:
        //   Sy = sum(y), Syy = sum(y^2), Smy = sum(m y)      -> NCC and colour scale (sum(m n), sum(n n))
        //   Sdm = sum(d m), Sdn = sum(d n), Sdd = sum(d^2)   -> Gauss-Newton numerator / denominator for any scale
        float Sya, Syb, Syc, Syya, Syyb, Syyc, Smya, Smyb, Smyc;
        float Sdma, Sdmb, Sdmc, Sdna, Sdnb, Sdnc, Sdda, Sddb, Sddc;
        // normal equations (patch_optimization.cc:324-343) on (1, di, dj) with the channels summed first; the (1, 1)
        // entry and the first right-hand side are the depth-only denominator and numerator
        float A1, A2, A3, A4, A5, B1, B2;

        __device__ __forceinline__ void clear()
        {
            Sya = Syb = Syc = Syya = Syyb = Syyc = Smya = Smyb = Smyc = 0.f;
            Sdma = Sdmb = Sdmc = Sdna = Sdnb = Sdnc = Sdda = Sddb = Sddc = 0.f;
            A1 = A2 = A3 = A4 = A5 = B1 = B2 = 0.f;
        }

        // Geometry of sample k (row-major in the 5x5 window, offsets from k_sample_offset), its quad load and its master
        // texel, without a branch.  Returns whether the sample projects inside the level (patch_sampler.cc:113-120); one
        // that does not fails the view, and its quad load reads from coordinate (0, 0), so no address is ever formed from an
        // outside projection.  The derivative step is evaluated for
        // every sample: a view without a derivative (r == 1 in pass()) never reads the sums it goes into.
        __device__ __forceinline__ bool stage(int k, Staged& s) const
        {
            const float di = k_sample_offset[k].di, dj = k_sample_offset[k].dj;
            const float ux = fma_rn(dj, ubx, fma_rn(di, uax, u0x)), uy = fma_rn(dj, uby, fma_rn(di, uay, u0y)), uz = fma_rn(dj, ubz, fma_rn(di, uaz, u0z));
            const float inv = rsqrt_fast(fma_rn(uz, uz, fma_rn(ux, ux, mul_rn(uy, uy))));
            const float s1 = mul_rn(fma_rn(dj, dzJ, fma_rn(di, dzI, depth)), inv);
            const float wx = fma_rn(dj, Wbx, fma_rn(di, Wax, W0x)), wy = fma_rn(dj, Wby, fma_rn(di, Way, W0y)), wz = fma_rn(dj, Wbz, fma_rn(di, Waz, W0z));
            const float hx = fma_rn(s1, wx, A0x), hy = fma_rn(s1, wy, A0y), hz = fma_rn(s1, wz, A0z);
            const float ih = rcp_fast(hz);
            const float qx = fma_rn(fma_rn(Lax, hx, mul_rn(Lcx, hz)), ih, -0.5f);
            const float qy = fma_rn(fma_rn(Lay, hy, mul_rn(Lcy, hz)), ih, -0.5f);
            const bool ok = qx > 0.f && qx < wm1 && qy > 0.f && qy < hm1;
            const float s2 = fma_rn(step, inv, s1);
            const float kx = fma_rn(s2, wx, A0x), ky = fma_rn(s2, wy, A0y), kz = fma_rn(s2, wz, A0z);
            const float ik = rcp_fast(kz);
            s.gx = sub_rn(fma_rn(fma_rn(Lax, kx, mul_rn(Lcx, kz)), ik, -0.5f), qx);
            s.gy = sub_rn(fma_rn(fma_rn(Lay, ky, mul_rn(Lcy, kz)), ik, -0.5f), qy);
            const float cx = ok ? qx : 0.f, cy = ok ? qy : 0.f;
            const int left = (int)floorf(cx), top = (int)floorf(cy);
#if defined(B200MVS_HOST_EMU)
            assert(left >= 0 && top >= 0 && (float)left < wm1 && (float)top < hm1);      // the 2x2 quad lies in the level
#endif
            s.fx = sub_rn(cx, (float)left);
            s.fy = sub_rn(cy, (float)top);
            s.Q = __ldg(quad + ((unsigned)top * qpitch + (unsigned)left));
            s.mt = mt[k * MT_STRIDE];
            return ok;
        }

        // Table look-ups, bilinear value and derivative (mvs_tools.cc:119-128,188-197) and the sums of sample k.
        __device__ __forceinline__ void sample(int k, const Staged& in)
        {
            const float fx = in.fx, fy = in.fy, gx = in.gx, gy = in.gy;
            const float m[3] = {mul_rn(lut_k<0>(lut, lane4, in.mt), inv_mm), mul_rn(lut_k<1>(lut, lane4, in.mt), inv_mm), mul_rn(lut_k<2>(lut, lane4, in.mt), inv_mm)};
            float a[3], b[3], c[3], e[3];
            a[0] = lut_k<0>(lut, lane4, in.Q.x); a[1] = lut_k<1>(lut, lane4, in.Q.x); a[2] = lut_k<2>(lut, lane4, in.Q.x);
            b[0] = lut_k<0>(lut, lane4, in.Q.y); b[1] = lut_k<1>(lut, lane4, in.Q.y); b[2] = lut_k<2>(lut, lane4, in.Q.y);
            c[0] = lut_k<0>(lut, lane4, in.Q.z); c[1] = lut_k<1>(lut, lane4, in.Q.z); c[2] = lut_k<2>(lut, lane4, in.Q.z);
            e[0] = lut_k<0>(lut, lane4, in.Q.w); e[1] = lut_k<1>(lut, lane4, in.Q.w); e[2] = lut_k<2>(lut, lane4, in.Q.w);
            // n = (1 - fy)((1 - fx) a + fx b) + fy((1 - fx) c + fx e)
            // d = (gx (b - a) + gy (c - a) + (gy fx + gx fy)(a - b - c + e)) * dd   (deriv /= stepSize, stepSize = 1 / dd,
            //     patch_sampler.cc:100,129-130)
            const float omfx = sub_rn(1.f, fx), omfy = sub_rn(1.f, fy), wxy = fma_rn(fy, gx, mul_rn(fx, gy));
            float n[3], d[3];
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float x0 = fma_rn(omfx, a[ch], mul_rn(fx, b[ch]));
                const float x3 = fma_rn(omfx, c[ch], mul_rn(fx, e[ch]));
                n[ch] = fma_rn(omfy, x0, mul_rn(fy, x3));
                const float t = fma_rn(gx, sub_rn(b[ch], a[ch]), mul_rn(gy, sub_rn(c[ch], a[ch])));
                d[ch] = mul_rn(fma_rn(wxy, add_rn(sub_rn(sub_rn(a[ch], b[ch]), c[ch]), e[ch]), t), dd);
            }
            const float y0 = sub_rn(n[0], pv0), y1 = sub_rn(n[1], pv1), y2 = sub_rn(n[2], pv2);
            Sya = add_rn(Sya, y0); Syb = add_rn(Syb, y1); Syc = add_rn(Syc, y2);
            Syya = fma_rn(y0, y0, Syya); Syyb = fma_rn(y1, y1, Syyb); Syyc = fma_rn(y2, y2, Syyc);
            Smya = fma_rn(m[0], y0, Smya); Smyb = fma_rn(m[1], y1, Smyb); Smyc = fma_rn(m[2], y2, Smyc);
            Sdma = fma_rn(d[0], m[0], Sdma); Sdmb = fma_rn(d[1], m[1], Sdmb); Sdmc = fma_rn(d[2], m[2], Sdmc);
            Sdna = fma_rn(d[0], n[0], Sdna); Sdnb = fma_rn(d[1], n[1], Sdnb); Sdnc = fma_rn(d[2], n[2], Sdnc);
            Sdda = fma_rn(d[0], d[0], Sdda); Sddb = fma_rn(d[1], d[1], Sddb); Sddc = fma_rn(d[2], d[2], Sddc);
            {
                // patch_optimization.cc:324-343: the rows of a sample are (1, ii, jj) * cs * deriv per channel, so its
                // products are (1, ii, jj)^T (1, ii, jj) * q and (1, ii, jj) * s with q = sum (cs d)^2 and
                // s = sum cs d (m - cs n) over the channels
                const float di = k_sample_offset[k].di, dj = k_sample_offset[k].dj;
                const float g0 = mul_rn(c0, d[0]), g1 = mul_rn(c1, d[1]), g2 = mul_rn(c2, d[2]);
                const float q = fma_rn(g2, g2, fma_rn(g0, g0, mul_rn(g1, g1)));
                const float s = fma_rn(g2, fma_rn(-c2, n[2], m[2]), fma_rn(g0, fma_rn(-c0, n[0], m[0]), mul_rn(g1, fma_rn(-c1, n[1], m[1]))));
                const float qi = mul_rn(di, q), qj = mul_rn(dj, q);
                A1 = add_rn(A1, qi); A2 = add_rn(A2, qj); A3 = fma_rn(di, qi, A3); A4 = fma_rn(dj, qi, A4); A5 = fma_rn(dj, qj, A5);
                B1 = fma_rn(di, s, B1); B2 = fma_rn(dj, s, B2);
            }
        }
    };

    // One pass at the current state (same contract as PatchW::pass).
    // `cand`: NCC per candidate global slot, written by a candidates pass for the lvs_greedy() that follows it.
    __device__ __forceinline__ void pass(bool candidates, bool cs_pending, bool want_ncc, bool want_normal, float* cand, PassOut& po)
    {
        // The object lives in shared memory (k_frontier): what the sample loop reads 25 times per sweep is copied into
        // registers here, everything else is read where it is needed.
        const float* const lut_tab = table();
        const unsigned lane4 = lane_offset();
        const float u0x = this->u0x, u0y = this->u0y, u0z = this->u0z, uax = this->uax, uay = this->uay, uaz = this->uaz;
        const float ubx = this->ubx, uby = this->uby, ubz = this->ubz;
        const float depth = this->depth, dzI = this->dzI, dzJ = this->dzJ;
        const float inv_mm = this->inv_mm;
        const JobParams* const job = this->job;
        float num = 0.f, den = 0.f;
        double D0 = 0.0, D1 = 0.0, D2 = 0.0, D3 = 0.0, D4 = 0.0, D5 = 0.0, E0 = 0.0, E1 = 0.0, E2 = 0.0;
        bool cs_active = cs_pending && st->use_color_scale;
        if (!candidates) pk &= want_ncc ? ~((0xFFu << SH_COL) | (0xFu << SH_DF)) : ~(0xFFu << SH_COL);     // p_col_ok = p_der_ok = 0
        const int count = candidates ? job->n_global : nsel();
        const float pv0 = mx0 * mm, pv1 = mx1 * mm, pv2 = mx2 * mm;      // pivots of the NCC sums (meanX: read after the sweeps)
#pragma unroll 1
        for (int k = 0; k < count; ++k) {
            int slot = k;
            if (candidates) { if (!((avail >> k) & 1u)) continue; }
            else slot = sel(k);
            const ViewParams* V = &views[job->gview[slot]];
            ++n_sets;
            float c0 = 1.f, c1 = 1.f, c2 = 1.f;
            if (!candidates) {
                c0 = k == 0 ? cs[0][0] : (k == 1 ? cs[1][0] : (k == 2 ? cs[2][0] : cs[3][0]));
                c1 = k == 0 ? cs[0][1] : (k == 1 ? cs[1][1] : (k == 2 ? cs[2][1] : cs[3][1]));
                c2 = k == 0 ? cs[0][2] : (k == 1 ? cs[1][2] : (k == 2 ? cs[2][2] : cs[3][2]));
            }
            // ---- view set-up: transform, level choice (patch_sampler.cc:76-91), derivative step (:94-100) ----
            unsigned r = 0u;
            float A0x = 0.f, A0y = 0.f, A0z = 0.f, W0x = 0.f, W0y = 0.f, W0z = 0.f, Wax = 0.f, Way = 0.f, Waz = 0.f, Wbx = 0.f, Wby = 0.f, Wbz = 0.f;
            float Lax = 0.f, Lay = 0.f, Lcx = 0.f, Lcy = 0.f, wm1 = 0.f, hm1 = 0.f, dd = 0.f, step = 0.f;
            int Lpitch = 0;
            const uint4* Lquad = nullptr;
            {
                const float4 wa = __ldg(reinterpret_cast<const float4*>(&V->w2c[0]));
                const float4 wb = __ldg(reinterpret_cast<const float4*>(&V->w2c[4]));
                const float4 wc = __ldg(reinterpret_cast<const float4*>(&V->w2c[8]));
                A0x = wa.x * c0x + wa.y * c0y + wa.z * c0z + wa.w;
                A0y = wb.x * c0x + wb.y * c0y + wb.z * c0z + wb.w;
                A0z = wc.x * c0x + wc.y * c0y + wc.z * c0z + wc.w;
                W0x = wa.x * u0x + wa.y * u0y + wa.z * u0z; W0y = wb.x * u0x + wb.y * u0y + wb.z * u0z; W0z = wc.x * u0x + wc.y * u0y + wc.z * u0z;
                Wax = wa.x * uax + wa.y * uay + wa.z * uaz; Way = wb.x * uax + wb.y * uay + wb.z * uaz; Waz = wc.x * uax + wc.y * uay + wc.z * uaz;
                Wbx = wa.x * ubx + wa.y * uby + wa.z * ubz; Wby = wb.x * ubx + wb.y * uby + wb.z * ubz; Wbz = wc.x * ubx + wc.y * uby + wc.z * ubz;
                const float nz = wc.x * cpx + wc.y * cpy + wc.z * cpz + wc.w;
                const float nfp = nz * __ldg(&V->inv_ax0);
                // mfp <= 0 makes the reference throw std::out_of_range (patch_sampler.cc:78-82); it cannot happen for
                // depth > 0 because the centre ray has positive camera z.  Treated as a failed view here.
                if (mfp > 0.f && !(nfp <= 0.f)) {
                    const int l = level_of(V, nfp, inv_mfp);
                    const float4 kk = __ldg(reinterpret_cast<const float4*>(&V->lv[l].ax));
                    const int4 g = __ldg(reinterpret_cast<const int4*>(&V->lv[l].w));
                    Lax = kk.x; Lay = kk.y; Lcx = kk.z; Lcy = kk.w; wm1 = (float)(g.x - 1); hm1 = (float)(g.y - 1); Lpitch = g.z;
                    Lquad = reinterpret_cast<const uint4*>(__ldg(reinterpret_cast<const unsigned long long*>(&V->lv[l].quad)));
                    // projections of patchPoints[12] and patchPoints[12] + masterViewDirs[12]
                    const float inv0 = rsqrt_fast(u0x * u0x + u0y * u0y + u0z * u0z);
                    const float sa = depth * inv0, sb = (depth + 1.f) * inv0;
                    const float hz1 = A0z + sa * W0z, hz2 = A0z + sb * W0z;
                    const float i1 = rcp_fast(hz1), i2 = rcp_fast(hz2);
                    const float ddx = (Lax * (A0x + sb * W0x) + Lcx * hz2) * i2 - (Lax * (A0x + sa * W0x) + Lcx * hz1) * i1;
                    const float ddy = (Lay * (A0y + sb * W0y) + Lcy * hz2) * i2 - (Lay * (A0y + sa * W0y) + Lcy * hz1) * i1;
                    const float dd2 = ddx * ddx + ddy * ddy;
                    dd = dd2 * rsqrt_fast(dd2);            // |.|; NaN for dd2 == 0, which fails `d > 0` like the reference's 0
                    step = rcp_fast(dd);
                    r = dd > 0.f ? 3u : 1u;
                }
            }
            const bool need_ncc = candidates || want_ncc;
            const bool cs_view = !candidates && cs_active;         // a colour-scale update is due for this view (if it samples)
            float nccv = -1.f;
            // ---- sweeps over the 25 samples ----
#pragma unroll 1
            for (int rep = 0; rep < 2 && r != 0u; ++rep) {
                const bool second = rep == 1;
                if (second && !(cs_view && want_normal && (r & 2u))) break;
                // Gauss-Newton terms of this view: from this sweep unless the colour scale is updated AND the normal step
                // follows (then the second sweep forms them with the new scale); the normal equations need the products
                // with the scale of the sweep, so they are formed only where it is known
                const bool gn = !candidates && (r & 2u) && (second || !(cs_view && want_normal));
                const bool nrm = gn && want_normal;
                Sweep sw;
                sw.lut = lut_tab; sw.lane4 = lane4; sw.inv_mm = inv_mm;
                sw.u0x = u0x; sw.u0y = u0y; sw.u0z = u0z; sw.uax = uax; sw.uay = uay; sw.uaz = uaz; sw.ubx = ubx; sw.uby = uby; sw.ubz = ubz;
                sw.mt = mt_tab();
                sw.depth = depth; sw.dzI = dzI; sw.dzJ = dzJ;
                sw.A0x = A0x; sw.A0y = A0y; sw.A0z = A0z; sw.W0x = W0x; sw.W0y = W0y; sw.W0z = W0z;
                sw.Wax = Wax; sw.Way = Way; sw.Waz = Waz; sw.Wbx = Wbx; sw.Wby = Wby; sw.Wbz = Wbz;
                sw.Lax = Lax; sw.Lay = Lay; sw.Lcx = Lcx; sw.Lcy = Lcy; sw.wm1 = wm1; sw.hm1 = hm1; sw.step = step; sw.dd = dd;
                sw.quad = Lquad; sw.qpitch = (unsigned)Lpitch;
                sw.pv0 = pv0; sw.pv1 = pv1; sw.pv2 = pv2; sw.c0 = c0; sw.c1 = c1; sw.c2 = c2;
                sw.clear();
                // The sample loop is software-pipelined two samples deep.  Two slots take turns: as soon as sample k has
                // been processed, sample k+2 is staged (geometry, quad and master loads) into the slot k was read from, so
                // its loads have all of sample k+1 to arrive.  The rotation is in the code - the loop is unrolled by two -
                // and no staged value is copied.  Samples 0..21 run in the loop and 22..24 after it, where only sample 24
                // is still staged: nothing past the last sample is ever staged.  All 25 samples run, without a branch;
                // `ok` collects their validity, and a view with an invalid sample fails (its sums are never read).
                Staged sa, sb;
                bool ok = sw.stage(0, sa);
                ok &= sw.stage(1, sb);
#pragma unroll 1
                for (int j = 0; j < NS - 3; j += 2) {
                    sw.sample(j, sa);
                    ok &= sw.stage(j + 2, sa);
                    sw.sample(j + 1, sb);
                    ok &= sw.stage(j + 3, sb);
                }
                sw.sample(NS - 3, sa);
                ok &= sw.stage(NS - 1, sa);
                sw.sample(NS - 2, sb);
                sw.sample(NS - 1, sa);
                const float Sya = sw.Sya, Syb = sw.Syb, Syc = sw.Syc, Syya = sw.Syya, Syyb = sw.Syyb, Syyc = sw.Syyc;
                const float Smya = sw.Smya, Smyb = sw.Smyb, Smyc = sw.Smyc, Sdma = sw.Sdma, Sdmb = sw.Sdmb, Sdmc = sw.Sdmc;
                const float Sdna = sw.Sdna, Sdnb = sw.Sdnb, Sdnc = sw.Sdnc, Sdda = sw.Sdda, Sddb = sw.Sddb, Sddc = sw.Sddc;
                const float A1 = sw.A1, A2 = sw.A2, A3 = sw.A3, A4 = sw.A4, A5 = sw.A5, B1 = sw.B1, B2 = sw.B2;
                if (!ok) { r = 0u; break; }
                if (!second && need_ncc) {                // getFastNCC (patch_sampler.cc:143-162)
                    const float inv_n = 1.f / (float)NS;
                    const float sqrDevY = (Syya - Sya * Sya * inv_n) + (Syyb - Syb * Syb * inv_n) + (Syyc - Syc * Syc * inv_n);
                    const float Sen = (Smya - mx0 * Sya) + (Smyb - mx1 * Syb) + (Smyc - mx2 * Syc);   // sum((m - meanX) y)
                    const float p = sqrDevX * sqrDevY;      // devXY / sqrt(p), -1 when sqrt(p) is not > 0
                    nccv = p > 0.f ? Sen * rsqrt_fast(p) : -1.f;
                }
                if (!second && cs_view) {                 // computeColorScale for this view (patch_optimization.cc:88-110)
                    // sum(m n) = sum(m y) + p sum(m), sum(m) = NS meanX;  sum(n n) = sum(y^2) + p (2 sum(y) + NS p)
                    const float Mna = Smya + pv0 * ((float)NS * mx0), Mnb = Smyb + pv1 * ((float)NS * mx1), Mnc = Smyc + pv2 * ((float)NS * mx2);
                    const float Nna = Syya + pv0 * (2.f * Sya + (float)NS * pv0), Nnb = Syyb + pv1 * (2.f * Syb + (float)NS * pv1);
                    const float Nnc = Syyc + pv2 * (2.f * Syc + (float)NS * pv2);
                    float cc[3] = {c0, c1, c2};
                    const float ab[3] = {Mna - c0 * Nna, Mnb - c1 * Nnb, Mnc - c2 * Nnc};
                    const float aa[3] = {Nna, Nnb, Nnc};
                    colour_scale_step(cc, ab, aa);
                    c0 = cc[0]; c1 = cc[1]; c2 = cc[2];
#pragma unroll
                    for (int i = 0; i < MAX_LOCAL; ++i) if (i == k) { cs[i][0] = c0; cs[i][1] = c1; cs[i][2] = c2; }
                }
                if (gn) {
                    // patch_optimization.cc:283-288 with the scale of this state (updated above when it was due):
                    // sum(cs d (m - cs n)) and sum((cs d)^2) per channel
                    const float vn = c0 * (Sdma - c0 * Sdna) + c1 * (Sdmb - c1 * Sdnb) + c2 * (Sdmc - c2 * Sdnc);
                    const float vd = c0 * c0 * Sdda + c1 * c1 * Sddb + c2 * c2 * Sddc;
                    num += vn; den += vd;
                    if (nrm) {
                        // a view's <= 75 products are summed in fp32, the views in fp64; the reference sums all 300 fp32 products
                        // in fp64 (patch_optimization.cc:336-342) - far below what the Gauss-Newton fixed point resolves
                        D0 += (double)vd; D1 += (double)A1; D2 += (double)A2; D3 += (double)A3; D4 += (double)A4; D5 += (double)A5;
                        E0 += (double)vn; E1 += (double)B1; E2 += (double)B2;
                    }
                }
            }
            if (!candidates) {
                if (r & 1u) pk |= 1u << (SH_COL + k);
                if (r & 2u) pk |= 1u << (SH_DER + k);
                // computeColorScale: a failed view ends the whole update (`return`, not `continue`, patch_optimization.cc:92-93)
                if (cs_active && !(r & 1u)) cs_active = false;
                if (want_ncc) {
                    const float v = (r & 1u) ? nccv : -1.f;
                    if (fabsf(v - get4(ncc, k)) > st->min_refine_diff) pk |= 1u << (SH_DF + k);
                    set4(ncc, k, v);
                }
            } else {
                const float v = (r & 1u) ? nccv : -1.f;
                if (v < st->min_ncc) avail &= ~(1u << k);
                else cand[k] = v;
            }
        }
        if (candidates) return;
        po.num = num; po.den = den;
        put(F_HAS_NORMAL, want_normal);
        put(F_HAS_NCC, want_ncc);
        if (want_normal) {
            // matrix_tools.h:392-398,460-475.  Written out here and in PatchW::pass: as a shared function it changes how nvcc
            // contracts the unpinned Gauss-Newton sums above (vn), and with them the last bits of dz.
            const double m[9] = {D0, D1, D2, D1, D3, D4, D2, D4, D5};
            const double det = m[0] * m[4] * m[8] + m[1] * m[5] * m[6] + m[2] * m[3] * m[7]
                             - m[2] * m[4] * m[6] - m[1] * m[3] * m[8] - m[0] * m[5] * m[7];
            put(F_SINGULAR, det == 0.0);
            double inv[9];
            inv[0] = m[4] * m[8] - m[5] * m[7];
            inv[1] = m[2] * m[7] - m[1] * m[8];
            inv[2] = m[1] * m[5] - m[2] * m[4];
            inv[3] = m[5] * m[6] - m[3] * m[8];
            inv[4] = m[0] * m[8] - m[2] * m[6];
            inv[5] = m[2] * m[3] - m[0] * m[5];
            inv[6] = m[3] * m[7] - m[4] * m[6];
            inv[7] = m[1] * m[6] - m[0] * m[7];
            inv[8] = m[0] * m[4] - m[1] * m[3];
#pragma unroll
            for (int q = 0; q < 9; ++q) inv[q] /= det;
            po.nX0 = (float)(inv[0] * E0 + inv[1] * E1 + inv[2] * E2);
            po.nX1 = (float)(inv[3] * E0 + inv[4] * E1 + inv[5] * E2);
            po.nX2 = (float)(inv[6] * E0 + inv[7] * E1 + inv[8] * E2);
        }
    }

    // ---- sorted insert / erase on the selected set (std::set semantics) ----
    __device__ __forceinline__ void sel_erase_mask(unsigned mask)       // bit k: remove element k
    {
        const int n = nsel();
        int cnt = 0;
        unsigned packed = 0xFFFFFFFFu;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) {
            if (k < n && !((mask >> k) & 1u)) {
                // element k moves to position cnt (cnt <= k)
                const unsigned s8 = (selp >> (8 * k)) & 0xFFu;
                const float a = cs[k][0], b = cs[k][1], c = cs[k][2], v = ncc[k];
                packed = (packed & ~(0xFFu << (8 * cnt))) | (s8 << (8 * cnt));
#pragma unroll
                for (int q = 0; q < MAX_LOCAL; ++q) if (q == cnt) { cs[q][0] = a; cs[q][1] = b; cs[q][2] = c; ncc[q] = v; }
                ++cnt;
            }
        }
        selp = packed;
        set_nsel(cnt);
    }
    __device__ __forceinline__ void sel_insert(int slot, float cs_init)
    {
        const int n = nsel();
        int pos = 0;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) if (k < n && sel(k) < slot) ++pos;
#pragma unroll
        for (int q = MAX_LOCAL - 1; q > 0; --q)
            if (q > pos && q <= n) { cs[q][0] = cs[q - 1][0]; cs[q][1] = cs[q - 1][1]; cs[q][2] = cs[q - 1][2]; ncc[q] = ncc[q - 1]; }
#pragma unroll
        for (int q = 0; q < MAX_LOCAL; ++q) if (q == pos) { cs[q][0] = cs[q][1] = cs[q][2] = cs_init; ncc[q] = 0.f; }
        // bytes below `pos` stay, the byte at `pos` becomes the new slot, the bytes above move up by one
        const unsigned low = pos == 0 ? 0u : (selp & (0xFFFFFFFFu >> (32 - 8 * pos)));
        const unsigned high = pos >= 3 ? 0u : ((selp >> (8 * pos)) << (8 * (pos + 1)));
        selp = low | ((unsigned)slot << (8 * pos)) | high;
        set_nsel(n + 1);
    }

    // Second half of LocalViewSelection::performVS (local_view_selection.cc:86-147)
    __device__ __forceinline__ void lvs_greedy(const float* cand)
    {
        const unsigned N = st->nr_recon_neighbors;
        const float cs_init = 1.f / mm;
        float rdx = cpx - c0x, rdy = cpy - c0y, rdz = cpz - c0z;
        {
            const float nn = sqrtf(rdx * rdx + rdy * rdy + rdz * rdz);
            rdx /= nn; rdy /= nn; rdz /= nn;
        }
        const int G = job->n_global;
        bool found = true;
        while ((unsigned)nsel() < N && found) {
            found = false;
            float maxScore = 0.f;
            int maxView = 0;
#pragma unroll 1
            for (int c = 0; c < G; ++c) {
                if (!((avail >> c) & 1u)) continue;
                float vdx, vdy, vdz, epx, epy, epz, nfp;
                view_geometry(&views[job->gview[c]], cpx, cpy, cpz, rdx, rdy, rdz, vdx, vdy, vdz, epx, epy, epz, nfp);
                float score = cand[c];
                if (mfp / nfp < 0.5f) score *= 0.01f;
                float dp = clamp1(rdx * vdx + rdy * vdy + rdz * vdz);
                score *= plx_weight(deg_acos(dp));
                const int ns = nsel();
#pragma unroll 1
                for (int k = 0; k < ns; ++k) {
                    float sx, sy, sz, ex, ey, ez, sfp;
                    view_geometry(&views[job->gview[sel(k)]], cpx, cpy, cpz, rdx, rdy, rdz, sx, sy, sz, ex, ey, ez, sfp);
                    lvs_weigh(score, vdx, vdy, vdz, epx, epy, epz, sx, sy, sz, ex, ey, ez, st->min_parallax);
                }
                if (score > maxScore) { maxScore = score; maxView = c; found = true; }     // local_view_selection.cc:133-137
            }
            if (found) {
                sel_insert(maxView, cs_init);
                avail &= ~(1u << maxView);
            }
        }
        if ((unsigned)nsel() == N) pk |= F_LVS_OK;
    }

    // PatchOptimization ctor (patch_optimization.cc:21-78) incl. LocalViewSelection ctor (local_view_selection.cc:19-54)
    __device__ __forceinline__ void begin(const JobParams* j, const PatchIn& in)
    {
        job = j;
        xy = ((unsigned)in.x & 0xFFFFu) | ((unsigned)in.y << 16);
        reset(in);
        u0x = u0y = u0z = uax = uay = uaz = ubx = uby = ubz = c0x = c0y = c0z = 0.f;
        init_sampler(in.x, in.y);
        selp = in.slots;                                 // propagated ids arrive ascending, 0xFF padded
        int n = 0;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) {
            if (sel(k) != 0xFF) n = k + 1;
            cs[k][0] = cs[k][1] = cs[k][2] = 0.f; ncc[k] = 0.f;
        }
        set_nsel(n);
        if (!is(F_REF_OK)) { pk &= ~F_OPTI; return; }
        const unsigned N = st->nr_recon_neighbors;
        if ((unsigned)n == N) pk |= F_LVS_OK;
        else if ((unsigned)n > N) {
            n = 0;
            set_nsel(0);
            selp = 0xFFFFFFFFu;
        }
        avail = job->n_global >= 32 ? FULL : ((1u << job->n_global) - 1u);
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) if (k < n) avail &= ~(1u << sel(k));
        const float ci = 1.f / mm;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) { cs[k][0] = cs[k][1] = cs[k][2] = ci; }
        set_stage(is(F_LVS_OK) ? CTOR : LVS_CTOR);
    }

    __device__ __forceinline__ unsigned low_ncc_mask() const
    {
        const int n = nsel();
        unsigned m = 0u;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k)
            if (k < n && ncc[k] < st->accept_ncc) m |= 1u << k;
        return m;
    }

    __device__ __forceinline__ bool step() { return auto_step(*this); }

    // PatchOptimization::computeConfidence (patch_optimization.cc:114-142) + getPatchNormal (patch_sampler.cc:243-256)
    __device__ __forceinline__ void finish(PatchOut& out)
    {
        finish_state(out);
        const int n = nsel();
        out.slots = n >= 4 ? selp : (selp | (0xFFFFFFFFu << (8 * n)));
        if (!is(F_CONVERGED)) return;
        float mean = 0.f;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) if (k < n) mean += ncc[k];
        mean /= (float)n;
        // patchPoints[14] - patchPoints[10] and patchPoints[2] - patchPoints[22]
        float px[4], py[4], pz[4];
        const float di_[4] = {2.f, -2.f, 0.f, 0.f}, dj_[4] = {0.f, 0.f, -2.f, 2.f};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float ux, uy, uz, inv;
            sample_ray(di_[q], dj_[q], ux, uy, uz, inv);
            const float s1 = (depth + di_[q] * dzI + dj_[q] * dzJ) * inv;
            px[q] = c0x + s1 * ux; py[q] = c0y + s1 * uy; pz[q] = c0z + s1 * uz;
        }
        const float ax_ = px[0] - px[1], ay_ = py[0] - py[1], az_ = pz[0] - pz[1];
        const float bx_ = px[2] - px[3], by_ = py[2] - py[3], bz_ = pz[2] - pz[3];
        confidence(out, ax_, ay_, az_, bx_, by_, bz_, crx, cry, crz, mean, st->accept_ncc);
    }
};

#if !defined(B200MVS_HOST_EMU)
// PatchT objects sit side by side in shared memory (k_frontier).  With 8-byte members the stride cannot be an odd number of
// words; 2 mod 4 words keeps the conflicts of a warp's accesses to one member at 2-way (these are the once-per-sweep
// accesses, not the table look-ups of the sample loop).
// How many fit beside the table and the master texels is checked with the kernels (b200mvs.cu, OPT_SMEM_BYTES).
static_assert(sizeof(PatchT) % 16 == 8, "PatchT stride in shared memory must be 8 mod 16 bytes");
#endif

__device__ __forceinline__ void bind_thread(PatchT& p, const DevSettings* st, const ViewParams* views, const float* lut_rep, int tid)
{
    p.st = st; p.views = views;
#if defined(B200MVS_HOST_EMU)
    p.lut_tab = lut_rep; p.lane4 = 4u * (unsigned)(tid & (LUT_REP - 1));
#else
    (void)lut_rep; (void)tid;      // the table is the start of the dynamic shared memory, the lane comes from threadIdx
#endif
    p.pk = (unsigned)PatchT::DONE << PatchT::SH_STAGE;
    p.n_sets = 0u;
}

} // namespace b200mvs
