// Device-side patch optimisation, LATENCY variant: one WARP per patch, lane k < 25 owns sample k of the 5x5 patch.
//
// Same function as PatchT (patch_thread.cuh) - one mvs::PatchOptimization of the reference
// (libs/dmrecon/patch_optimization.cc:21-364 with PatchSampler patch_sampler.cc:19-393, LocalViewSelection
// local_view_selection.cc:19-160 and mvs_tools.cc:98-199) - organised for SMALL frontier rounds (the tail of the region
// growing, the confidence-ordered modes), where the number of queue entries is far below the number of lanes on the chip
// and what counts is the latency of one optimisation: the 25 samples of a sample set are drawn by 25 lanes at once and
// reduced with warp-shuffle butterflies; the spare lane 25 projects patchPoints[12] + masterViewDirs[12] so that the
// derivative step (patch_sampler.cc:94-100) costs no extra instructions.
//   * ONE fused sample set per (state, view): computeNeighColorSamples and fastColAndDeriv use identical bilinear formulas
//     (mvs_tools.cc:119-128 vs :188-197);
//   * one PASS per patch state (depth, dzI, dzJ) with a single pass() call site, driven by the flat begin / step / finish
//     loop of the kernels (a warp that finishes a patch fetches the next one at once);
//   * small per-view arrays (selected slots, colour scales, NCCs) live one element per lane and are read with shuffles;
//     the sums of the 3x3 normal equations (patch_optimization.cc:326-343) are formed per lane in fp32 (<= 12 products) and
//     across the lanes in fp64, then solved in fp64 inside the pass;
//   * the four bilinear taps of a sample come from ONE 16-byte load of a quad texel, sRGB code values are linearised through
//     the lane-replicated table (patch_opt.cuh).
#pragma once
#include "patch_opt.cuh"

namespace b200mvs {

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL, v, o));
    return v;
}

// Batched butterflies: reducing K values together halves the number of live values at each of the first log2(K)
// steps, so 4 sums cost 10 shuffles instead of 20 (2 sums: 7 instead of 10).  Every lane receives all totals, and all
// lanes receive bitwise identical totals (each total is formed in exactly one lane group and then broadcast).
__device__ __forceinline__ void warp_sum4(int lane, float& a, float& b, float& c, float& d)
{
    const bool h16 = lane & 16, h8 = lane & 8;
    float k0 = h16 ? c : a, k1 = h16 ? d : b;
    const float s0 = h16 ? a : c, s1 = h16 ? b : d;
    k0 += __shfl_xor_sync(FULL, s0, 16);
    k1 += __shfl_xor_sync(FULL, s1, 16);
    float k = h8 ? k1 : k0;
    const float s = h8 ? k0 : k1;
    k += __shfl_xor_sync(FULL, s, 8);
    k += __shfl_xor_sync(FULL, k, 4);
    k += __shfl_xor_sync(FULL, k, 2);
    k += __shfl_xor_sync(FULL, k, 1);
    a = __shfl_sync(FULL, k, 0); b = __shfl_sync(FULL, k, 8); c = __shfl_sync(FULL, k, 16); d = __shfl_sync(FULL, k, 24);
}
__device__ __forceinline__ void warp_sum2(int lane, float& a, float& b)
{
    const bool h16 = lane & 16;
    float k = h16 ? b : a;
    const float s = h16 ? a : b;
    k += __shfl_xor_sync(FULL, s, 16);
    k += __shfl_xor_sync(FULL, k, 8);
    k += __shfl_xor_sync(FULL, k, 4);
    k += __shfl_xor_sync(FULL, k, 2);
    k += __shfl_xor_sync(FULL, k, 1);
    a = __shfl_sync(FULL, k, 0); b = __shfl_sync(FULL, k, 16);
}

struct PatchW : PatchState {       // the PatchState is warp-uniform
    // ---- constants of the patch ----
    const DevSettings* st;
    const JobParams* job;
    const ViewParams* views;
    const ViewParams* rv;
    const float* lut_tab;      // lane-replicated srgb2lin table in shared memory (lut_k)
    unsigned lane4;            // 4 * (lane of this thread)
    int lane;
    bool act;                  // lane < 25
    float fi, fj;              // sample offsets (patch_optimization.cc:56-64)
    // ---- per-lane sample state ----
    float rx, ry, rz;          // masterViewDirs[k]
    float px, py, pz;          // patchPoints[k]
    float m0, m1, m2;          // masterColorSamples[k] (normalised)
    float e0, e1, e2;          // masterColorSamples[k] - meanX
    // ---- warp-uniform state ----
    float crx, cry, crz;       // masterViewDirs[12]
    float cpx, cpy, cpz;       // patchPoints[12]
    float mfp, inv_mfp;        // footPrintScaled(patchPoints[12]) and its reciprocal
    float mm, sqrDevX;         // masterMeanCol, sqrDevX
    // ---- lane-distributed small arrays: lane k (< nsel) holds element k ----
    int sel_l;                 // selected global slot (ascending over lanes)
    float cs0_l, cs1_l, cs2_l; // colorScale of selected view k
    float ncc_l;               // NCC of selected view k at the state of the last pass
    float cand_ncc_l;          // NCC of candidate global slot `lane` (local view selection)

    // single_view.h:188-195 (K has the sparsity of camera.cc:125-144).  x = (K cp).x / cp.z - 0.5 is evaluated with one
    // correctly rounded reciprocal shared by x and y (<= 1 ulp from the reference's two divisions; measured effect on
    // parity in tests/test_gpu_parity.py).
    __device__ __forceinline__ void project(const float (&w)[12], const LevelParams& L, float X, float Y, float Z,
                                            float& x, float& y) const
    {
        const float c0 = w[0] * X + w[1] * Y + w[2] * Z + w[3];
        const float c1 = w[4] * X + w[5] * Y + w[6] * Z + w[7];
        const float c2 = w[8] * X + w[9] * Y + w[10] * Z + w[11];
        const float ic2 = rcp_fast(c2);
        x = (L.ax * c0 + L.cx * c2) * ic2 - 0.5f;
        y = (L.ay * c1 + L.cy * c2) * ic2 - 0.5f;
    }

    // patch_sampler.cc:274-295 (+ the centre point / master footprint used by every sample set)
    __device__ __forceinline__ void compute_points()
    {
        const float t = depth + fi * dzI + fj * dzJ;
        const bool bad = act && (t <= 0.f);
        if (__any_sync(FULL, bad)) pk &= ~F_REF_OK;
        px = __ldg(&rv->campos[0]) + t * rx;
        py = __ldg(&rv->campos[1]) + t * ry;
        pz = __ldg(&rv->campos[2]) + t * rz;
        cpx = __shfl_sync(FULL, px, CENTER);
        cpy = __shfl_sync(FULL, py, CENTER);
        cpz = __shfl_sync(FULL, pz, CENTER);
        const float z = __ldg(&rv->w2c[8]) * cpx + __ldg(&rv->w2c[9]) * cpy + __ldg(&rv->w2c[10]) * cpz + __ldg(&rv->w2c[11]);
        mfp = z * job->ki0;     // single_view.h:160-164
        inv_mfp = rcp_fast(mfp);
    }

    // PatchSampler ctor (patch_sampler.cc:19-62) + computeMasterSamples (:298-345)
    __device__ __forceinline__ void init_sampler(int x, int y)
    {
        act = lane < NS;
        const int di = act ? (lane % 5) - 2 : 0, dj = act ? (lane / 5) - 2 : 0;
        fi = (float)di; fj = (float)dj;
        pk &= ~F_REF_OK; mm = 0.f; sqrDevX = 0.f;
        rx = ry = rz = px = py = pz = 0.f; m0 = m1 = m2 = e0 = e1 = e2 = 0.f;
        crx = cry = crz = cpx = cpy = cpz = mfp = inv_mfp = 0.f;
        if (x - 2 < 0 || y - 2 < 0 || x + 2 > job->W - 1 || y + 2 > job->H - 1) return;
        // viewRayScaled (single_view.cc:99-106, depthmap.cc:149-156)
        {
            const float fx = (float)(x + di) + 0.5f, fy = (float)(y + dj) + 0.5f;
            float vx = job->ki0 * fx + job->ki2;
            float vy = job->ki4 * fy + job->ki5;
            float vz = 1.0f;
            const float nrm = sqrtf(vx * vx + vy * vy + vz * vz);
            vx /= nrm; vy /= nrm; vz /= nrm;
            rx = __ldg(&rv->rot[0]) * vx + __ldg(&rv->rot[3]) * vy + __ldg(&rv->rot[6]) * vz;
            ry = __ldg(&rv->rot[1]) * vx + __ldg(&rv->rot[4]) * vy + __ldg(&rv->rot[7]) * vz;
            rz = __ldg(&rv->rot[2]) * vx + __ldg(&rv->rot[5]) * vy + __ldg(&rv->rot[8]) * vz;
        }
        crx = __shfl_sync(FULL, rx, CENTER);
        cry = __shfl_sync(FULL, ry, CENTER);
        crz = __shfl_sync(FULL, rz, CENTER);
        pk |= F_REF_OK;
        // master colours
        const unsigned t = reinterpret_cast<const unsigned*>(job->ref_img)[(size_t)(y + dj) * job->ref_pitch + (x + di)];
        m0 = act ? lut_k<0>(lut_tab, lane4, t) : 0.f; m1 = act ? lut_k<1>(lut_tab, lane4, t) : 0.f; m2 = act ? lut_k<2>(lut_tab, lane4, t) : 0.f;
        mm = warp_sum(m0 + m1 + m2) / (3.f * NS);
        if (mm < 0.01f || mm > 0.99f) { pk &= ~F_REF_OK; return; }
        m0 /= mm; m1 /= mm; m2 /= mm;
        const float mx0 = warp_sum(m0) / (float)NS, mx1 = warp_sum(m1) / (float)NS, mx2 = warp_sum(m2) / (float)NS;
        e0 = act ? m0 - mx0 : 0.f; e1 = act ? m1 - mx1 : 0.f; e2 = act ? m2 - mx2 : 0.f;
        sqrDevX = warp_sum(e0 * e0 + e1 * e1 + e2 * e2);
        compute_points();
    }

    // One fused sample set in view V at the current state: fastColAndDeriv (patch_sampler.cc:65-133 +
    // mvs_tools.cc:98-145) and computeNeighColorSamples (patch_sampler.cc:348-393 + mvs_tools.cc:169-199).
    // Returns bit0 = colour path succeeded, bit1 = derivative path succeeded.
    __device__ __forceinline__ unsigned sample(const ViewParams* V, float (&n)[3], float (&d)[3])
    {
        if (lane == 0) ++n_sets;
        n[0] = n[1] = n[2] = 0.f; d[0] = d[1] = d[2] = 0.f;
        float w[12];
        {
            const float4 a = __ldg(reinterpret_cast<const float4*>(&V->w2c[0]));
            const float4 b = __ldg(reinterpret_cast<const float4*>(&V->w2c[4]));
            const float4 c = __ldg(reinterpret_cast<const float4*>(&V->w2c[8]));
            w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w; w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
            w[8] = c.x; w[9] = c.y; w[10] = c.z; w[11] = c.w;
        }
        const float nz = w[8] * cpx + w[9] * cpy + w[10] * cpz + w[11];
        const float nfp = nz * __ldg(&V->inv_ax0);
        // mfp <= 0 makes the reference throw std::out_of_range (patch_sampler.cc:78-82); it cannot happen for
        // depth > 0 because the centre ray has positive camera z.  Treated as a failed view here.
        if (!(mfp > 0.f) || nfp <= 0.f) return 0u;
        const int l = level_of(V, nfp, inv_mfp);
        LevelParams L;
        {
            const float4 k = __ldg(reinterpret_cast<const float4*>(&V->lv[l].ax));
            const int4 g = __ldg(reinterpret_cast<const int4*>(&V->lv[l].w));
            L.ax = k.x; L.ay = k.y; L.cx = k.z; L.cy = k.w; L.w = g.x; L.h = g.y; L.pitch = g.z;
            L.quad = reinterpret_cast<const uint4*>(__ldg(reinterpret_cast<const unsigned long long*>(&V->lv[l].quad)));
        }
        // every lane projects its own patch point; the spare lane 25 projects patchPoints[12] + masterViewDirs[12]
        // so that the derivative step (patch_sampler.cc:94-100) costs no extra instructions
        const bool aux = lane == NS;
        float qx, qy;
        project(w, L, aux ? cpx + crx : px, aux ? cpy + cry : py, aux ? cpz + crz : pz, qx, qy);
        const float ddx = __shfl_sync(FULL, qx, NS) - __shfl_sync(FULL, qx, CENTER);
        const float ddy = __shfl_sync(FULL, qy, NS) - __shfl_sync(FULL, qy, CENTER);
        const float dd2 = ddx * ddx + ddy * ddy;
        const float dd = dd2 * rsqrt_fast(dd2);        // |.|; NaN for dd2 == 0, which fails `d > 0` like the reference's 0
        const bool dok = dd > 0.f;
        const float step = rcp_fast(dd);
        const bool inb = qx > 0.f && qx < (float)(L.w - 1) && qy > 0.f && qy < (float)(L.h - 1);
        if (!__all_sync(FULL, inb || !act)) return 0u;
        if (act) {
            float gx = 0.f, gy = 0.f;
            if (dok) {
                float tx, ty;
                project(w, L, px + rx * step, py + ry * step, pz + rz * step, tx, ty);
                gx = tx - qx; gy = ty - qy;
            }
            const int left = (int)floorf(qx), top = (int)floorf(qy);
            const float fx = qx - (float)left, fy = qy - (float)top;
            const uint4 Q = __ldg(L.quad + (size_t)top * L.pitch + left);
            const float a[3] = {lut_k<0>(lut_tab, lane4, Q.x), lut_k<1>(lut_tab, lane4, Q.x), lut_k<2>(lut_tab, lane4, Q.x)};
            const float b[3] = {lut_k<0>(lut_tab, lane4, Q.y), lut_k<1>(lut_tab, lane4, Q.y), lut_k<2>(lut_tab, lane4, Q.y)};
            const float c[3] = {lut_k<0>(lut_tab, lane4, Q.z), lut_k<1>(lut_tab, lane4, Q.z), lut_k<2>(lut_tab, lane4, Q.z)};
            const float e[3] = {lut_k<0>(lut_tab, lane4, Q.w), lut_k<1>(lut_tab, lane4, Q.w), lut_k<2>(lut_tab, lane4, Q.w)};
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                const float x0 = (1.f - fx) * a[ch] + fx * b[ch];
                const float x3 = (1.f - fx) * c[ch] + fx * e[ch];
                n[ch] = (1.f - fy) * x0 + fy * x3;
                const float der = gx * (b[ch] - a[ch]) + gy * (c[ch] - a[ch]) + (gy * fx + gx * fy) * (a[ch] - b[ch] - c[ch] + e[ch]);
                d[ch] = dok ? der * dd : 0.f;        // deriv /= stepSize with stepSize = 1 / d (patch_sampler.cc:100,129-130)
            }
        }
        return dok ? 3u : 1u;
    }

    // getFastNCC on given colour samples (patch_sampler.cc:143-162)
    __device__ __forceinline__ float ncc_of(const float (&n)[3]) const
    {
        const float inv_n = 1.f / (float)NS;
        float my0 = n[0], my1 = n[1], my2 = n[2], pad = 0.f;
        warp_sum4(lane, my0, my1, my2, pad);
        my0 *= inv_n; my1 *= inv_n; my2 *= inv_n;
        const float y0 = act ? n[0] - my0 : 0.f, y1 = act ? n[1] - my1 : 0.f, y2 = act ? n[2] - my2 : 0.f;
        float sqrDevY = y0 * y0 + y1 * y1 + y2 * y2;
        float devXY = e0 * y0 + e1 * y1 + e2 * y2;
        warp_sum2(lane, sqrDevY, devXY);
        const float p = sqrDevX * sqrDevY;              // devXY / sqrt(p), -1 when sqrt(p) is not > 0
        return p > 0.f ? devXY * rsqrt_fast(p) : -1.f;
    }

    // One pass at the current state (see the header comment).
    //   candidates : false -> over the selected views; true -> over the AVAILABLE global views, only their NCC is
    //                computed (first half of LocalViewSelection::performVS, local_view_selection.cc:73-85)
    //   cs_pending : a computeColorScale() is due at this state (patch_optimization.cc:77,198,230)
    //   want_ncc   : the NCCs of this state are read by the reference (getFastNCC, patch_optimization.cc:192,213,126)
    //   want_normal: the next Gauss-Newton step is optimizeDepthAndNormal (else optimizeDepthOnly)
    // This is the only place a sample set is drawn, so its code exists once in the kernel.  The candidates' NCCs stay one
    // per lane (cand_ncc_l), so `cand` is not used.
    __device__ __forceinline__ void pass(bool candidates, bool cs_pending, bool want_ncc, bool want_normal, float*, PassOut& po)
    {
        float num = 0.f, den = 0.f;
        float A0 = 0.f, A1 = 0.f, A2 = 0.f, A3 = 0.f, A4 = 0.f, A5 = 0.f, B0 = 0.f, B1 = 0.f, B2 = 0.f;
        bool cs_active = cs_pending && st->use_color_scale;
        bool df_l = false;         // |NCC - previous NCC| > minRefineDiff of selected view `lane` (DF bits)
        unsigned bits = 0u;        // COL / DER bits of this pass, merged into pk at its end
        const int count = candidates ? job->n_global : nsel();
        for (int k = 0; k < count; ++k) {
            int slot = k;
            if (candidates) { if (!((avail >> k) & 1u)) continue; }
            else slot = __shfl_sync(FULL, sel_l, k);
            float n[3], d[3];
            const unsigned r = sample(&views[job->gview[slot]], n, d);
            if (candidates) {
                const float v = (r & 1u) ? ncc_of(n) : -1.f;
                if (v < st->min_ncc) avail &= ~(1u << k);
                else if (lane == k) cand_ncc_l = v;
                continue;
            }
            if (r & 1u) bits |= 1u << (SH_COL + k);
            if (r & 2u) bits |= 1u << (SH_DER + k);
            if (want_ncc) {
                const float v = (r & 1u) ? ncc_of(n) : -1.f;
                if (lane == k) { df_l = fabsf(v - ncc_l) > st->min_refine_diff; ncc_l = v; }
            }
            float c0 = __shfl_sync(FULL, cs0_l, k), c1 = __shfl_sync(FULL, cs1_l, k), c2 = __shfl_sync(FULL, cs2_l, k);
            // computeColorScale for this view (patch_optimization.cc:88-110); a failed view ends the whole
            // update (`return`, not `continue`, :92-93)
            if (cs_active) {
                if (!(r & 1u)) cs_active = false;
                else {
                    float cc[3] = {c0, c1, c2};
                    float ab[3] = {(m0 - n[0] * c0) * n[0], (m1 - n[1] * c1) * n[1], (m2 - n[2] * c2) * n[2]};
                    float aa[3] = {n[0] * n[0], n[1] * n[1], n[2] * n[2]};
                    warp_sum4(lane, ab[0], ab[1], ab[2], aa[0]);
                    warp_sum2(lane, aa[1], aa[2]);
                    colour_scale_step(cc, ab, aa);
                    c0 = cc[0]; c1 = cc[1]; c2 = cc[2];
                    if (lane == k) { cs0_l = c0; cs1_l = c1; cs2_l = c2; }
                }
            }
            // Gauss-Newton terms (patch_optimization.cc:283-288 / :324-343); only meaningful when every view's
            // derivative path succeeded, which the caller checks through the DER bits
            if ((r & 2u) && act) {
                const float g0 = c0 * d[0], g1 = c1 * d[1], g2 = c2 * d[2];
                const float r0 = m0 - c0 * n[0], r1 = m1 - c1 * n[1], r2 = m2 - c2 * n[2];
                num += g0 * r0 + g1 * r1 + g2 * r2;
                den += g0 * g0 + g1 * g1 + g2 * g2;
                if (want_normal) {
                    const float gg[3] = {g0, g1, g2};
                    const float rr[3] = {r0, r1, r2};
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        const float a0 = gg[ch];
                        const float a1 = fi * a0;      // (ii * cs) * deriv == ii * (cs * deriv) exactly for ii in {-2..2}
                        const float a2 = fj * a0;
                        A0 += a0 * a0; A1 += a0 * a1; A2 += a0 * a2;
                        A3 += a1 * a1; A4 += a1 * a2; A5 += a2 * a2;
                        B0 += a0 * rr[ch]; B1 += a1 * rr[ch]; B2 += a2 * rr[ch];
                    }
                }
            }
        }
        if (candidates) return;
        warp_sum2(lane, num, den);
        po.num = num; po.den = den;
        if (want_ncc) bits |= F_HAS_NCC | ((__ballot_sync(FULL, df_l) & 0xFu) << SH_DF);
        if (want_normal) bits |= F_HAS_NORMAL;
        // the bits of the last pass replace those of the pass before (the DF bits only when this pass overwrote the NCCs)
        pk = (pk & ~((0xFFu << SH_COL) | (want_ncc ? 0xFu << SH_DF : 0u) | F_HAS_NORMAL | F_HAS_NCC)) | bits;
        if (want_normal) {
            // solve here so that the nine fp64 sums die with the pass (matrix_tools.h:392-398,460-475)
            // the lane's <= 12 products (3 channels x <= 4 views) are summed in fp32, the 25 lanes in fp64; the reference sums
            // all 300 fp32 products in fp64 (patch_optimization.cc:336-342).  The difference (~1e-7 relative on ATA) is far
            // below what the Gauss-Newton fixed point resolves; measured in tests/test_gpu_parity.py.
            const double D0 = warp_sum((double)A0), D1 = warp_sum((double)A1), D2 = warp_sum((double)A2), D3 = warp_sum((double)A3);
            const double D4 = warp_sum((double)A4), D5 = warp_sum((double)A5);
            const double E0 = warp_sum((double)B0), E1 = warp_sum((double)B1), E2 = warp_sum((double)B2);
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

    // ---- sorted insert / erase on the lane-distributed selected set (std::set semantics) ----
    __device__ __forceinline__ void sel_erase_mask(unsigned mask)       // bit k: remove element k
    {
        // gather: new position p takes the p-th kept element
        int src = 0, cnt = 0;
        for (int k = 0; k < MAX_LOCAL; ++k) {
            const bool kk = k < nsel() && !((mask >> k) & 1u);
            if (kk) { if (cnt == lane) src = k; ++cnt; }
        }
        const int s = __shfl_sync(FULL, sel_l, src);
        const float a = __shfl_sync(FULL, cs0_l, src), b = __shfl_sync(FULL, cs1_l, src), c = __shfl_sync(FULL, cs2_l, src);
        const float v = __shfl_sync(FULL, ncc_l, src);
        set_nsel(cnt);
        if (lane < cnt) { sel_l = s; cs0_l = a; cs1_l = b; cs2_l = c; ncc_l = v; }
        else { sel_l = 0xFF; }
    }
    __device__ __forceinline__ void sel_insert(int slot, float cs_init)
    {
        // position = number of selected slots smaller than `slot`
        const int n = nsel();
        const unsigned smaller = __ballot_sync(FULL, lane < n && sel_l < slot);
        const int pos = __popc(smaller);
        const int s_up = __shfl_up_sync(FULL, sel_l, 1);
        const float a_up = __shfl_up_sync(FULL, cs0_l, 1), b_up = __shfl_up_sync(FULL, cs1_l, 1), c_up = __shfl_up_sync(FULL, cs2_l, 1);
        const float v_up = __shfl_up_sync(FULL, ncc_l, 1);
        if (lane > pos && lane <= n) { sel_l = s_up; cs0_l = a_up; cs1_l = b_up; cs2_l = c_up; ncc_l = v_up; }
        if (lane == pos) { sel_l = slot; cs0_l = cs1_l = cs2_l = cs_init; ncc_l = 0.f; }
        set_nsel(n + 1);
    }
    __device__ __forceinline__ unsigned low_ncc_mask() const
    {
        return __ballot_sync(FULL, lane < nsel() && ncc_l < st->accept_ncc);
    }

    // Second half of LocalViewSelection::performVS (local_view_selection.cc:86-147): greedy selection among the
    // candidates that survived the NCC test of pass(candidates = true); lane i evaluates candidate slot i.
    __device__ __forceinline__ void lvs_greedy(const float*)
    {
        const unsigned N = st->nr_recon_neighbors;
        const float cs_init = 1.f / mm;
        float rdx = cpx - __ldg(&rv->campos[0]), rdy = cpy - __ldg(&rv->campos[1]), rdz = cpz - __ldg(&rv->campos[2]);
        {
            const float nn = sqrtf(rdx * rdx + rdy * rdy + rdz * rdz);
            rdx /= nn; rdy /= nn; rdz /= nn;
        }
        const int G = job->n_global;
        // per-lane candidate geometry (viewDir, epipolarPlane, footprint)
        float vdx = 0.f, vdy = 0.f, vdz = 1.f, epx = 0.f, epy = 0.f, epz = 1.f, nfp = 1.f;
        if (lane < G) view_geometry(&views[job->gview[lane]], cpx, cpy, cpz, rdx, rdy, rdz, vdx, vdy, vdz, epx, epy, epz, nfp);
        bool found = true;
        while ((unsigned)nsel() < N && found) {
            found = false;
            const bool mine = lane < G && ((avail >> lane) & 1u);
            float score = -1.f;
            if (mine) {
                score = cand_ncc_l;
                if (mfp / nfp < 0.5f) score *= 0.01f;
                float dp = clamp1(rdx * vdx + rdy * vdy + rdz * vdz);
                score *= plx_weight(deg_acos(dp));
            }
            // parallax / epipolar terms against every already selected view (geometry broadcast from its lane)
            for (int k = 0; k < nsel(); ++k) {
                const int s = __shfl_sync(FULL, sel_l, k);
                const float sx = __shfl_sync(FULL, vdx, s), sy = __shfl_sync(FULL, vdy, s), sz = __shfl_sync(FULL, vdz, s);
                const float ex = __shfl_sync(FULL, epx, s), ey = __shfl_sync(FULL, epy, s), ez = __shfl_sync(FULL, epz, s);
                if (mine) lvs_weigh(score, vdx, vdy, vdz, epx, epy, epz, sx, sy, sz, ex, ey, ez, st->min_parallax);
            }
            const bool cand = mine && (score > 0.f);       // NaN compares false, like `score > maxScore`
            const float best = warp_max(cand ? score : -1.f);
            const unsigned winners = __ballot_sync(FULL, cand && score == best);
            if (best > 0.f && winners) {
                const int w = __ffs(winners) - 1;           // strict '>' in index order: lowest index wins ties
                found = true;
                sel_insert(w, cs_init);
                avail &= ~(1u << w);
            }
        }
        if ((unsigned)nsel() == N) pk |= F_LVS_OK;
    }

    // PatchOptimization ctor (patch_optimization.cc:21-78) incl. LocalViewSelection ctor (local_view_selection.cc:19-54),
    // up to the point where the first sample sets are needed; sets the first stage of the state machine.
    __device__ __forceinline__ void begin(const JobParams* j, const PatchIn& in)
    {
        job = j;
        rv = &views[job->ref_view];
        reset(in);
        sel_l = 0xFF; cs0_l = cs1_l = cs2_l = 0.f; ncc_l = 0.f; cand_ncc_l = 0.f;
        init_sampler(in.x, in.y);
        // propagated ids arrive ascending, 0xFF padded
        if (lane < MAX_LOCAL) sel_l = (in.slots >> (8 * lane)) & 0xFF;
        int n = __popc(__ballot_sync(FULL, lane < MAX_LOCAL && sel_l != 0xFF));
        set_nsel(n);
        if (!is(F_REF_OK)) { pk &= ~F_OPTI; return; }
        const unsigned N = st->nr_recon_neighbors;
        if ((unsigned)n == N) pk |= F_LVS_OK;
        else if ((unsigned)n > N) { n = 0; set_nsel(0); sel_l = 0xFF; }
        avail = job->n_global >= 32 ? FULL : ((1u << job->n_global) - 1u);
        unsigned m = 0u;
        for (int k = 0; k < n; ++k) m |= 1u << __shfl_sync(FULL, sel_l, k);
        avail &= ~m;
        cs0_l = cs1_l = cs2_l = 1.f / mm;
        set_stage(is(F_LVS_OK) ? CTOR : LVS_CTOR);
    }

    __device__ __forceinline__ bool step() { return auto_step(*this); }

    // PatchOptimization::computeConfidence (patch_optimization.cc:114-142) + getPatchNormal (patch_sampler.cc:243-256)
    __device__ __forceinline__ void finish(PatchOut& out)
    {
        finish_state(out);
        const int n = nsel();
        unsigned s = 0u;
#pragma unroll
        for (int k = 0; k < MAX_LOCAL; ++k) {
            const int v = __shfl_sync(FULL, sel_l, k);
            s |= (unsigned)((k < n) ? (v & 0xFF) : 0xFF) << (8 * k);
        }
        out.slots = s;
        if (!is(F_CONVERGED)) return;
        // mean NCC of the final state (the NCCs of the last pass)
        float mean = 0.f;
        for (int k = 0; k < n; ++k) mean += __shfl_sync(FULL, ncc_l, k);
        mean /= (float)n;
        const float ax_ = __shfl_sync(FULL, px, CENTER + 2) - __shfl_sync(FULL, px, CENTER - 2);
        const float ay_ = __shfl_sync(FULL, py, CENTER + 2) - __shfl_sync(FULL, py, CENTER - 2);
        const float az_ = __shfl_sync(FULL, pz, CENTER + 2) - __shfl_sync(FULL, pz, CENTER - 2);
        const float bx_ = __shfl_sync(FULL, px, 2) - __shfl_sync(FULL, px, NS - 1 - 2);
        const float by_ = __shfl_sync(FULL, py, 2) - __shfl_sync(FULL, py, NS - 1 - 2);
        const float bz_ = __shfl_sync(FULL, pz, 2) - __shfl_sync(FULL, pz, NS - 1 - 2);
        confidence(out, ax_, ay_, az_, bx_, by_, bz_, crx, cry, crz, mean, st->accept_ncc);
    }
};


__device__ __forceinline__ void bind_thread(PatchW& p, const DevSettings* st, const ViewParams* views, const float* lut_rep, int tid)
{
    p.st = st; p.views = views;
    p.lane = tid & 31;
    p.lut_tab = lut_rep; p.lane4 = 4u * (unsigned)(p.lane & (LUT_REP - 1));
    p.pk = (unsigned)PatchW::DONE << PatchW::SH_STAGE;
    p.n_sets = 0u;
}

} // namespace b200mvs
