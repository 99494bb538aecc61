/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 * The rules of a relative prior (mve_b200/csrc/prior_align.cuh: align_pixel, align_observation, align_fit and
 * align_apply, called by k_align_observe, k_align_fit and k_align_apply) compiled by g++, so that
 * tests/test_prior_align_emulated.py can compare them with tests/prior_align_reference.py.  align_fit runs with
 * sequential collective steps: an exact selection by std::nth_element and sums in index order. */
#define B200MVS_HOST_EMU 1
#include "simt_emu.h"

namespace simt_emu {
thread_local Warp* t_warp = nullptr;
thread_local int t_lane = 0;
thread_local int t_sense_full = 0;
thread_local int t_sense_sub = 0;
}

#include "../../mve_b200/csrc/prior_align.cuh"

#include <algorithm>
#include <vector>

using namespace b200mvs;

namespace {

struct SeqOps {
    template <typename K> double select(unsigned m, unsigned k, K&& key)
    {
        std::vector<unsigned long long> v(m);
        for (unsigned i = 0; i < m; ++i) v[i] = key(i);
        std::nth_element(v.begin(), v.begin() + k, v.end());
        return align_unkey(v[k]);
    }
    template <typename F> void sum2(unsigned m, F&& f, double* A, double* B)
    {
        double a = 0.0, b = 0.0;
        for (unsigned i = 0; i < m; ++i) {
            double x, z;
            f(i, &x, &z);
            a += x;
            b += z;
        }
        *A = a;
        *B = b;
    }
    template <typename P> unsigned count(unsigned m, P&& pred)
    {
        unsigned c = 0;
        for (unsigned i = 0; i < m; ++i) c += pred(i) ? 1u : 0u;
        return c;
    }
};

AlignCam make_cam(const double* R, const double* t, const double* calib, int W0, int H0)
{
    AlignCam c;
    for (int k = 0; k < 9; ++k) c.R[k] = R[k];
    for (int k = 0; k < 3; ++k) c.t[k] = t[k];
    c.ax = calib[0]; c.ay = calib[1]; c.cx = calib[2]; c.cy = calib[3];
    c.W0 = W0; c.H0 = H0;
    return c;
}

} // namespace

extern "C" {

/* n features pos[3 i..] in a w x h map: out_px[i], out_py[i] the prior pixel (-1 without one), out_dy[2 i..] the
 * observation (d, y), (0, 0) without one.  calib = ax, ay, cx, cy. */
void emu_align_observe(int n, const float* pos, const double* R, const double* t, const double* calib, int W0, int H0,
                       const float* values, int w, int h, int kind, int* out_px, int* out_py, double* out_dy)
{
    const AlignCam c = make_cam(R, t, calib, W0, H0);
    for (int i = 0; i < n; ++i) {
        int px = -1, py = -1;
        double z, d = 0.0, y = 0.0;
        if (align_pixel(c, pos[3 * i], pos[3 * i + 1], pos[3 * i + 2], w, h, &px, &py, &z)) {
            if (!align_observation(kind, z, values[(size_t)py * w + px], &d, &y)) d = y = 0.0;
        } else {
            px = py = -1;
        }
        out_px[i] = px; out_py[i] = py;
        out_dy[2 * i] = d; out_dy[2 * i + 1] = y;
    }
}

/* The fit of m slots d[i], y[i] (d = 0: no observation).  out = s, t, median_rel_err; counts = n_obs, n_inliers;
 * returns the AlignStatus. */
int emu_align_fit(unsigned m, const double* d, const double* y, int kind, double* out, unsigned* counts)
{
    SeqOps ops;
    const AlignFit f = align_fit(ops, d, y, m, kind);
    out[0] = f.s; out[1] = f.t; out[2] = f.med_rel;
    counts[0] = f.n_obs; counts[1] = f.n_in;
    return f.status;
}

/* The apply over a w x h map into out (w x h floats) */
void emu_align_apply(const double* calib, int W0, int H0, int kind, double s, double t, const float* values, int w, int h,
                     float* out)
{
    const double R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, tr[3] = {0, 0, 0};
    const AlignCam c = make_cam(R, tr, calib, W0, H0);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) out[(size_t)y * w + x] = align_apply(c, kind, s, t, values[(size_t)y * w + x], x, y, w, h);
}

}
