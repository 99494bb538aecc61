/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 * The gather of the product's import and undistortion (mve_b200/csrc/undistort.cuh) compiled by g++ as host code, over a
 * whole image given as a device image source describes it: base, row pitch and plane pitch (0 = interleaved HWC, else
 * planar CHW).  Without coefficients every channel is copied through texel() and channel_offset(), as k_import_rgb reads
 * them; with coefficients it is what k_undistort_k2k4 computes before the RGBX conversion.  Built by
 * tests/test_device_source.py with -ffp-contract=off, so that the header's unfused operations stay unfused. */
#define B200MVS_HOST_EMU 1
#include "../../mve_b200/csrc/undistort.cuh"

using namespace b200mvs_undistort;

template <bool Planar>
static void run(const Src& src, int w, int h, int ch, float flen, float k2, float k4, uint8_t* out)
{
    const bool undistort = active(k2, k4);
    const Params P = make_params(w, h, ch, flen, k2, k4);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            uint8_t* o = out + ((size_t)y * w + x) * ch;
            if (undistort) {
                const uint32_t v = undistort_px<Planar>(P, src, x, y);
                for (int c = 0; c < ch; ++c) o[c] = (uint8_t)(v >> (8 * c));
            } else {
                const uint8_t* p = texel<Planar>(src, ch, x, y);
                for (int c = 0; c < ch; ++c) o[c] = p[channel_offset<Planar>(src, c)];
            }
        }
}

extern "C" void emu_undistort_src(const uint8_t* base, int64_t row_pitch, int64_t plane_pitch, int w, int h, int ch,
                                  float flen, float k2, float k4, uint8_t* out)
{
    const Src src{base, row_pitch, plane_pitch};
    if (plane_pitch) run<true>(src, w, h, ch, flen, k2, k4, out);
    else             run<false>(src, w, h, ch, flen, k2, k4, out);
}
