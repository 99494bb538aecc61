/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 * The product's per-pixel undistortion (mve_b200/csrc/undistort.cuh) compiled by g++ as host code, over a whole image:
 * what k_undistort_k2k4 computes before the RGBX conversion.  Built by tests/test_undistort_reference.py with
 * -ffp-contract=off, so that the header's unfused operations stay unfused. */
#define B200MVS_HOST_EMU 1
#include "../../mve_b200/csrc/undistort.cuh"

#include <cstring>

extern "C" void emu_undistort(const uint8_t* src, int w, int h, int ch, float flen, float k2, float k4, uint8_t* out)
{
    using namespace b200mvs_undistort;
    if (!active(k2, k4)) { std::memcpy(out, src, (size_t)w * h * ch); return; }
    const Params P = make_params(w, h, ch, flen, k2, k4);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const uint32_t v = undistort_px(P, src, x, y);
            for (int c = 0; c < ch; ++c) out[((size_t)y * w + x) * ch + c] = (uint8_t)(v >> (8 * c));
        }
}
