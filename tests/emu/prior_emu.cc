/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 * The state rule of a prior seed (mve_b200/csrc/prior_seed.cuh prior_seed_state, called by k_prior_seeds) compiled by
 * g++, so that tests/test_prior_state_emulated.py can compare it with tests/prior_state_reference.py. */
#define B200MVS_HOST_EMU 1
#include "simt_emu.h"

namespace simt_emu {
thread_local Warp* t_warp = nullptr;
thread_local int t_lane = 0;
thread_local int t_sense_full = 0;
thread_local int t_sense_sub = 0;
}

#include "../../mve_b200/csrc/prior_seed.cuh"

using namespace b200mvs;

extern "C" {

/* n candidates: dz[2 i..], ids[4 i..] (either may be null = no such map); out_dz[2 i..] and out_slots[i] receive the
 * state of candidate i for a w x h prior read by an entry with a W x H map, global selection gview[0, n_global) and N. */
void emu_prior_seed_state(int n, const float* dz, const int32_t* ids, int w, int h, int W, int H, const int* gview,
                          int n_global, unsigned N, float* out_dz, unsigned* out_slots)
{
    for (int i = 0; i < n; ++i) {
        PriorPixel p = {dz != nullptr, ids != nullptr, {0.f, 0.f}, {-1, -1, -1, -1}};
        if (dz) { p.dz[0] = dz[2 * i]; p.dz[1] = dz[2 * i + 1]; }
        if (ids) for (int k = 0; k < 4; ++k) p.ids[k] = ids[4 * i + k];
        const PriorState s = prior_seed_state(p, w, h, W, H, gview, n_global, N);
        out_dz[2 * i] = s.dzI;
        out_dz[2 * i + 1] = s.dzJ;
        out_slots[i] = s.slots;
    }
}

}
