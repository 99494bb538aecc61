// The state a prior seed carries besides its depth (b200mvs_set_view_prior_state, include/b200mvs.h): its dz, scaled to
// the entry's pixel size, and its local views as slots of the entry's global selection.  k_prior_seeds calls it for
// every seed; tests/emu compiles the same function with g++ and checks it against tests/prior_state_reference.py.
#pragma once
#if defined(B200MVS_HOST_EMU)
#include "simt_emu.h"      // tests/emu: runs this very file on the CPU (test infrastructure)
#else
#include <cuda_runtime.h>
#endif
#include <cmath>
#include <stdint.h>

namespace b200mvs {

struct PriorState {
    float dzI, dzJ;
    unsigned slots;        // 4 x uint8 global slots, ascending, 0xFF padded; 0xFFFFFFFF = no local views
};

// What the prior holds at the pixel a candidate reads, besides its depth
struct PriorPixel {
    bool has_dz, has_ids;  // whether the prior has a dz map / an id map
    float dz[2];
    int32_t ids[4];
};

// p: the prior pixel.  w x h: the prior's size, W x H: the entry's map.  gview[0, n_global): the entry's global
// selection, ascending (slot -> id).  N: nr_recon_neighbors.  A dz that is not finite after scaling gives (0, 0); the
// distinct ids >= 0 that are in gview become the local views when there are exactly N of them, else there are none.
__host__ __device__ inline PriorState prior_seed_state(const PriorPixel& p, int w, int h, int W, int H, const int* gview,
                                                       int n_global, unsigned N)
{
    PriorState s{0.f, 0.f, 0xFFFFFFFFu};
    if (p.has_dz) {
        const float di = p.dz[0] * ((float)w / (float)W), dj = p.dz[1] * ((float)h / (float)H);
        // |v| <= FLT_MAX: finite (NaN fails the comparison)
        if (fabsf(di) <= 3.40282347e38f && fabsf(dj) <= 3.40282347e38f) { s.dzI = di; s.dzJ = dj; }
    }
    if (p.has_ids) {
        unsigned found = 0;            // a bit per global slot: distinct by construction
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int id = p.ids[k];
            if (id < 0) continue;
            for (int g = 0; g < n_global; ++g)
                if (gview[g] == id) { found |= 1u << g; break; }
        }
        unsigned word = 0xFFFFFFFFu, n = 0;    // n <= 4: four ids
        for (int g = 0; g < n_global && found; ++g, found >>= 1)
            if (found & 1u) { word = (word & ~(0xFFu << (8 * n))) | ((unsigned)g << (8 * n)); ++n; }
        if (n == N) s.slots = word;
    }
    return s;
}

} // namespace b200mvs
