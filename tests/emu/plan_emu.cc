/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 * Runs the product's device planner for one reference view (mve_b200/csrc/plan_device.cuh, compiled by g++) on the CPU:
 * one CTA = `nt` host threads that run the phases of plan_view with a barrier between two, as the kernel's threads do.
 * Also checks the device's parallax-factor look-up against the host planner's plx_factor over ranges of floats.
 * Built by tests/emu/build.py into tests/emu/libplan_emu.so. */
#define B200MVS_HOST_EMU 1
#include "simt_emu.h"

namespace simt_emu {
thread_local Warp* t_warp = nullptr;
thread_local int t_lane = 0;
thread_local int t_sense_full = 0;
thread_local int t_sense_sub = 0;
}

#include "../../mve_b200/csrc/plan_device.cuh"

#include <thread>
#include <vector>

using namespace b200mvs_plan;

extern "C" {

int emu_plan_view_size(void) { return (int)sizeof(PlanView); }

/* The plan of view `ref`: selection into sel (up to MAX_SEL), seeds {x, y, depth} into seeds (up to seed_cap).
 * Returns the number of seeds, -1 when the factor table would exceed its cap, -2 when seed_cap is too small. */
int emu_plan_view(const PlanView* views, int nv, const float* fpos, const int* foff, const int* frefs, int nf,
                  const int* vfoff, const int* vfids, float min_parallax, const float* aabb, int gvs_max, int ref, int nt,
                  int* sel, int* n_sel, SeedOut* seeds, int seed_cap)
{
    const float dot_skip = host_dot_skip(min_parallax);
    const uint64_t n_table = table_entries(dot_skip);
    if (n_table == 0) return -1;
    std::vector<float> table(n_table);
    fill_table(table.data(), n_table, dot_skip, min_parallax);
    PlanInput in = {};
    in.views = views; in.feat_pos = fpos; in.feat_off = foff; in.feat_refs = frefs; in.vf_off = vfoff; in.vf_ids = vfids;
    in.table = table.data(); in.nv = nv; in.nf = nf; in.dot_skip = dot_skip; in.gvs_max = gvs_max;
    for (int i = 0; i < 3; ++i) { in.aabb_min[i] = aabb[i]; in.aabb_max[i] = aabb[3 + i]; }
    PlanJob job = {};
    job.ref = ref;
    job.F = vfoff[ref + 1] - vfoff[ref];
    for (int t = vfoff[ref]; t < vfoff[ref + 1]; ++t) job.E += (uint64_t)(foff[vfids[t] + 1] - foff[vfids[t]]);
    job.seed_cap = (uint64_t)nf;
    std::vector<uint32_t> ws(job_layout(job.F, job.E, nv, nf).words + 1, 0xDEADBEEFu);   // garbage: nothing may read it unwritten
    std::vector<uint32_t> out(out_words(job.seed_cap), 0);
    simt_emu::Barrier bar;
    bar.n = nt;
    std::vector<std::thread> th;
    for (int tid = 0; tid < nt; ++tid)
        th.emplace_back([&, tid]() {
            int sense = 0;
            PlanBlock B;
            B.bind(&in, &job, ws.data(), out.data());
            plan_view(B, tid, nt, [&]() { bar.wait(sense); });
        });
    for (std::thread& t : th) t.join();
    *n_sel = (int)out[0];
    for (uint32_t k = 0; k < out[0] && k < (uint32_t)MAX_SEL; ++k) sel[k] = (int)out[OUT_SEL + k];
    if ((int)out[1] > seed_cap) return -2;
    const SeedOut* so = reinterpret_cast<const SeedOut*>(out.data() + OUT_HEAD);
    for (uint32_t i = 0; i < out[1]; ++i) seeds[i] = so[i];
    return (int)out[1];
}

/* Every float with bits in [bits(dot_skip) - below, bits(1) + above]: how many give a look-up that differs (bitwise) from
 * the host's plx_factor; *n_checked receives the count of floats checked.  -1 when the table would exceed its cap. */
long long emu_check_lookup(float min_parallax, unsigned below, unsigned above, long long* n_checked)
{
    const float dot_skip = host_dot_skip(min_parallax);
    const uint64_t n_table = table_entries(dot_skip);
    if (n_table == 0) return -1;
    std::vector<float> table(n_table);
    fill_table(table.data(), n_table, dot_skip, min_parallax);
    const uint32_t lo = __float_as_uint(dot_skip) - below, hi = __float_as_uint(1.f) + above;
    long long bad = 0, n = 0;
    for (uint64_t b = lo; b <= hi; ++b, ++n) {
        float dt;
        const uint32_t u = (uint32_t)b;
        std::memcpy(&dt, &u, 4);
        const float want = host_plx_factor(dt, dot_skip, min_parallax), got = plx_lookup(dt, dot_skip, table.data());
        bad += __float_as_uint(want) != __float_as_uint(got);
    }
    *n_checked = n;
    return bad;
}

} // extern "C"
