// libb200mvs.so - C ABI of include/b200mvs.h: context, image pyramids, host-side view selection and seeds,
// frontier (region growing) orchestration and all CUDA kernels.  sm_90a only; no CPU fallback.
#include "../../include/b200mvs.h"
#include "patch_opt.cuh"
#include "patch_warp.cuh"
#include "patch_thread.cuh"
#include "pset_device.cuh"
#include "host_common.cuh"
#include "plan_device.cuh"
#include "prior_seed.cuh"
#include "prior_align.cuh"
#include "undistort.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstddef>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <functional>
#include <map>
#include <memory>
#include <chrono>
#include <ctime>
#include <mutex>
#include <string>
#include <thread>
#include <atomic>
#include <vector>

using namespace b200mvs;
using namespace b200mvs_host;
namespace PL = b200mvs_plan;

// ------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------
namespace {

// Every device allocation of a context goes through these two (defined after b200mvs_ctx): they keep the resident / peak
// byte counts of b200mvs_memory_stats and make room within the budget first.
cudaError_t dev_alloc(b200mvs_ctx* ctx, void** p, size_t bytes);
void dev_free(b200mvs_ctx* ctx, void* p, size_t bytes);

// A device buffer of context `ctx`, allocated through its accounted allocator and freed when it goes out of scope
template <typename T> struct DevBuf {
    b200mvs_ctx* ctx;
    T* p = nullptr;
    size_t cap = 0;
    explicit DevBuf(b200mvs_ctx* c) : ctx(c) {}
    DevBuf(DevBuf&& o) noexcept : ctx(o.ctx), p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    ~DevBuf() { release(); }
    size_t bytes() const { return cap * sizeof(T); }
    cudaError_t reserve(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        release();
        cudaError_t e = dev_alloc(ctx, reinterpret_cast<void**>(&p), n * sizeof(T));
        if (e == cudaSuccess) cap = n;
        return e;
    }
    void release() { dev_free(ctx, p, bytes()); p = nullptr; cap = 0; }
    // grows to n elements keeping the first `keep`: the copy has finished before the old buffer is freed
    cudaError_t grow(size_t n, size_t keep, cudaStream_t st)
    {
        if (n <= cap) return cudaSuccess;
        if (keep == 0) return reserve(n);
        T* q = nullptr;
        cudaError_t e = dev_alloc(ctx, reinterpret_cast<void**>(&q), n * sizeof(T));
        if (e != cudaSuccess) return e;
        e = cudaMemcpyAsync(q, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { dev_free(ctx, q, n * sizeof(T)); return e; }
        release();
        p = q; cap = n;
        return cudaSuccess;
    }
};

// Owners of the pinned host blocks, events and stream of a context
struct FreeHost { void operator()(void* p) const { cudaFreeHost(p); } };
struct DestroyEvent { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
struct DestroyStream { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
template <typename T> using Pinned = std::unique_ptr<T, FreeHost>;
using Event = std::unique_ptr<CUevent_st, DestroyEvent>;
using Stream = std::unique_ptr<CUstream_st, DestroyStream>;

struct HostLevel {
    int w = 0, h = 0, pitch = 0;
    float proj[9], invproj[9];
    uchar4* d_img = nullptr;
    uint4* d_quad = nullptr;       // 2x2 neighbourhood of every texel, 16 bytes (patch_opt.cuh LevelParams::quad)
};

struct HostView {
    bool valid = false;            // a SingleView exists (camera + image dimensions known)
    bool has_image = false;        // loadColorImage done: pyramid resident on the device
    int w = 0, h = 0;
    float flen = 0, paspect = 1, pp[2] = {0.5f, 0.5f}, rot[9], trans[3];
    float k2 = 0, k4 = 0;          // radial distortion of the images it is given (b200mvs_set_view_distortion)
    std::vector<uint8_t> mask;     // reconstruction mask, mask_w x mask_h, 0 = background (b200mvs_set_view_mask); empty: none
    DevBuf<uint8_t> mask_dev;      // ... or the same in device memory (b200mvs_set_view_mask_device); at most one of the two
    int mask_w = 0, mask_h = 0;
    DevBuf<float> prior;           // prior depth map, prior_w x prior_h (b200mvs_set_view_prior[_state][_device]); null: none
    DevBuf<float2> prior_dz;       // ... its dz map (b200mvs_set_view_prior_state[_device]); null: none
    DevBuf<int4> prior_ids;        // ... its view-id map; null: none
    int prior_w = 0, prior_h = 0, prior_stride = 0;
    float campos[3];
    float w2c[12];
    std::vector<HostLevel> lv;
    DevBuf<uchar4> pyr;            // one allocation for every level: the RGBX8 images, then their quad images
    uint64_t last_use = 0;         // eviction order: least recently used first
    explicit HostView(b200mvs_ctx* ctx) : mask_dev(ctx), prior(ctx), prior_dz(ctx), prior_ids(ctx), pyr(ctx) {}
    bool masked() const { return !mask.empty() || mask_dev.p; }
};

// Device bytes of a view's pyramid: every level of buildPyramid, RGBX8 + quad image (16 B) per texel at a pitch of 4 texels
size_t pyramid_bytes(const HostView& v)
{
    size_t texels = 0;
    for (const HostLevel& L : v.lv) texels += (size_t)L.pitch * L.h;
    return texels * (sizeof(uchar4) + sizeof(uint4));
}

// b200mvs_set_view_mask: the mask column (row) under the centre of column (row) x of a map n pixels wide (high), for a
// mask m pixels wide (high): floor((2x+1) m / 2n)
__host__ __device__ inline int mask_coord(int x, int n, int m) { return (int)((2ll * x + 1) * m / (2ll * n)); }
// whether pixel (x, y) of view v's W x H map is background under its host mask; a pixel outside the map is not
bool background(const HostView& v, int W, int H, int x, int y)
{
    if (v.mask.empty() || x < 0 || y < 0 || x >= W || y >= H) return false;
    return v.mask[(size_t)mask_coord(y, H, v.mask_h) * v.mask_w + mask_coord(x, W, v.mask_w)] == 0;
}
// bg[y * W + x] = 1 where pixel (x, y) of view v's W x H map is background, else 0 (v has a host mask)
void mark_background(const HostView& v, int W, int H, unsigned char* bg)
{
    std::vector<int> col(W);
    for (int x = 0; x < W; ++x) col[x] = mask_coord(x, W, v.mask_w);
    for (int y = 0; y < H; ++y) {
        const uint8_t* row = v.mask.data() + (size_t)mask_coord(y, H, v.mask_h) * v.mask_w;
        unsigned char* out = bg + (size_t)y * W;
        if (v.mask_w == W) for (int x = 0; x < W; ++x) out[x] = row[x] == 0;          // col[x] == x: no gather
        else for (int x = 0; x < W; ++x) out[x] = row[col[x]] == 0;
    }
}

// b200mvs_set_view_prior: the candidate columns (rows) of a map n pixels wide (high) at `stride`, x = 2 + stride i <= n - 3;
// a pixel nearer the edge fails in the PatchSampler ctor (patch_sampler.cc:47-50)
__host__ __device__ inline int prior_cells(int n, int stride) { return n >= 5 ? (n - 5) / stride + 1 : 0; }
// the candidate bound nx x ny of view v's prior at level `scale`: the most seeds it can add to an entry; 0 without a prior
uint64_t prior_bound(const HostView& v, int scale)
{
    if (!v.prior.p) return 0;
    const HostLevel& L = v.lv[scale];
    return (uint64_t)prior_cells(L.w, v.prior_stride) * (uint64_t)prior_cells(L.h, v.prior_stride);
}

struct HostPlan {                    // what DMRecon::start computes on the host before the queue runs (dmrecon.cc:179-292)
    b200mvs_settings settings;       // the settings it was made for
    std::vector<int> gsel;           // globalViewSelection result, ascending
    std::vector<PL::SeedOut> seeds;  // the feature loop of processFeatures
};

struct Entry {                     // frontier queue entry = QueueData (dmrecon.h:28-38)
    int xy;                        // x | y << 16
    int jobdir;                    // job | dir << 24 ; -1 = dropped
    float conf, depth, dzI, dzJ;
    unsigned slots;
    int pad;
};
static_assert(sizeof(Entry) == 32, "Entry layout");

// The Entry encodings of the host and the kernels.  dir: the side of the parent a neighbour was pushed from (0-3), 4 = seed.
__host__ __device__ __forceinline__ int pack_xy(int x, int y) { return x | (y << 16); }
__host__ __device__ __forceinline__ Entry make_entry(int xy, int job, int dir, float conf, float depth, float dzI, float dzJ, unsigned slots)
{
    return Entry{xy, job | (dir << 24), conf, depth, dzI, dzJ, slots, 0};
}
__device__ __forceinline__ int entry_x(const Entry& e) { return e.xy & 0xFFFF; }
__device__ __forceinline__ int entry_y(const Entry& e) { return (e.xy >> 16) & 0xFFFF; }
__device__ __forceinline__ int entry_job(const Entry& e) { return e.jobdir & 0xFFFFFF; }
__device__ __forceinline__ int entry_dir(const Entry& e) { return (e.jobdir >> 24) & 7; }
__device__ __forceinline__ int pixel_of(const JobParams& J, const Entry& e) { return entry_y(e) * J.W + entry_x(e); }
// the entry's 16x16-pixel tile among the tiles of all jobs of the launch
__device__ __forceinline__ long long tile_of(const JobParams& J, const Entry& e) { return J.tile_base + (long long)(entry_y(e) >> 4) * J.tiles_x + (entry_x(e) >> 4); }
__device__ __forceinline__ Entry child_entry(int xy, int job, int dir, const PatchOut& r) { return make_entry(xy, job, dir, r.conf, r.depth, r.dzI, r.dzJ, r.slots); }
// the bid of seed i with confidence c for its pixel: larger confidence first, then the earlier seed
__device__ __forceinline__ unsigned long long seed_key(float c, size_t i) { return ((unsigned long long)__float_as_uint(c) << 32) | (0xFFFFFFFFu - (unsigned)i); }

enum Counter { C_RUN = 0, C_NEXT = 1, C_OVERFLOW = 2, C_SETS = 3, C_OPTS = 4, C_SEED_OK = 5, C_FILLED = 6, C_TICKET = 7, C_NUM = 8 };

constexpr int HIST_FINE = 8192;                 // confidence bins of the eligibility threshold: bin = conf * 8192
constexpr int HIST_COARSE = 64;                 // one coarse bin per 128 fine bins
constexpr int HIST_PER_JOB = HIST_FINE + HIST_COARSE;
constexpr int DEFER_BIT = 1 << 27;              // Entry::jobdir flag: below this round's threshold, carried unchanged
enum Phase { PH_SEED = 0, PH_SELECT = 1, PH_THRESHOLD = 2, PH_PICK = 3, PH_OPT = 4, PH_COMMIT = 5, PH_EXPAND = 6, PH_SORT = 7, PH_OPT_THREAD = 8, PH_NUM = 9 };
// ST_GROW: the pushes of phase E might not fit the frontier arrays; the kernel stopped before them, the host grows the
// arrays and k_frontier_resume finishes the round (FrontierCtl::resume_*)
enum Stop { ST_RUN = 0, ST_CANCELLED = 2, ST_OVERFLOW = 3, ST_GROW = 4 };

struct FrontierCtl {                            // device memory, zeroed before the first launch of a group
    unsigned long long bar;                     // grid barrier ticket counter
    unsigned long long nlist[2];                // entries in list[0] / list[1]
    unsigned long long nrun;                    // winners of the current round
    unsigned long long ticket;                  // next patch of the current optimise phase
    unsigned long long ticket2;                 // ... of the tail of a large round (warp-per-patch path)
    unsigned long long sort_cursor;             // next free position of run2 while a round is being grouped by tile
    unsigned long long small_cursor;            // ... behind the grouped entries, for the views that run one warp per patch
    unsigned long long rounds, peak, barriers;
    unsigned long long ns[PH_NUM];              // %globaltimer time per phase, measured by CTA 0
    unsigned long long need;                    // bound on the next list after phase D: carried entries + 4 x pixels written
    unsigned long long resume_ncur, resume_nrun;   // ST_GROW: the stopped round's queue and winners
    int resume_p, resume_sorted;                // ... its parity and whether its winners are in run2
    int stop;
    int pad;
};

struct HostMirror {                             // mapped pinned host memory; followed by filled[n_jobs] (device -> host)
    volatile int cancel;                        // host -> device: stop the whole batch at the next round
    volatile int pad;
    volatile unsigned long long round, queue;   // device -> host
};                                              // ... and by cancel_job[n_jobs] (host -> device: drop this view's queue)

constexpr int MAX_GROUP_VIEWS = 4000;           // reference views per frontier launch
constexpr size_t MIRROR_BYTES = sizeof(HostMirror) + (sizeof(unsigned long long) + sizeof(int)) * MAX_GROUP_VIEWS;
static_assert(sizeof(HostMirror) % alignof(unsigned long long) == 0, "filled[] follows the mirror, aligned");

struct HostCounters {                           // pinned: what the host reads back after a launch
    unsigned long long count[C_NUM + MAX_GROUP_VIEWS];   // the Counter totals, then `filled` of every job of the group
    FrontierCtl ctl;
};
static_assert(offsetof(HostCounters, ctl) >= sizeof(unsigned long long) * (C_NUM + MAX_GROUP_VIEWS),
              "the counters of a full group end before the control block");

// Initial frontier capacity of a launch: max(ceil(per_px x pixels), seeds, min) entries (b200mvs_set_frontier_capacity).
struct FrontierCapacity {
    double per_px = 2.0;
    uint64_t min = 1u << 16;
};

// Sizes of one frontier launch (b200mvs_working_set): reference pixels at level `scale`, 16x16 tiles, seeds, views.
struct Workspace {
    size_t px = 0, tiles = 0, seeds = 0, jobs = 0;
    bool thresholded = false;
    FrontierCapacity fc;
    Workspace() = default;
    Workspace(const b200mvs_settings& s, const FrontierCapacity& c) : thresholded(s.frontier_band > 0.f || s.frontier_topk > 0), fc(c) {}
    // The seed round pushes at most one entry per seed, so `seeds` always fits it.  A later round that might not fit stops
    // the kernel before its pushes, and the launch resumes with larger arrays (run_group).
    size_t cap() const
    {
        return std::max<size_t>(std::max<size_t>((size_t)std::ceil(fc.per_px * (double)px), seeds), (size_t)fc.min);
    }
    void add(const Workspace& o) { px += o.px; tiles += o.tiles; seeds += o.seeds; jobs += o.jobs; }
};
constexpr size_t MAP_BYTES_PER_PX = 4 + 4 + 8 + 12 + 4 + 8;   // depth, conf, dz, normal, slots, sel
static_assert(sizeof(JobParams) == 232 && sizeof(PatchOut) == 40, "per-view and per-entry bytes of b200mvs_working_set (include/b200mvs.h)");

} // namespace

// Members are destroyed in reverse order: the accounting outlives every owner that updates it, the stream outlives the
// buffers, and the device buffers go before the pinned blocks and events.  A planning context (B200MVS_DEVICE_NONE) owns
// none of them, so destroying it makes no CUDA call.
struct b200mvs_ctx {
    int device = 0;
    // device memory accounting (dev_alloc), with the budget of the image source (b200mvs_set_image_source)
    b200mvs_memory mem = {};
    uint64_t pyr_resident = 0;         // part of mem.resident held by pyramids
    Stream stream;
    Event ev_begin, ev_end;            // the timing of a launch
    Event ev_copied;                   // a frontier launch's counters and control block are on the host
    Event ev_caller;                   // what a *_device call waits for on the caller's stream
    Event ev_source;                   // a device source's image is ready, and later the pyramids built from it
    Pinned<HostCounters> h_counters;
    Pinned<HostMirror> h_mirror;       // mapped, MIRROR_BYTES
    // b200mvs_upload_view staging: two slots used alternately, so that the host copy of view k+1 overlaps the H2D transfer
    // and the pyramid kernels of view k (SURVEY 8f rank 1).  For a host image a slot holds a pinned host block and a device
    // block; for a device image, read in place, it only charges the budget (next_stage).
    struct Stage {
        Pinned<uint8_t> host;
        DevBuf<uint8_t> dev;
        size_t charged = 0;            // bytes charged with dev_charge, without `dev`
        Event done;
        bool busy = false;
        explicit Stage(b200mvs_ctx* ctx) : dev(ctx) {}
        size_t cap() const { return dev.p ? dev.cap : charged; }
    };
    Stage stage[2] = {Stage(this), Stage(this)};
    unsigned stage_next = 0;
    std::mutex mtx;
    std::vector<HostView> views;
    // the features of b200mvs_set_features in the arrays of PL::PlanInput: positions, each feature's refs as registered,
    // and the inverted index, each view's ascending ids of the features that reference it
    std::vector<float> feat_pos;
    std::vector<int> feat_off{0}, feat_refs;
    std::vector<int> vf_off, vf_ids;
    DevBuf<ViewParams> d_views{this};
    bool views_dirty = true;
    DevBuf<float> d_lut{this};
    // workspace (grown on demand, reused across calls)
    DevBuf<Entry> ent_a{this}, ent_b{this}, run_in{this}, run_sorted{this};
    DevBuf<unsigned> tile_cnt{this};
    DevBuf<unsigned long long> tile_off{this};
    DevBuf<PatchOut> run_out{this};
    DevBuf<unsigned char> written{this};
    DevBuf<unsigned long long> counters{this};
    DevBuf<JobParams> d_jobs{this};
    DevBuf<DevSettings> d_settings{this};
    DevBuf<unsigned char> maps{this};  // all per-job maps of the current batch
    DevBuf<FrontierCtl> ctl{this};
    DevBuf<unsigned> hist{this};
    DevBuf<int> thr_bin{this};
    DevBuf<int> job_cancel{this};
    DevBuf<unsigned long long> job_run{this};
    int frontier_grid = 0;             // CTAs of the cooperative launch (= what fits on the chip)
    int optimize_grid = 0;             // resident CTAs of k_optimize
    long long thread_min = -1;         // reconstruct: rounds with at least this many patches run one thread per patch (-1: default)
    int optimize_mode = 0;             // b200mvs_optimize_patches: 0 by batch size, 1 one warp per patch, 2 one thread per patch
    // host plans prepared ahead by b200mvs_plan_views (global view selection + seed list of a reference view)
    std::mutex plan_mtx;
    std::map<int, HostPlan> plans;
    // pyramid eviction and the optional image source
    uint64_t use_clock = 0;
    b200mvs_fetch_fn fetch = nullptr;              // a host image source, or
    b200mvs_device_fetch_fn fetch_device = nullptr; // a device image source (at most one of the two is set)
    b200mvs_release_fn release = nullptr;
    void* user = nullptr;
    std::vector<char> pinned;          // views whose pyramids the running call needs: never evicted
    bool ws_busy = false;              // the workspace buffers belong to a launch being prepared: never dropped
    FrontierCapacity frontier_cap;     // b200mvs_set_frontier_capacity
    uint64_t fr_initial = 0, fr_final = 0, fr_resumes = 0;   // b200mvs_frontier_info of the last b200mvs_reconstruct
    b200mvs_plan_info plan_info = {};  // of the last b200mvs_reconstruct
    std::vector<float> plx_table;      // the device planner's parallax factors for min_parallax = plx_table_mp
    float plx_table_mp = -1.f;

    b200mvs_ctx(int device_, int n_views) : device(device_), vf_off(n_views + 1, 0)
    {
        views.reserve(n_views);
        for (int i = 0; i < n_views; ++i) views.emplace_back(this);
    }
};

namespace {

// ---- device memory: the one accounted allocator, eviction, workspace sizes ----
// The frontier arrays: one element per frontier entry each (169 bytes per entry), grown together when a launch resumes.
template <typename F> void for_each_frontier_array(b200mvs_ctx* ctx, F&& f)
{
    f(ctx->ent_a); f(ctx->ent_b); f(ctx->run_in); f(ctx->run_sorted); f(ctx->run_out); f(ctx->written);
}
// The workspace buffers of a frontier launch with their sizes in elements, in reservation order.  b200mvs_working_set
// sums the same list, so the estimate and the allocation cannot drift apart.
template <typename F> void for_each_workspace(b200mvs_ctx* ctx, const Workspace& w, F&& f)
{
    const size_t cap = w.cap();
    f(ctx->maps, w.px * MAP_BYTES_PER_PX + 256 * 8);
    for_each_frontier_array(ctx, [&](auto& buf) { f(buf, cap); });
    f(ctx->tile_cnt, w.tiles); f(ctx->tile_off, w.tiles);
    f(ctx->counters, C_NUM + w.jobs); f(ctx->d_jobs, w.jobs);
    f(ctx->thr_bin, w.jobs); f(ctx->job_cancel, w.jobs); f(ctx->job_run, w.jobs);
    f(ctx->hist, w.thresholded ? w.jobs * HIST_PER_JOB : 0);
}
uint64_t workspace_bytes(b200mvs_ctx* ctx, const Workspace& w)
{
    uint64_t b = 0;
    for_each_workspace(ctx, w, [&](auto& buf, size_t n) { b += n * sizeof(*buf.p); });
    return b;
}
// bytes the workspace holds after reserving for `w` without releasing anything first (buffers only grow)
uint64_t workspace_grown_bytes(b200mvs_ctx* ctx, const Workspace& w)
{
    uint64_t b = 0;
    for_each_workspace(ctx, w, [&](auto& buf, size_t n) { b += std::max(n, buf.cap) * sizeof(*buf.p); });
    return b;
}
void shrink_workspace(b200mvs_ctx* ctx, const Workspace& w)
{
    for_each_workspace(ctx, w, [&](auto& buf, size_t n) { if (buf.cap > n) buf.release(); });
}
void release_workspace(b200mvs_ctx* ctx)
{
    for_each_workspace(ctx, Workspace{}, [&](auto& buf, size_t) { buf.release(); });
}

// Allocations that do not depend on the batch: view table, sRGB table, settings, frontier control block and the two
// upload staging buffers, bounded by the largest registered image at 4 channels, the device reconstruction masks and the
// priors' depth, dz and view-id blocks.
uint64_t fixed_bytes(const b200mvs_ctx* ctx)
{
    size_t stage = 0, masks = 0;
    for (const HostView& v : ctx->views) {
        if (v.valid) stage = std::max(stage, (size_t)v.w * v.h * 4);
        masks += v.mask_dev.bytes() + v.prior.bytes() + v.prior_dz.bytes() + v.prior_ids.bytes();
    }
    return sizeof(ViewParams) * ctx->views.size() + 256 * sizeof(float) + sizeof(DevSettings) + sizeof(FrontierCtl) + 2 * stage + masks;
}

bool has_source(const b200mvs_ctx* ctx) { return ctx->fetch || ctx->fetch_device; }

// Device bytes the context may hold: the budget of its image source, no limit without one (b200mvs_memory::budget = 0)
uint64_t budget_limit(const b200mvs_ctx* ctx) { return ctx->mem.budget ? ctx->mem.budget : UINT64_MAX; }

void drop_pyramid(b200mvs_ctx* ctx, HostView& v)
{
    ctx->pyr_resident -= v.pyr.bytes();
    v.pyr.release();
    v.has_image = false;
    for (HostLevel& L : v.lv) { L.d_img = nullptr; L.d_quad = nullptr; }
    ctx->views_dirty = true;
}

// Whether the running call needs view v's pyramid (pin_views): it is never evicted
bool pinned(const b200mvs_ctx* ctx, size_t v) { return v < ctx->pinned.size() && ctx->pinned[v]; }

// Bytes of the resident pyramids that evict_lru may drop
uint64_t evictable_bytes(const b200mvs_ctx* ctx)
{
    uint64_t b = 0;
    for (size_t v = 0; v < ctx->views.size(); ++v)
        if (!pinned(ctx, v)) b += ctx->views[v].pyr.bytes();
    return b;
}

// Device bytes the running call may still allocate, keeping `reserve` free, when every evictable pyramid is dropped
uint64_t headroom(const b200mvs_ctx* ctx, uint64_t reserve)
{
    if (!ctx->mem.budget) return UINT64_MAX;
    const uint64_t limit = ctx->mem.budget + evictable_bytes(ctx);
    return limit > ctx->mem.resident + reserve ? limit - ctx->mem.resident - reserve : 0;
}

bool evict_lru(b200mvs_ctx* ctx)
{
    HostView* lru = nullptr;
    for (size_t i = 0; i < ctx->views.size(); ++i) {
        HostView& v = ctx->views[i];
        if (!v.pyr.p || pinned(ctx, i)) continue;
        if (!lru || v.last_use < lru->last_use) lru = &v;
    }
    if (!lru) return false;
    drop_pyramid(ctx, *lru);
    ctx->mem.n_evictions++;
    return true;
}

struct WorkspaceInUse {                         // the workspace belongs to the launch being prepared until the scope ends
    b200mvs_ctx* c;
    explicit WorkspaceInUse(b200mvs_ctx* c_) : c(c_) { c->ws_busy = true; }
    ~WorkspaceInUse() { c->ws_busy = false; }
};

// Frees pyramids of views the running call does not need, least recently used first, until `bytes` more fit the budget;
// outside a launch's preparation the workspace is dropped first.  Returns whether they fit.
bool make_room(b200mvs_ctx* ctx, uint64_t bytes)
{
    auto fits = [&]() { return ctx->mem.resident + bytes <= budget_limit(ctx); };
    if (fits()) return true;
    if (!ctx->ws_busy) release_workspace(ctx);
    while (!fits()) if (!evict_lru(ctx)) return false;
    return true;
}

void pin_views(b200mvs_ctx* ctx, const std::vector<int>& ids)
{
    ctx->pinned.assign(ctx->views.size(), 0);
    for (int id : ids) if (id >= 0 && id < (int)ctx->pinned.size()) { ctx->pinned[id] = 1; ctx->views[id].last_use = ++ctx->use_clock; }
}

struct PinsOfCall {                             // the views an entry point pins are unpinned when the call returns
    b200mvs_ctx* c;
    explicit PinsOfCall(b200mvs_ctx* c_) : c(c_) {}
    ~PinsOfCall() { c->pinned.assign(c->views.size(), 0); }
};

// The only cudaMalloc / cudaFree of the library (tests/test_device_budget.py checks the source).
cudaError_t dev_alloc(b200mvs_ctx* ctx, void** p, size_t bytes)
{
    *p = nullptr;
    if (bytes == 0) return cudaSuccess;
    if (!make_room(ctx, bytes)) return cudaErrorMemoryAllocation;
    const cudaError_t e = cudaMalloc(p, bytes);
    if (e != cudaSuccess) return e;
    ctx->mem.resident += bytes;
    ctx->mem.peak = std::max(ctx->mem.peak, ctx->mem.resident);
    return cudaSuccess;
}

// Charges `bytes` to the budget as dev_alloc does, without allocating them; dev_uncharge gives them back
cudaError_t dev_charge(b200mvs_ctx* ctx, size_t bytes)
{
    if (!make_room(ctx, bytes)) return cudaErrorMemoryAllocation;
    ctx->mem.resident += bytes;
    ctx->mem.peak = std::max(ctx->mem.peak, ctx->mem.resident);
    return cudaSuccess;
}

void dev_uncharge(b200mvs_ctx* ctx, size_t bytes) { ctx->mem.resident -= bytes; }

void dev_free(b200mvs_ctx* ctx, void* p, size_t bytes)
{
    if (!p) return;
    cudaFree(p);
    ctx->mem.resident -= bytes;
}

// The planning input of one call at level s.scale (plan_device.cuh): a PlanView of every registered camera into `views`
// (zero for a view without a camera) and the registered features, as host arrays.  Both planners read it, and
// plan_on_device uploads its arrays.  It reads only cameras and features: b200mvs_plan_views calls it without ctx->mtx.
PL::PlanInput plan_input(const b200mvs_ctx* c, const b200mvs_settings& s, std::vector<PL::PlanView>& views)
{
    const int nv = (int)c->views.size();
    views.assign(nv, PL::PlanView{});
    for (int v = 0; v < nv; ++v) {
        const HostView& hv = c->views[v];
        if (!hv.valid) continue;
        PL::PlanView& o = views[v];
        std::memcpy(o.campos, hv.campos, 12);
        std::memcpy(o.w2c, hv.w2c, 48);
        std::memcpy(o.proj0, hv.lv[0].proj, 36);
        o.inv0 = hv.lv[0].invproj[0];
        if (s.scale < (int)hv.lv.size()) { std::memcpy(o.proj_s, hv.lv[s.scale].proj, 36); o.inv_s = hv.lv[s.scale].invproj[0]; }
        o.w0 = hv.lv[0].w; o.h0 = hv.lv[0].h;
        o.valid = 1;
    }
    PL::PlanInput in = {};
    in.views = views.data();
    in.feat_pos = c->feat_pos.data();
    in.feat_off = c->feat_off.data(); in.feat_refs = c->feat_refs.data();
    in.vf_off = c->vf_off.data(); in.vf_ids = c->vf_ids.data();
    in.nv = nv; in.nf = (int)c->feat_off.size() - 1;
    in.dot_skip = PL::host_dot_skip(s.min_parallax);
    in.gvs_max = (int)s.global_vs_max;
    for (int i = 0; i < 3; ++i) { in.aabb_min[i] = s.aabb_min[i]; in.aabb_max[i] = s.aabb_max[i]; }
    return in;
}

// DMRecon::analyzeFeatures (dmrecon.cc:179-208) + GlobalViewSelection (global_view_selection.cc:17-101) on the host: the
// path of planning contexts, b200mvs_plan_views and the inspection calls, and what the device planner must equal.
// Its INTEGER result must match the reference bit for bit, so every float is produced by the reference's expression order:
// the geometry and the per-feature steps are plan_device.cuh's, shared with the device planner.  What is restructured is
// only WHEN things are computed:
//   * (feature - camera centre).normalized() is computed once per (view, feature) instead of inside every parallax()
//     call (mvs_tools.h:46-53) - same operations, same values;
//   * `if (plx < minParallax) score *= sqr(plx / 10)` (global_view_selection.cc:80-81,93-97) needs acos only when the
//     directions are nearly parallel: for dot < cos(minParallax + 0.05 deg) the branch is certainly not taken;
//   * the factor of a selected view s on (candidate i, feature k) does not change between rounds; multiplying by the
//     exact 1.0f of a not-taken branch cannot change a rounding, so only the factors != 1 are stored (ascending s,
//     the std::set iteration order) and re-multiplied each round;
//   * the (candidate, feature) records are laid out feature-major, the order the greedy loop walks them in.
std::vector<int> global_view_selection(const PL::PlanInput& in, float min_parallax, int ref)
{
    const int nv = in.nv;
    const PL::PlanView& rv = in.views[ref];
    // parallax factor of global_view_selection.cc:80-81 / :93-97 from two unit directions
    auto plx_factor = [&](const float* d1, const float* d2) { return PL::host_plx_factor(PL::dot3(d1, d2), in.dot_skip, min_parallax); };
    struct Extra { int k, view; float f; };       // a factor != 1 of selected view `view` on entry k of a candidate
    struct Cand {
        std::vector<float> base;         // per entry k (= SingleView::featInd order): parallax-with-ref and resolution terms (:78-87)
        std::vector<int> feat;           // per entry k: local index of its feature
        std::vector<int> ent;            // per entry k: its index in the feature-major arrays below
        std::vector<Extra> extra;        // ascending (k, view): the std::set iteration order of :90
        std::vector<Extra> fresh;        // the factors of the view selected last, before they are merged into `extra`
        float benefit = 0.f;             // benefitFromView of the last evaluation
        bool dirty = true;
    };
    std::vector<Cand> cand(nv);
    std::vector<char> avail(nv, 1);
    avail[ref] = 0;
    for (int v = 0; v < nv; ++v) if (!in.views[v].valid) avail[v] = 0;
    // Feature-major entries: everything the candidates hold about ONE feature is contiguous, because that is how the greedy
    // loop walks it - "which candidates see a feature the new view sees" is SingleView::seesFeature (single_view.h:166-174)
    // turned around.  A candidate's entries keep the order of the reference's featInd (ascending feature, then refs order).
    std::vector<int> foff(1, 0), ecand, ek;
    std::vector<float> edir;
    // the features with contains_view_id(refViewNr), ascending (dmrecon.cc:186-188)
    for (int t = in.vf_off[ref]; t < in.vf_off[ref + 1]; ++t) {
        const int fi = in.vf_ids[t];
        const float* p = in.feat_pos + 3 * (size_t)fi;
        if (!PL::seen_in_box(in, rv, p)) continue;
        const int fl = (int)foff.size() - 1;
        bool have_ref = false;
        float dr[3] = {0.f, 0.f, 0.f}, mfp = 0.f;
        for (int r = in.feat_off[fi]; r < in.feat_off[fi + 1]; ++r) {
            const int vid = in.feat_refs[r];
            if (vid < 0 || vid >= nv || !avail[vid]) continue;            // the reference view itself is never a candidate
            const PL::PlanView& tv = in.views[vid];
            if (!PL::point_in_frustum(tv, p)) continue;
            if (!have_ref) { PL::unit_dir(rv, p, dr); mfp = PL::foot_print(rv, rv.inv_s, p); have_ref = true; }
            Cand& C = cand[vid];
            const int e = (int)ecand.size();
            float d[3];
            PL::unit_dir(tv, p, d);
            float score = 1.f;
            score *= plx_factor(dr, d);
            score *= PL::footprint_ratio(tv, p, mfp);
            ecand.push_back(vid); ek.push_back((int)C.base.size());
            edir.push_back(d[0]); edir.push_back(d[1]); edir.push_back(d[2]);
            C.base.push_back(score); C.feat.push_back(fl); C.ent.push_back(e);
        }
        if ((int)ecand.size() > foff.back()) foff.push_back((int)ecand.size());
    }
    std::vector<int> selected;
    std::vector<Extra> merged;
    bool found = true;
    while (found && (int)selected.size() < in.gvs_max) {
        float maxBenefit = 0.f;
        int maxView = 0;
        found = false;
        for (int i = 0; i < nv; ++i) {
            if (!avail[i]) continue;
            Cand& C = cand[i];
            if (C.dirty) {
                // recomputed only when a factor of this candidate changed since the last round: the same operations on
                // the same operands give the same float, so caching cannot change the result
                float benefit = 0;
                const size_t n = C.base.size();
                size_t x = 0;
                for (size_t k = 0; k < n; ++k) {
                    float score = C.base[k];
                    for (; x < C.extra.size() && C.extra[x].k == (int)k; ++x) score *= C.extra[x].f;
                    benefit += score;
                }
                C.benefit = benefit;
                C.dirty = false;
            }
            if (C.benefit > maxBenefit) { maxBenefit = C.benefit; maxView = i; found = true; }
        }
        if (!found) break;
        selected.insert(std::upper_bound(selected.begin(), selected.end(), maxView), maxView);
        avail[maxView] = 0;
        // fold the new view's factors into every remaining candidate.  Only (candidate, feature) entries whose feature
        // the new view sees can change (global_view_selection.cc:90-92).
        const Cand& S = cand[maxView];
        for (size_t ks = 0; ks < S.base.size(); ++ks) {
            const int fl = S.feat[ks];
            if (ks > 0 && S.feat[ks - 1] == fl) continue;              // seesFeature() is a predicate: a duplicate adds nothing
            const float* ds = &edir[3 * (size_t)S.ent[ks]];
            for (int e = foff[fl]; e < foff[fl + 1]; ++e) {
                const int i = ecand[e];
                if (!avail[i]) continue;
                const float f = plx_factor(ds, &edir[3 * (size_t)e]);
                if (f != 1.f) cand[i].fresh.push_back(Extra{ek[e], maxView, f});      // arrives with ascending k
            }
        }
        for (int i = 0; i < nv; ++i) {
            Cand& C = cand[i];
            if (C.fresh.empty()) continue;
            merged.resize(C.extra.size() + C.fresh.size());
            std::merge(C.extra.begin(), C.extra.end(), C.fresh.begin(), C.fresh.end(), merged.begin(),
                       [](const Extra& a, const Extra& b) { return a.k != b.k ? a.k < b.k : a.view < b.view; });
            C.extra.swap(merged);
            C.fresh.clear();
            C.dirty = true;
        }
    }
    return selected;
}

// Host threads for the per-view host phase (global view selection + seed lists).  One process per GPU on a shared box
// should not start hardware_concurrency() threads each: B200MVS_HOST_THREADS caps it (bench.py sets cores / (2 * ranks)).
int host_threads(int n_jobs)
{
    int cap = (int)std::thread::hardware_concurrency();
    if (const char* e = std::getenv("B200MVS_HOST_THREADS")) { const int v = std::atoi(e); if (v > 0) cap = v; }
    return std::max(1, std::min(n_jobs, cap));
}

// The feature loop of DMRecon::processFeatures (dmrecon.cc:258-292): which features seed, at which pixel, with
// which initial depth.  The optimisation of the seeds runs on the device.
std::vector<PL::SeedOut> collect_seeds(const PL::PlanInput& in, int ref, const std::vector<int>& gsel)
{
    const PL::PlanView& rv = in.views[ref];
    std::vector<PL::SeedOut> out;
    // "use feature if visible in reference view or at least one neighboring view" (dmrecon.cc:260-276), in feature order
    std::vector<char> wanted(in.nf, 0);
    auto want = [&](int v) { for (int t = in.vf_off[v]; t < in.vf_off[v + 1]; ++t) wanted[in.vf_ids[t]] = 1; };
    want(ref);
    for (int g : gsel) want(g);
    for (int fi = 0; fi < in.nf; ++fi) {
        const float* p = in.feat_pos + 3 * (size_t)fi;
        if (!wanted[fi] || !PL::seen_in_box(in, rv, p)) continue;
        out.emplace_back();
        PL::seed_of(rv, p, out.back());
    }
    return out;
}

// One entry of a batch: a reference view reconstructed at one pyramid level.  Everything below the entry points reads
// an entry's facts from here; the batch's builder (check_batch, plan_batch) computes each of them once.
struct BatchEntry {
    int view = -1, level = 0;
    HostPlan plan;
    Workspace ws;                  // the entry's launch sizes; seeds = planned feature seeds + prior candidate bound
    std::vector<int> need;         // the views whose pyramids it reads: itself and its global selection, ascending
};

// The entries of one call, with its settings and progress records (progress[j] belongs to e[j]; may be null)
struct Batch {
    b200mvs_settings s = {};
    std::vector<BatchEntry> e;
    b200mvs_progress* progress = nullptr;
    int failed = -1;               // the entry whose view the call names in failed_view; -1: none
    // the one writer of an entry point's failed_view, once the call's entries are being checked; returns rc
    int report(int rc, int32_t* failed_view) const { if (failed_view) *failed_view = failed >= 0 ? e[failed].view : -1; return rc; }
};

// The host phase of B.e[j] for every j in `todo` into its plan: analyzeFeatures + globalViewSelection + seed list
// (dmrecon.cc:179-292), with `s` the settings at the entries' level.  The per-view host work is independent (the
// reference runs whole DMRecons on OpenMP threads, apps/dmrecon/dmrecon.cc:285): spread it over host threads.
void make_plans(const PL::PlanInput& in, const b200mvs_settings& s, Batch& B, const std::vector<int>& todo)
{
    std::atomic<size_t> next_job(0);
    auto worker = [&]() {
        for (;;) {
            const size_t k = next_job.fetch_add(1);
            if (k >= todo.size()) break;
            const int j = todo[k];
            HostPlan& p = B.e[j].plan;
            p.settings = s;
            p.gsel = global_view_selection(in, s.min_parallax, B.e[j].view);
            if (p.gsel.empty()) continue;
            if (B.progress) B.progress[j].status = 2;
            p.seeds = collect_seeds(in, B.e[j].view, p.gsel);
        }
    };
    const int n_threads = host_threads((int)todo.size());
    std::vector<std::thread> pool;
    for (int t = 1; t < n_threads; ++t) pool.emplace_back(worker);
    worker();
    for (std::thread& t : pool) t.join();
}

// The plan b200mvs_plan_views prepared for view `ref` under these settings, or nullptr.  The caller holds plan_mtx.
HostPlan* find_plan(b200mvs_ctx* c, const b200mvs_settings& s, int ref)
{
    auto it = c->plans.find(ref);
    return it != c->plans.end() && std::memcmp(&it->second.settings, &s, sizeof(s)) == 0 ? &it->second : nullptr;
}

// ------------------------------------------------------------------------------------------------
// kernels: image import + pyramid
// ------------------------------------------------------------------------------------------------
// `undistorted` bytes -> RGBX8 (alpha dropped, grey expanded: image_pyramid.cc:65-73), read through the source's layout
template <bool Planar>
__global__ void k_import_rgb(const b200mvs_undistort::Src src, int w, int h, int ch, uchar4* __restrict__ dst, int pitch)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const uint8_t* p = b200mvs_undistort::texel<Planar>(src, ch, x, y);
    uchar4 o;
    if (ch >= 3) {
        o.x = p[0];
        o.y = p[b200mvs_undistort::channel_offset<Planar>(src, 1)];
        o.z = p[b200mvs_undistort::channel_offset<Planar>(src, 2)];
    } else {
        o.x = o.y = o.z = p[0];
    }
    o.w = 255;
    dst[(size_t)y * pitch + x] = o;
}

// `original` bytes -> RGBX8 of their image_undistort_k2k4 (undistort.cuh), converted as k_import_rgb converts
template <bool Planar>
__global__ void k_undistort_k2k4(const b200mvs_undistort::Src src, const b200mvs_undistort::Params P, uchar4* __restrict__ dst, int pitch)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= P.w || y >= P.h) return;
    const uint32_t p = b200mvs_undistort::undistort_px<Planar>(P, src, x, y);
    uchar4 o;
    if (P.ch >= 3) { o.x = p & 0xFF; o.y = (p >> 8) & 0xFF; o.z = (p >> 16) & 0xFF; }
    else           { o.x = o.y = o.z = p & 0xFF; }
    o.w = 255;
    dst[(size_t)y * pitch + x] = o;
}

// mve::image::rescale_half_size_gaussian<uint8_t>(img, 1.f) (image_tools.h:617-694) with Accum<uint8>
// (accum.h:117-170): same 16 taps in the same order, fp32 accumulate, true division, math::round.
// Bit-exact with the reference (tests/test_gpu_parity.py::test_pyramid_bit_exact); products and sums are kept un-fused on purpose.
__global__ void k_half_gaussian(const uchar4* __restrict__ in, int iw, int ih, int ipitch,
                                uchar4* __restrict__ out, int ow, int oh, int opitch,
                                float w1, float w2, float w3)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= ow || y >= oh) return;
    const int y2 = y * 2, x2 = x * 2;
    const int ys[4] = {max(0, y2 - 1), y2, min(ih - 1, y2 + 1), min(ih - 1, y2 + 2)};
    const int xs[4] = {max(0, x2 - 1), x2, min(iw - 1, x2 + 1), min(iw - 1, x2 + 2)};
    const float wr[4][4] = {{w3, w2, w2, w3}, {w2, w1, w1, w2}, {w2, w1, w1, w2}, {w3, w2, w2, w3}};
    float v0 = 0.f, v1 = 0.f, v2 = 0.f, ws = 0.f;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const uchar4* row = in + (size_t)ys[r] * ipitch;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uchar4 t = row[xs[k]];
            v0 = __fadd_rn(v0, __fmul_rn((float)t.x, wr[r][k]));
            v1 = __fadd_rn(v1, __fmul_rn((float)t.y, wr[r][k]));
            v2 = __fadd_rn(v2, __fmul_rn((float)t.z, wr[r][k]));
            ws = __fadd_rn(ws, wr[r][k]);
        }
    }
    const float q0 = __fdiv_rn(v0, ws), q1 = __fdiv_rn(v1, ws), q2 = __fdiv_rn(v2, ws);
    uchar4 o;
    o.x = (unsigned char)(q0 > 0.f ? floorf(q0 + 0.5f) : ceilf(q0 - 0.5f));
    o.y = (unsigned char)(q1 > 0.f ? floorf(q1 + 0.5f) : ceilf(q1 - 0.5f));
    o.z = (unsigned char)(q2 > 0.f ? floorf(q2 + 0.5f) : ceilf(q2 - 0.5f));
    o.w = 255;
    out[(size_t)y * opitch + x] = o;
}

// The bilinear footprint of a sample at (x + fx, y + fy) is the 2x2 block {(x,y), (x+1,y), (x,y+1), (x+1,y+1)}
// (mvs_tools.cc:110-124): stored contiguously per (x, y) it is ONE aligned 16-byte load instead of four 4-byte ones.
__global__ void k_make_quads(const uchar4* __restrict__ img, int w, int h, int pitch, uint4* __restrict__ quad)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const int x1 = min(x + 1, w - 1), y1 = min(y + 1, h - 1);
    const unsigned* p = reinterpret_cast<const unsigned*>(img);
    uint4 q;
    q.x = p[(size_t)y * pitch + x]; q.y = p[(size_t)y * pitch + x1];
    q.z = p[(size_t)y1 * pitch + x]; q.w = p[(size_t)y1 * pitch + x1];
    quad[(size_t)y * pitch + x] = q;
}

__global__ void k_export_rgb(const uchar4* __restrict__ src, int w, int h, int pitch, uint8_t* __restrict__ dst)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const uchar4 t = src[(size_t)y * pitch + x];
    uint8_t* p = dst + ((size_t)y * w + x) * 3;
    p[0] = t.x; p[1] = t.y; p[2] = t.z;
}

// The view ids of the four slots of `word` under a job's slot -> id table gview[0, n_global), -1 for an empty slot; returns
// how many are set.  The host maps, b200mvs_optimize_patches and k_slots_to_ids all map slots through this one function.
__host__ __device__ inline int slots_to_ids(const int* gview, int n_global, unsigned word, int32_t ids[4])
{
    int n = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const unsigned sl = (word >> (8 * k)) & 0xFF;
        ids[k] = sl < (unsigned)n_global ? gview[sl] : -1;
        n += ids[k] >= 0;
    }
    return n;
}

// view_ids of one reference view in device memory (b200mvs_reconstruct_device): 4 x int32 per pixel from the job's slot
// words.  `out` need only be 4-byte aligned; a 16-byte-aligned one is written one pixel per store.
__global__ void k_slots_to_ids(const JobParams job, int32_t* __restrict__ out, bool aligned16)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= (size_t)job.W * job.H) return;
    int32_t ids[4];
    slots_to_ids(job.gview, job.n_global, __ldg(job.slots + p), ids);
    int32_t* o = out + 4 * p;
    if (aligned16) *reinterpret_cast<int4*>(o) = make_int4(ids[0], ids[1], ids[2], ids[3]);
    else { o[0] = ids[0]; o[1] = ids[1]; o[2] = ids[2]; o[3] = ids[3]; }
}

// Reconstruction masks (b200mvs_set_view_mask).  For the whole frontier launch a background pixel holds conf = +inf, which
// no confidence (<= 1) passes: the stale test drops an entry of it, the commit test (old < conf) never writes it and the
// push rule (c < conf - 0.05 || c == 0) never queues it, in k_frontier and k_frontier_resume alike.  `bg` has one byte per
// pixel of the batch, nonzero = background; it lies in scratch map memory and is cleared as it is read.
__global__ void k_mask_background(float* __restrict__ conf, unsigned char* __restrict__ bg, size_t n)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n || !bg[p]) return;
    bg[p] = 0;
    conf[p] = INFINITY;
}
// The bytes of `bg` for one view's W x H map from its device mask (b200mvs_set_view_mask_device), as mark_background
// makes them from a host mask
__global__ void k_mark_background(const uint8_t* __restrict__ mask, int mw, int mh, int W, int H, unsigned char* __restrict__ bg)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= W || y >= H) return;
    bg[(size_t)y * W + x] = mask[(size_t)mask_coord(y, H, mh) * mw + mask_coord(x, W, mw)] == 0;
}
// The device mask of one view for k_seed_background, with the size of the view's map
struct SeedMask { const uint8_t* mask; int mw, mh, W, H; };
// bg[i] = whether seed i, pixel (x, y) of view `view` of seeds[i] = (x, y, view, -), lies on a background pixel; a seed
// outside the map does not (background())
__global__ void k_seed_background(const SeedMask* __restrict__ views, const int4* __restrict__ seeds, size_t n, unsigned char* __restrict__ bg)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int4 q = seeds[i];
    const SeedMask V = views[q.z];
    bg[i] = q.x >= 0 && q.y >= 0 && q.x < V.W && q.y < V.H &&
            V.mask[(size_t)mask_coord(q.y, V.H, V.mh) * V.mw + mask_coord(q.x, V.W, V.mw)] == 0;
}
// The prior seeds of one entry (b200mvs_set_view_prior): candidate c = (i, k) of the nx x ny grid is pixel
// (2 + stride i, 2 + stride k) of the entry's W x H map; it reads prior pixel (mask_coord(x, W, pw), mask_coord(y, H, ph))
// and becomes a seed when that depth is finite and > 0 and the pixel is not background (conf = +inf after
// k_mask_background).  Seeds are appended at out[*cursor] in whatever order the atomic gives.  That order cannot change a
// map: every prior seed comes after the feature seeds of the launch, and the prior seeds of one entry lie on distinct
// pixels, so the seed round's per-pixel rule (most confident first, then the earlier seed) resolves them alike in any order.
// A seed's dz and local views come from the prior's dz and id maps where they exist (prior_seed_state with the job's
// global selection and N = nr_recon_neighbors), else it has dz 0 and no local views.
__global__ void k_prior_seeds(const float* __restrict__ prior, const float2* __restrict__ prior_dz, const int4* __restrict__ prior_ids,
                              int pw, int ph, int stride, int nx, size_t n, const JobParams J, unsigned N, int job,
                              Entry* __restrict__ out, unsigned long long* __restrict__ cursor)
{
    const size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    const int x = 2 + stride * (int)(c % nx), y = 2 + stride * (int)(c / nx);
    const size_t q = (size_t)mask_coord(y, J.H, ph) * pw + mask_coord(x, J.W, pw);
    const float d = __ldg(prior + q);
    if (!(d > 0.f) || isinf(d) || isinf(J.conf[(size_t)y * J.W + x])) return;
    PriorPixel px = {prior_dz != nullptr, prior_ids != nullptr, {0.f, 0.f}, {-1, -1, -1, -1}};
    if (prior_dz) { const float2 t = __ldg(prior_dz + q); px.dz[0] = t.x; px.dz[1] = t.y; }
    if (prior_ids) { const int4 t = __ldg(prior_ids + q); px.ids[0] = t.x; px.ids[1] = t.y; px.ids[2] = t.z; px.ids[3] = t.w; }
    const PriorState s = prior_seed_state(px, pw, ph, J.W, J.H, J.gview, J.n_global, N);
    out[atomicAdd(cursor, 1ull)] = make_entry(pack_xy(x, y), job, 4, 0.f, d, s.dzI, s.dzJ, s.slots);
}
// after the launch: background pixels leave the device as unfilled ones, conf = 0
__global__ void k_unmask_background(float* __restrict__ conf, size_t n)
{
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n && isinf(conf[p])) conf[p] = 0.f;
}

// ------------------------------------------------------------------------------------------------
// kernels: patch optimisation + frontier
// ------------------------------------------------------------------------------------------------
// OPT_TPB, the threads per CTA of the patch-optimisation kernels, is set in patch_thread.cuh (it lays out shared memory)
#ifndef OPT_MIN_BLOCKS
#define OPT_MIN_BLOCKS 1     // CTAs per SM: registers per thread <= 65536 / (OPT_MIN_BLOCKS * OPT_TPB) = 170; shared memory 189 KB per CTA
#endif
constexpr int OPT_WARPS = OPT_TPB / 32;
using PatchT = b200mvs::PatchW;    // one warp per patch (latency: small rounds)
using PatchT1 = b200mvs::PatchT;   // one thread per patch (throughput: large rounds)
// dynamic shared memory of the kernels that optimise patches: the lane-replicated sRGB table, then one PatchT1 per thread,
// then the master-texel table of the PatchT1s (PatchT1::mt_tab).
// The state of a thread's patch is live across the whole sample loop, which needs every register there is: left to the
// compiler it is spilled to local memory (~100 slots x 128 B per warp - more than L1 holds, so every reload in the per-view
// set-up and tear-down was an L2 round trip: 19 % of the kernel's time in ncu's stall samples).  In shared memory a reload
// costs a fixed ~30 cycles.  64 KB + 384 x 232 B + 37.5 KB = 193 024 B: with the 8 B of static shared memory and the 1 KB
// the system reserves per CTA this is the 196 KB carve-out, which leaves 60 KB of L1 for the texels.  The next carve-out
// (228 KB, 28 KB of L1) costs far more than any table it could hold: with 75 KB of unused shared memory added to the
// layout without master texels, the C2 step took 169 ms instead of 117 ms (H100 80GB HBM3, 700 W; DESIGN.md §6).
constexpr size_t OPT_LUT_BYTES = sizeof(float) * (256 * LUT_STRIDE);
constexpr size_t OPT_SMEM_BYTES = OPT_LUT_BYTES + (size_t)OPT_TPB * sizeof(PatchT1) + PatchT1::MT_BYTES;
static_assert(OPT_SMEM_BYTES + 8 + 1024 <= 196 * 1024, "the patch kernels' shared memory must stay within the 196 KB carve-out");
__device__ __forceinline__ PatchT1& thread_patch(float* smem)
{
    return reinterpret_cast<PatchT1*>(reinterpret_cast<unsigned char*>(smem) + OPT_LUT_BYTES)[threadIdx.x];
}

__device__ __forceinline__ Entry load_entry(const Entry* p)       // lists are rewritten by other SMs every round: bypass L1
{
    const int4 a = __ldcg(reinterpret_cast<const int4*>(p));
    const int4 b = __ldcg(reinterpret_cast<const int4*>(p) + 1);
    Entry e;
    e.xy = a.x; e.jobdir = a.y; e.conf = __int_as_float(a.z); e.depth = __int_as_float(a.w);
    e.dzI = __int_as_float(b.x); e.dzJ = __int_as_float(b.y); e.slots = (unsigned)b.z; e.pad = b.w;
    return e;
}

__device__ __forceinline__ PatchIn patch_in(const Entry& e)
{
    PatchIn pi;
    pi.x = entry_x(e); pi.y = entry_y(e);
    pi.depth = e.depth; pi.dzI = e.dzI; pi.dzJ = e.dzJ; pi.slots = e.slots;
    return pi;
}

__device__ __forceinline__ unsigned long long global_timer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// The PatchOptimizations of list[0..n): every warp takes entries through the ticket counter until none is left; a warp that
// finishes one fetches the next at once.  PatchOptimization ctor + doAutoOptimization + computeConfidence per entry.
__device__ __forceinline__ void optimise_entries(PatchT& p, const Entry* list, PatchOut* res, unsigned long long n,
                                                 unsigned long long* ticket, const JobParams* jobs, unsigned long long* counters)
{
    unsigned opts = 0u;
    for (;;) {
        unsigned long long w = 0ull;
        if (p.lane == 0) w = atomicAdd(ticket, 1ull);
        w = __shfl_sync(FULL, w, 0);
        if (w >= n) break;
        const Entry e = load_entry(&list[w]);
        p.begin(&jobs[entry_job(e)], patch_in(e));
        ++opts;
        while (!p.step()) {}
        PatchOut po;
        p.finish(po);
        if (p.lane == 0) res[w] = po;
    }
    if (p.lane == 0 && opts) {
        atomicAdd(&counters[C_SETS], (unsigned long long)p.n_sets);
        atomicAdd(&counters[C_OPTS], (unsigned long long)opts);
        p.n_sets = 0u;
    }
}

// The same for LARGE lists: one thread per entry (patch_thread.cuh).  Lanes that need an entry take consecutive tickets with
// one atomic per converged subset of the warp; a lane that finishes fetches its next entry at once and meets the other
// lanes of its warp again at the pass() call site.
__device__ __forceinline__ void optimise_entries_t(PatchT1& p, const Entry* list, PatchOut* res, unsigned long long n,
                                                   unsigned long long* ticket, const JobParams* jobs, unsigned long long* counters)
{
    const int lane = threadIdx.x & 31;
    bool have = false;
    unsigned long long idx = 0ull;
    unsigned opts = 0u;
    for (;;) {
        if (!have) {
            const unsigned act = __activemask();
            const int leader = __ffs(act) - 1;
            unsigned long long base = 0ull;
            if (lane == leader) base = atomicAdd(ticket, (unsigned long long)__popc(act));
            base = __shfl_sync(act, base, leader);
            const unsigned long long w = base + (unsigned long long)__popc(act & ((1u << lane) - 1u));
            if (w >= n) break;
            idx = w;
            const Entry e = load_entry(&list[w]);
            p.begin(&jobs[entry_job(e)], patch_in(e));
            have = true;
            ++opts;
        }
        if (p.step()) {
            PatchOut po;
            p.finish(po);
            res[idx] = po;
            have = false;
        }
    }
    if (opts) {
        atomicAdd(&counters[C_SETS], (unsigned long long)p.n_sets);
        atomicAdd(&counters[C_OPTS], (unsigned long long)opts);
        p.n_sets = 0u;
    }
}

#ifndef OPT_THREAD_MIN
#define OPT_THREAD_MIN 8192    // lists at least this long are optimised one thread per patch, shorter ones one warp per patch
#endif

// A batch of independent PatchOptimizations (b200mvs_optimize_patches).  mode: 0 = by list length, 1 = one warp per patch,
// 2 = one thread per patch.
__global__ void __launch_bounds__(OPT_TPB, OPT_MIN_BLOCKS)
k_optimize(const Entry* __restrict__ in, PatchOut* __restrict__ out, int n, int mode,
           const DevSettings* __restrict__ st, const JobParams* __restrict__ jobs, const ViewParams* __restrict__ views,
           const float* __restrict__ g_lut, unsigned long long* counters)
{
    extern __shared__ float smem[];
    for (int i = threadIdx.x; i < 256 * LUT_STRIDE; i += blockDim.x) smem[i] = g_lut[i / LUT_STRIDE];
    __syncthreads();
    if (mode == 2 || (mode == 0 && n >= OPT_THREAD_MIN)) {
        PatchT1& p = thread_patch(smem);
        bind_thread(p, st, views, smem, (int)threadIdx.x);
        optimise_entries_t(p, in, out, (unsigned long long)n, &counters[C_TICKET], jobs, counters);
    } else {
        PatchT p;
        bind_thread(p, st, views, smem, (int)threadIdx.x);
        optimise_entries(p, in, out, (unsigned long long)n, &counters[C_TICKET], jobs, counters);
    }
}

__device__ __forceinline__ unsigned long long entry_key(const Entry& e)
{
    // larger confidence first, then smaller direction code (DESIGN.md "Frontier schedule")
    return ((unsigned long long)__float_as_uint(e.conf) << 8) | (unsigned long long)(7 - entry_dir(e));
}

// ---- the whole region growing of a batch in ONE persistent kernel -------------------------------------------------------
// processFeatures + processQueue (dmrecon.cc:244-434) as frontier rounds (DESIGN.md "Frontier schedule").  The grid is
// launched cooperatively with exactly as many CTAs as fit on the chip; the phases of a round are separated by a grid-wide
// barrier instead of kernel boundaries, the patch optimisations of a round are handed out warp by warp through a ticket
// counter, and the host is not involved until the queue is empty: progress goes out and the cancel flag comes in through
// mapped pinned memory once per round (Progress, progress.h:27-43; dmrecon.cc:353).
struct FrontierParams {
    Entry* list[2];
    Entry* run;
    Entry* run2;                                // the round's winners grouped by 16x16 tile (large rounds)
    unsigned* tile_cnt;                         // [n_tiles] entries per tile, zero between rounds
    unsigned long long* tile_off;               // [n_tiles] start of the tile's segment in run2
    long long n_tiles;
    PatchOut* res;
    unsigned char* written;
    unsigned long long cap;
    int n_seeds, n_jobs;
    const DevSettings* st;
    const JobParams* jobs;
    const ViewParams* views;
    const float* lut;
    unsigned long long* counters;               // Counter + filled per job
    FrontierCtl* ctl;
    unsigned* hist;                             // [n_jobs][HIST_PER_JOB], zero on entry (only with a threshold)
    int* thr_bin;                               // [n_jobs]
    HostMirror* host;
    volatile unsigned long long* host_filled;   // [n_jobs], mapped
    volatile int* host_cancel_job;              // [n_jobs], mapped
    int* job_cancel;                            // [n_jobs], device copy refreshed every round
    long long thread_min;                       // a view with at least this many patches in a round runs them one thread per patch
    unsigned long long* job_run;                // [n_jobs] winners of the round per view
    int band_bins;                              // frontier_band in fine bins (0 = off)
    int topk;                                   // frontier_topk (0 = off)
    int first_list;                             // parity of the first round: 1 (the seed round), or after ST_GROW the
                                                // list the resumed round pushed into (n_seeds = 0)
};

__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p)
{
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
// All CTAs are co-resident (cooperative launch), so a monotone ticket counter is a barrier: the k-th generation is
// complete when the counter reaches k * gridDim.x.  The wait polls with a RELAXED load: an acquire load in the loop
// (ld.acquire = LDG + CCTL.IVALL) would invalidate the SM's L1 on every poll and starve the CTAs of the same SM that are
// still sampling; one fence after the wait orders the phase.  Data that
// other SMs write during the kernel is read with ld.cg everywhere, so no L1 invalidation is needed for correctness.
__device__ __forceinline__ void grid_barrier(unsigned long long* bar)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long nb = gridDim.x;
        const unsigned long long t = atomicAdd(bar, 1ull);
        const unsigned long long target = (t / nb + 1ull) * nb;
        while (ld_relaxed_u64(bar) < target) __nanosleep(64);
        __threadfence();
    }
    __syncthreads();
}
__device__ __forceinline__ int conf_bin(float c)
{
    const int b = (int)(c * (float)HIST_FINE);
    return b < 0 ? 0 : (b > HIST_FINE - 1 ? HIST_FINE - 1 : b);
}
__device__ __forceinline__ PatchOut load_result(const PatchOut* p)  // written by another SM in the optimise phase: bypass L1
{
    static_assert(sizeof(PatchOut) == 40, "PatchOut layout");
    const int2* q = reinterpret_cast<const int2*>(p);
    const int2 a = __ldcg(q), b = __ldcg(q + 1), c = __ldcg(q + 2), d = __ldcg(q + 3), e = __ldcg(q + 4);
    PatchOut r;
    r.conf = __int_as_float(a.x); r.depth = __int_as_float(a.y); r.dzI = __int_as_float(b.x); r.dzJ = __int_as_float(b.y);
    r.nx = __int_as_float(c.x); r.ny = __int_as_float(c.y); r.nz = __int_as_float(d.x); r.slots = (unsigned)d.y;
    r.iterations = e.x; r.flags = e.y;
    return r;
}
// Warp-aggregated slot allocation: the lanes of a warp that reach this point together take consecutive slots with ONE atomic
// (the queue bookkeeping appends ~20 M entries per step to three counters; one same-address atomic per entry cost ~20 ms).
__device__ __forceinline__ unsigned long long take_slot(unsigned long long* counter)
{
    const unsigned m = __activemask();
    const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
    unsigned long long base = 0ull;
    if (lane == leader) base = atomicAdd(counter, (unsigned long long)__popc(m));
    base = __shfl_sync(m, base, leader);
    return base + (unsigned long long)__popc(m & ((1u << lane) - 1u));
}
// the same for a counter per job: lanes with the same job share one atomic
__device__ __forceinline__ void count_for_job(unsigned long long* per_job, int j)
{
    const unsigned m = __match_any_sync(__activemask(), j);
    if ((int)(threadIdx.x & 31) == __ffs(m) - 1) atomicAdd(&per_job[j], (unsigned long long)__popc(m));
}
__device__ __forceinline__ void push_entry(const FrontierParams& P, int q, const Entry& o)
{
    const unsigned long long pos = take_slot(&P.ctl->nlist[q]);
    if (pos < P.cap) P.list[q][pos] = o; else P.counters[C_OVERFLOW] = 1ull;
}
__device__ __forceinline__ void write_pixel(const JobParams& J, int idx, const PatchOut& r)
{
    J.depth[idx] = r.depth;
    J.conf[idx] = r.conf;
    J.dz[2 * idx] = r.dzI; J.dz[2 * idx + 1] = r.dzJ;
    J.normal[3 * idx] = r.nx; J.normal[3 * idx + 1] = r.ny; J.normal[3 * idx + 2] = r.nz;
    J.slots[idx] = r.slots;
}

// Eligibility threshold of one job from its confidence histogram (one warp).  topk: the largest bin t such that at least
// `topk` entries have bin >= t (0 when there are fewer); band: (highest non-empty bin) - band_bins.  Both: the larger.
__device__ __forceinline__ int threshold_of(const unsigned* hist, int lane, int band_bins, int topk)
{
    const unsigned* coarse = hist + HIST_FINE;
    int t_top = 0, t_band = 0;
    // coarse scan, descending: lane l looks at coarse bins 63 - l and 31 - l
    const unsigned c_hi = __ldcg(&coarse[63 - lane]), c_lo = __ldcg(&coarse[31 - lane]);
    if (band_bins > 0) {
        const unsigned m_hi = __ballot_sync(FULL, c_hi != 0u), m_lo = __ballot_sync(FULL, c_lo != 0u);
        int cb = -1;
        if (m_hi) cb = 63 - (__ffs(m_hi) - 1); else if (m_lo) cb = 31 - (__ffs(m_lo) - 1);
        if (cb >= 0) {
            int top = -1;
            for (int q = 3; q >= 0 && top < 0; --q) {
                const unsigned v = __ldcg(&hist[cb * 128 + q * 32 + (31 - lane)]);
                const unsigned m = __ballot_sync(FULL, v != 0u);
                if (m) top = cb * 128 + q * 32 + 31 - (__ffs(m) - 1);
            }
            t_band = top - band_bins;
            if (t_band < 0) t_band = 0;
        }
    }
    if (topk > 0) {
        unsigned need = (unsigned)topk, before = 0u;
        int cb = -1;
        for (int half = 0; half < 2 && cb < 0; ++half) {
            const unsigned c = half == 0 ? c_hi : c_lo;
            unsigned incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
            const unsigned m = __ballot_sync(FULL, before + incl >= need);
            if (m) {
                const int l = __ffs(m) - 1;
                cb = (half == 0 ? 63 : 31) - l;
                before += __shfl_sync(FULL, incl, l) - __shfl_sync(FULL, c, l);
            } else
                before += __shfl_sync(FULL, incl, 31);
        }
        if (cb >= 0) {
            for (int q = 3; q >= 0; --q) {
                const unsigned c = __ldcg(&hist[cb * 128 + q * 32 + (31 - lane)]);
                unsigned incl = c;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const unsigned v = __shfl_up_sync(FULL, incl, o); if (lane >= o) incl += v; }
                const unsigned m = __ballot_sync(FULL, before + incl >= need);
                if (m) { t_top = cb * 128 + q * 32 + 31 - (__ffs(m) - 1); break; }
                before += __shfl_sync(FULL, incl, 31);
            }
        }
    }
    return t_top > t_band ? t_top : t_band;
}

// Phase E of a round with parity p (dmrecon.cc:400-431): every committed pixel pushes its 4-neighbours into list[1 - p]
// under conf[nb] < conf - 0.05 || conf[nb] == 0; children inherit the parent's result as init and key.
__device__ __forceinline__ void push_neighbours(const FrontierParams& P, int p, const Entry* run_cur, unsigned long long n_run,
                                                size_t gtid, size_t gthreads)
{
    for (size_t i = gtid; i < n_run; i += gthreads) {
        if (!P.written[i]) continue;
        const Entry e = load_entry(&run_cur[i]);
        const PatchOut r = load_result(&P.res[i]);
        const int j = entry_job(e);
        const JobParams& J = P.jobs[j];
        const int x = entry_x(e), y = entry_y(e);
        const int nx[4] = {x - 1, x + 1, x, x};
        const int ny[4] = {y, y, y - 1, y + 1};
#pragma unroll
        for (int d = 0; d < 4; ++d) {
            const float c = __ldcg(&J.conf[ny[d] * J.W + nx[d]]);
            if (c < r.conf - 0.05f || c == 0.f) push_entry(P, 1 - p, child_entry(pack_xy(nx[d], ny[d]), j, d, r));
        }
    }
}

// After phase E of a round whose queue held n_cur entries (one thread): counts it, and returns whether the host cancelled
__device__ __forceinline__ bool end_round(FrontierCtl* ctl, unsigned long long n_cur, const HostMirror* host)
{
    ctl->rounds += 1ull;
    if (n_cur > ctl->peak) ctl->peak = n_cur;
    return host->cancel != 0;
}

// Phase E and the bookkeeping of the round k_frontier stopped with ST_GROW, after the host grew the frontier arrays and
// copied the round's carried entries, winners, results and `written` flags into them.  The next k_frontier launch goes on
// with the round after it.  A kernel of its own rather than an entry into the middle of k_frontier's round loop: that
// second entry changed the register allocation of the sample loop.
__global__ void k_frontier_resume(const FrontierParams P)
{
    FrontierCtl* const ctl = P.ctl;
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, gthreads = (size_t)gridDim.x * blockDim.x;
    push_neighbours(P, ctl->resume_p, ctl->resume_sorted ? P.run2 : P.run, ctl->resume_nrun, gtid, gthreads);
    if (gtid == 0) ctl->stop = end_round(ctl, ctl->resume_ncur, P.host) ? ST_CANCELLED : ST_RUN;
}

__global__ void __launch_bounds__(OPT_TPB, OPT_MIN_BLOCKS)
k_frontier(const FrontierParams P)
{
    extern __shared__ float smem[];
    for (int i = threadIdx.x; i < 256 * LUT_STRIDE; i += blockDim.x) smem[i] = P.lut[i / LUT_STRIDE];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, gthreads = (size_t)gridDim.x * blockDim.x;
    FrontierCtl* const ctl = P.ctl;
    unsigned long long* const cnt = P.counters;
    unsigned long long* const filled = cnt + C_NUM;
    const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
    const bool thresholded = P.band_bins > 0 || P.topk > 0;
    unsigned long long t_prev = lead ? global_timer_ns() : 0ull;
    unsigned long long n_bar = 0ull;
#define PHASE_END(ph) do { grid_barrier(&ctl->bar); ++n_bar; if (lead) { const unsigned long long t_ = global_timer_ns(); ctl->ns[ph] += t_ - t_prev; t_prev = t_; } } while (0)

    // ---- processQueue as frontier rounds (dmrecon.cc:334-434) ----
    // Round 0 optimises the seeds (processFeatures, dmrecon.cc:293-326: per pixel the most confident seed is committed, first
    // in feature order on ties), every later round one frontier.  The optimise phase has ONE call site so that the patch
    // optimisation code exists once in the instruction stream.
    int p = P.first_list;                                        // 1: the seed round pushes into list[0]
    bool seed_round = P.n_seeds > 0;
    for (;;) {
        unsigned long long n_cur = seed_round ? (unsigned long long)P.n_seeds : __ldcg(&ctl->nlist[p]);
        if (n_cur > P.cap) n_cur = P.cap;
        if (__ldcg(&ctl->stop) != ST_RUN || n_cur == 0ull) break;
        unsigned long long n_run = n_cur;
        if (!seed_round) {
        Entry* const cur = P.list[p];
        if (blockIdx.x == 0) {                                  // progress out (dmrecon.cc:355-364)
            if (threadIdx.x == 0) { P.host->round = ctl->rounds; P.host->queue = n_cur; }
            for (int j = threadIdx.x; j < P.n_jobs; j += blockDim.x) {
                P.host_filled[j] = __ldcg(&filled[j]);
                if (P.host_cancel_job[j]) P.job_cancel[j] = 1;   // this view's entries are dropped from now on (Progress::cancelled)
            }
        }
        // A: stale test (dmrecon.cc:371-373); without a threshold the per-pixel bid follows immediately
        for (size_t i = gtid; i < n_cur; i += gthreads) {
            const Entry e = load_entry(&cur[i]);
            const int j = entry_job(e);
            const JobParams& J = P.jobs[j];
            const int idx = pixel_of(J, e);
            if (__ldcg(&J.conf[idx]) > e.conf || __ldcg(&P.job_cancel[j])) { cur[i].jobdir = -1; continue; }
            if (!thresholded) atomicMax(&J.sel[idx], entry_key(e));
            else {
                const int b = conf_bin(e.conf);
                atomicAdd(&P.hist[(size_t)j * HIST_PER_JOB + b], 1u);
                atomicAdd(&P.hist[(size_t)j * HIST_PER_JOB + HIST_FINE + (b >> 7)], 1u);
            }
        }
        PHASE_END(PH_SELECT);
        if (thresholded) {
            // B: this round's eligibility threshold of every job, then the bids of the eligible entries
            for (int j = blockIdx.x * OPT_WARPS + (threadIdx.x >> 5); j < P.n_jobs; j += gridDim.x * OPT_WARPS) {
                const int t = threshold_of(P.hist + (size_t)j * HIST_PER_JOB, lane, P.band_bins, P.topk);
                if (lane == 0) P.thr_bin[j] = t;
            }
            PHASE_END(PH_THRESHOLD);
            for (size_t i = gtid; i < n_cur; i += gthreads) {
                const Entry e = load_entry(&cur[i]);
                if (e.jobdir == -1) continue;
                const int j = entry_job(e);
                if (conf_bin(e.conf) < __ldcg(&P.thr_bin[j])) { cur[i].jobdir = e.jobdir | DEFER_BIT; continue; }
                const JobParams& J = P.jobs[j];
                atomicMax(&J.sel[pixel_of(J, e)], entry_key(e));
            }
            PHASE_END(PH_THRESHOLD);
        }
        // C: the winning bid of each pixel runs, every other live entry is carried to the next round (the reference would
        // pop it later and apply the stale test then)
        for (size_t i = gtid; i < n_cur; i += gthreads) {
            Entry e = load_entry(&cur[i]);
            if (e.jobdir == -1) continue;
            if (e.jobdir & DEFER_BIT) { e.jobdir &= ~DEFER_BIT; push_entry(P, 1 - p, e); continue; }
            const JobParams& J = P.jobs[entry_job(e)];
            const int idx = pixel_of(J, e);
            const unsigned long long key = entry_key(e);
            if (__ldcg(&J.sel[idx]) == key && atomicCAS(&J.sel[idx], key, 0ull) == key) {
                const unsigned long long pos = take_slot(&ctl->nrun);
                P.run[pos] = e;
                count_for_job(P.job_run, entry_job(e));                                        // |run| <= n_cur <= capacity
            } else
                push_entry(P, 1 - p, e);
        }
        if (thresholded)
            for (size_t i = gtid; i < (size_t)P.n_jobs * HIST_PER_JOB; i += gthreads) P.hist[i] = 0u;
        PHASE_END(PH_PICK);
        n_run = __ldcg(&ctl->nrun);
        if (lead) { ctl->nlist[p] = 0ull; ctl->need = 0ull; }     // consumed; the round after the next pushes into it
        }
        // Which implementation optimises an entry is decided PER VIEW: a view with at least thread_min winners in this round runs
        // one thread per patch, a view with fewer one warp per patch.  The rule depends on the view alone, so its maps do not
        // depend on which other views share the batch (the two implementations differ in rounding).  The entries of the
        // "thread" views are grouped by 16x16-pixel tile first, so that the lanes of a warp and the warps of an SM sample
        // overlapping windows of the neighbour images (L1 / coalescing): count per tile, one atomic cursor bump per non-empty
        // tile, scatter; the entries of the other views follow behind them.
        unsigned long long n_thread = 0ull;
        const Entry* run_cur = P.run;
        if (!seed_round && P.n_tiles > 0) {
            __shared__ unsigned long long s_big;
            if (threadIdx.x == 0) s_big = 0ull;
            __syncthreads();
            unsigned long long mine = 0ull;
            for (int j = threadIdx.x; j < P.n_jobs; j += blockDim.x) {
                const unsigned long long c = __ldcg(&P.job_run[j]);
                if (c >= (unsigned long long)P.thread_min) mine += c;
            }
            if (mine) atomicAdd(&s_big, mine);
            __syncthreads();
            n_thread = s_big;
        }
        if (n_thread > 0ull) {
            for (size_t i = gtid; i < n_run; i += gthreads) {
                const Entry e = load_entry(&P.run[i]);
                const int j = entry_job(e);
                if (__ldcg(&P.job_run[j]) < (unsigned long long)P.thread_min) continue;
                atomicAdd(&P.tile_cnt[tile_of(P.jobs[j], e)], 1u);
            }
            PHASE_END(PH_SORT);
            for (size_t b = gtid; b < (size_t)P.n_tiles; b += gthreads) {
                const unsigned c = __ldcg(&P.tile_cnt[b]);
                if (c) P.tile_off[b] = atomicAdd(&ctl->sort_cursor, (unsigned long long)c);
            }
            PHASE_END(PH_SORT);
            for (size_t i = gtid; i < n_run; i += gthreads) {
                const Entry e = load_entry(&P.run[i]);
                const int j = entry_job(e);
                if (__ldcg(&P.job_run[j]) < (unsigned long long)P.thread_min) {
                    P.run2[n_thread + take_slot(&ctl->small_cursor)] = e;
                    continue;
                }
                const long long bin = tile_of(P.jobs[j], e);
                // the tile's counter is consumed downwards: it is zero again when the tile's last entry has been placed
                const unsigned k = atomicSub(&P.tile_cnt[bin], 1u) - 1u;
                P.run2[__ldcg(&P.tile_off[bin]) + k] = e;
            }
            PHASE_END(PH_SORT);
            run_cur = P.run2;
        }
        const bool by_thread = n_thread > 0ull;
        // the PatchOptimizations of the round
        if (by_thread) {
            PatchT1& pt = thread_patch(smem);
            bind_thread(pt, P.st, P.views, smem, (int)threadIdx.x);
            optimise_entries_t(pt, run_cur, P.res, n_thread, &ctl->ticket, P.jobs, cnt);
            __syncwarp();
        }
        if (n_run > n_thread) {
            PatchT pg;
            bind_thread(pg, P.st, P.views, smem, (int)threadIdx.x);
            optimise_entries(pg, run_cur + n_thread, P.res + n_thread, n_run - n_thread, by_thread ? &ctl->ticket2 : &ctl->ticket, P.jobs, cnt);
        }
        if (seed_round) {
            PHASE_END(PH_SEED);
            for (size_t i = gtid; i < (size_t)P.n_seeds; i += gthreads) {
                const float c = __ldcg(&P.res[i].conf);
                if (!(c > 0.f)) continue;
                atomicAdd(&cnt[C_SEED_OK], 1ull);
                const Entry e = load_entry(&run_cur[i]);
                const JobParams& J = P.jobs[entry_job(e)];
                atomicMax(&J.sel[pixel_of(J, e)], seed_key(c, i));
            }
            PHASE_END(PH_SELECT);
            for (size_t i = gtid; i < (size_t)P.n_seeds; i += gthreads) {
                const float c = __ldcg(&P.res[i].conf);
                if (!(c > 0.f)) continue;
                const Entry e = load_entry(&run_cur[i]);
                const int j = entry_job(e);
                const JobParams& J = P.jobs[j];
                const int idx = pixel_of(J, e);
                if (__ldcg(&J.sel[idx]) != seed_key(c, i)) continue;
                J.sel[idx] = 0ull;
                count_for_job(filled, j);
                const PatchOut r = load_result(&P.res[i]);
                write_pixel(J, idx, r);
                push_entry(P, 0, child_entry(e.xy, j, 4, r));
            }
            if (lead) ctl->ticket = 0ull;
            PHASE_END(PH_COMMIT);
            seed_round = false;
            p = 0;
            continue;
        }
        if (by_thread) PHASE_END(PH_OPT_THREAD); else PHASE_END(PH_OPT);
        // D: commit (dmrecon.cc:377-398).  One winner per pixel, so plain stores.
        for (size_t i = gtid; i < n_run; i += gthreads) {
            const Entry e = load_entry(&run_cur[i]);
            const PatchOut r = load_result(&P.res[i]);
            const int j = entry_job(e);
            const JobParams& J = P.jobs[j];
            const int idx = pixel_of(J, e);
            unsigned char w = 0;
            if (!(r.conf == 0.f)) {
                const float old = __ldcg(&J.conf[idx]);
                if (old <= 0.f) count_for_job(filled, j);
                if (old < r.conf) { write_pixel(J, idx, r); w = 1; }
            }
            P.written[i] = w;
            const unsigned act = __activemask(), wm = __ballot_sync(act, w);
            if (wm && lane == __ffs(act) - 1) atomicAdd(&ctl->need, 4ull * (unsigned long long)__popc(wm));
        }
        // The round's counters are reset here, in a phase in which no thread takes from them: a reset inside the phase that
        // uses a counter lets CTAs that are still working restart at slot 0 (lost and duplicated entries).
        if (lead) {
            ctl->nrun = 0ull; ctl->ticket = 0ull; ctl->ticket2 = 0ull; ctl->sort_cursor = 0ull; ctl->small_cursor = 0ull;
            atomicAdd(&ctl->need, __ldcg(&ctl->nlist[1 - p]));  // the carried entries: phase C ended, E has not begun
        }
        if (blockIdx.x == 0) for (int j = threadIdx.x; j < P.n_jobs; j += blockDim.x) P.job_run[j] = 0ull;
        PHASE_END(PH_COMMIT);
        // Checkpoint: E pushes at most 4 entries per written pixel behind the carried ones.  When that bound exceeds the
        // capacity, every thread stops here (all read the same `need`, which no phase before the next round's C changes);
        // the host grows the arrays and k_frontier_resume runs this round's E, so no entry is ever dropped.
        if (__ldcg(&ctl->need) > P.cap) {
            if (lead) {
                ctl->resume_p = p; ctl->resume_ncur = n_cur; ctl->resume_nrun = n_run; ctl->resume_sorted = run_cur == P.run2;
                ctl->stop = ST_GROW;
            }
            break;
        }
        // E: after ALL commits, push the 4-neighbours of every committed pixel (dmrecon.cc:400-431)
        push_neighbours(P, p, run_cur, n_run, gtid, gthreads);
        if (lead) {
            if (end_round(ctl, n_cur, P.host)) ctl->stop = ST_CANCELLED;
            else if (__ldcg(&cnt[C_OVERFLOW])) ctl->stop = ST_OVERFLOW;
        }
        PHASE_END(PH_EXPAND);
        p ^= 1;
    }
    if (lead) ctl->barriers += n_bar;
    if (blockIdx.x == 0) {
        if (threadIdx.x == 0) { P.host->round = ctl->rounds; P.host->queue = 0ull; }
        for (int j = threadIdx.x; j < P.n_jobs; j += blockDim.x) P.host_filled[j] = __ldcg(&filled[j]);
    }
#undef PHASE_END
}

// ------------------------------------------------------------------------------------------------
// host: view upload
// ------------------------------------------------------------------------------------------------
// ---- argument checks shared by the entry points ----
int require_device(const b200mvs_ctx* ctx)
{
    return ctx->device != B200MVS_DEVICE_NONE ? 0 : fail(B200MVS_ERR_CUDA, "planning context (B200MVS_DEVICE_NONE): no CUDA device, b200mvs has no CPU fallback");
}

// The arguments of the view-registration entry point `fn`; `image` is false when it takes an image and got NULL
int check_camera_args(const b200mvs_ctx* ctx, const char* fn, int id, bool image, int w, int h, const float* pp, const float* rot, const float* trans)
{
    if (id < 0 || id >= (int)ctx->views.size() || !image || w < 2 || h < 2 || !pp || !rot || !trans)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: bad arguments", fn);
    return 0;
}

// `scale`: whether s->scale is the level of the call (false for the *_levels entry points, which take one per entry)
int check_settings(const b200mvs_settings* s, bool scale = true)
{
    if (!s) return fail(B200MVS_ERR_INVALID_ARG, "settings is NULL");
    if (s->filter_width != 5)
        return fail(B200MVS_ERR_UNSUPPORTED, "filterWidth must be 5 (the reference hard-codes patchPoints[12], patch_sampler.cc:96)");
    if (scale && s->scale < 0) return fail(B200MVS_ERR_INVALID_ARG, "Invalid scale factor");
    if (s->nr_recon_neighbors < 1 || s->nr_recon_neighbors > B200MVS_MAX_LOCAL_VIEWS)
        return fail(B200MVS_ERR_UNSUPPORTED, "nrReconNeighbors must be in 1..%d", B200MVS_MAX_LOCAL_VIEWS);
    if (s->global_vs_max < 1 || s->global_vs_max > B200MVS_MAX_GLOBAL_VIEWS)
        return fail(B200MVS_ERR_UNSUPPORTED, "globalVSMax must be in 1..%d", B200MVS_MAX_GLOBAL_VIEWS);
    if (!(s->frontier_band >= 0.f) || s->frontier_band > 1.f)
        return fail(B200MVS_ERR_INVALID_ARG, "frontier_band must be in [0, 1]");
    return 0;
}

// A reference view reconstructed at pyramid level `scale` (dmrecon.cc:37-75): registered and with that level
int check_ref_view(const b200mvs_ctx* ctx, int scale, int ref)
{
    if (ref < 0 || ref >= (int)ctx->views.size()) return fail(B200MVS_ERR_INVALID_ARG, "Master view index out of bounds");
    if (!ctx->views[ref].valid) return fail(B200MVS_ERR_INVALID_ARG, "Invalid master view");
    if (scale < 0 || scale >= (int)ctx->views[ref].lv.size()) return fail(B200MVS_ERR_INVALID_ARG, "Invalid scale factor");
    return 0;
}

// The settings `s` at pyramid level `scale`: what a single-level call of an entry at that level is given
b200mvs_settings at_level(const b200mvs_settings& s, int scale)
{
    b200mvs_settings o = s;
    o.scale = scale;
    return o;
}

DevSettings to_dev(const b200mvs_settings& s)
{
    DevSettings d;
    d.min_ncc = s.min_ncc; d.min_parallax = s.min_parallax; d.accept_ncc = s.accept_ncc; d.min_refine_diff = s.min_refine_diff;
    d.max_iterations = s.max_iterations; d.nr_recon_neighbors = s.nr_recon_neighbors;
    d.scale = s.scale; d.use_color_scale = s.use_color_scale;
    return d;
}

// SingleView::create (single_view.cc:24-53): camera, image size and pyramid levels of view `id`.  A changed camera drops
// the prepared plans, and the view stays invalid until the caller builds its pyramid or marks it camera-only.
int set_camera(b200mvs_ctx* ctx, int id, int w, int h, float flen, float paspect, const float* pp, const float* rot, const float* trans)
{
    HostView& v = ctx->views[id];
    // Prepared plans depend on cameras and image sizes only: a re-upload of the same view with the same camera keeps them.
    // An unchanged camera keeps its host-side record untouched: b200mvs_plan_views of other views may be reading it right
    // now (cameras, calibrations and level sizes; never the device pointers build_pyramid writes).
    const bool same_camera = v.valid && !v.lv.empty() && v.w == w && v.h == h && v.flen == flen && v.paspect == paspect && v.pp[0] == pp[0] &&
                             v.pp[1] == pp[1] && std::memcmp(v.rot, rot, sizeof(v.rot)) == 0 && std::memcmp(v.trans, trans, sizeof(v.trans)) == 0;
    if (!same_camera) {
        { std::lock_guard<std::mutex> pl(ctx->plan_mtx); ctx->plans.clear(); }
        v.valid = false;
        v.has_image = false;
        v.w = w; v.h = h; v.flen = flen; v.paspect = paspect; v.pp[0] = pp[0]; v.pp[1] = pp[1];
        std::memcpy(v.rot, rot, sizeof(v.rot));
        std::memcpy(v.trans, trans, sizeof(v.trans));
        // CameraInfo::fill_camera_pos / fill_world_to_cam (camera.cc:34-39,61-67)
        v.campos[0] = -rot[0] * trans[0] - rot[3] * trans[1] - rot[6] * trans[2];
        v.campos[1] = -rot[1] * trans[0] - rot[4] * trans[1] - rot[7] * trans[2];
        v.campos[2] = -rot[2] * trans[0] - rot[5] * trans[1] - rot[8] * trans[2];
        for (int r = 0; r < 3; ++r) {
            v.w2c[4 * r] = rot[3 * r]; v.w2c[4 * r + 1] = rot[3 * r + 1]; v.w2c[4 * r + 2] = rot[3 * r + 2]; v.w2c[4 * r + 3] = trans[r];
        }
        // buildPyramid (image_pyramid.cc:22-53)
        v.lv.clear();
        float ppx = pp[0], ppy = pp[1];
        int cw = w, chh = h;
        auto push_level = [&]() {
            HostLevel L; L.w = cw; L.h = chh; L.pitch = (cw + 3) & ~3;
            fill_calibration(v.flen, v.paspect, ppx, ppy, (float)cw, (float)chh, L.proj, L.invproj);
            v.lv.push_back(L);
        };
        push_level();
        while (std::min(cw, chh) >= 30) {
            if (cw % 2 == 1) ppx = ppx * float(cw) / float(cw + 1);
            if (chh % 2 == 1) ppy = ppy * float(chh) / float(chh + 1);
            cw = (cw + 1) / 2; chh = (chh + 1) / 2;
            push_level();
        }
    }
    if ((int)v.lv.size() > MAX_LEVELS) return fail(B200MVS_ERR_UNSUPPORTED, "image too large: %d pyramid levels", (int)v.lv.size());
    return 0;
}

// loadColorImage (image_pyramid.cc:56-95): the pyramid of view `id` from a device image of the size set_camera registered,
// with `ch` channels laid out as `src` says (planar CHW when src.plane != 0, else HWC); with distortion coefficients, level 0
// is sfmrecon's undistortion of that image (sfmrecon.cc:425-437)
int build_pyramid(b200mvs_ctx* ctx, int id, const b200mvs_undistort::Src& src, int ch, cudaStream_t stream)
{
    HostView& v = ctx->views[id];
    size_t total = 0;
    for (HostLevel& L : v.lv) total += (size_t)L.pitch * L.h;
    const size_t need = pyramid_bytes(v);
    v.last_use = ++ctx->use_clock;
    if (v.pyr.bytes() != need) {
        // the view holds no pyramid while room is made for its new one, so it is never the one evicted for it
        drop_pyramid(ctx, v);
        const cudaError_t e = v.pyr.reserve(need / sizeof(uchar4));
        if (e != cudaSuccess)
            return fail(has_source(ctx) && e == cudaErrorMemoryAllocation ? B200MVS_ERR_NO_MEMORY : B200MVS_ERR_CUDA,
                        "pyramid of view %d (%zu bytes): %s", id, need, cudaGetErrorString(e));
        ctx->pyr_resident += need;
    }
    size_t off = 0;
    uint4* qbase = reinterpret_cast<uint4*>(v.pyr.p + total);       // total is a multiple of 4 texels: 16-byte aligned
    for (HostLevel& L : v.lv) { L.d_img = v.pyr.p + off; L.d_quad = qbase + off; off += (size_t)L.pitch * L.h; }
    const dim3 blk(32, 8);
    const dim3 grid0((v.w + 31) / 32, (v.h + 7) / 8);
    const bool planar = src.plane != 0;
    if (b200mvs_undistort::active(v.k2, v.k4)) {
        const b200mvs_undistort::Params P = b200mvs_undistort::make_params(v.w, v.h, ch, v.flen, v.k2, v.k4);
        if (planar) k_undistort_k2k4<true><<<grid0, blk, 0, stream>>>(src, P, v.lv[0].d_img, v.lv[0].pitch);
        else        k_undistort_k2k4<false><<<grid0, blk, 0, stream>>>(src, P, v.lv[0].d_img, v.lv[0].pitch);
    } else {
        if (planar) k_import_rgb<true><<<grid0, blk, 0, stream>>>(src, v.w, v.h, ch, v.lv[0].d_img, v.lv[0].pitch);
        else        k_import_rgb<false><<<grid0, blk, 0, stream>>>(src, v.w, v.h, ch, v.lv[0].d_img, v.lv[0].pitch);
    }
    // ensureImages (image_pyramid.cc:56-95): rescale_half_size_gaussian(img, 1.f) level by level
    const float w1 = std::exp(-0.5f / (2.0f * 1.0f)), w2 = std::exp(-2.5f / (2.0f * 1.0f)), w3 = std::exp(-4.5f / (2.0f * 1.0f));
    for (size_t i = 1; i < v.lv.size(); ++i) {
        const HostLevel& a = v.lv[i - 1];
        const HostLevel& b = v.lv[i];
        k_half_gaussian<<<dim3((b.w + 31) / 32, (b.h + 7) / 8), blk, 0, stream>>>(a.d_img, a.w, a.h, a.pitch, b.d_img, b.w, b.h, b.pitch, w1, w2, w3);
    }
    for (const HostLevel& L : v.lv)
        k_make_quads<<<dim3((L.w + 31) / 32, (L.h + 7) / 8), blk, 0, stream>>>(L.d_img, L.w, L.h, L.pitch, L.d_quad);
    CK(cudaGetLastError());
    v.valid = true;
    v.has_image = true;
    ctx->views_dirty = true;
    return 0;
}

int sync_view_params(b200mvs_ctx* ctx)
{
    if (!ctx->views_dirty) return 0;
    std::vector<ViewParams> hp(ctx->views.size());
    std::memset(hp.data(), 0, hp.size() * sizeof(ViewParams));
    for (size_t i = 0; i < ctx->views.size(); ++i) {
        const HostView& v = ctx->views[i];
        ViewParams& p = hp[i];
        p.valid = v.valid ? 1 : 0;
        if (!v.valid) continue;
        std::memcpy(p.campos, v.campos, 12);
        std::memcpy(p.w2c, v.w2c, 48);
        std::memcpy(p.rot, v.rot, 36);
        p.inv_ax0 = v.lv[0].invproj[0];
        p.nlevels = (int)v.lv.size();
        for (size_t l = 0; l < v.lv.size(); ++l) {
            const HostLevel& L = v.lv[l];
            p.lv[l].ax = L.proj[0]; p.lv[l].ay = L.proj[4]; p.lv[l].cx = L.proj[2]; p.lv[l].cy = L.proj[5];
            p.lv[l].w = L.w; p.lv[l].h = L.h; p.lv[l].pitch = L.pitch; p.lv[l].img = v.has_image ? L.d_img : nullptr;
            p.lv[l].quad = v.has_image ? L.d_quad : nullptr;
        }
    }
    CK(cudaMemcpyAsync(ctx->d_views.p, hp.data(), hp.size() * sizeof(ViewParams), cudaMemcpyHostToDevice, ctx->stream.get()));
    CK(cudaStreamSynchronize(ctx->stream.get()));
    ctx->views_dirty = false;
    return 0;
}

// Opt-in to > 48 KB of dynamic shared memory and size the grids to what is resident on the chip (once per context).
int prepare_kernels(b200mvs_ctx* ctx)
{
    if (ctx->frontier_grid) return 0;
    CK(cudaFuncSetAttribute(k_frontier, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM_BYTES));
    CK(cudaFuncSetAttribute(k_optimize, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)OPT_SMEM_BYTES));
    int per_sm = 0, per_sm_opt = 0, sms = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_frontier, OPT_TPB, OPT_SMEM_BYTES));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_opt, k_optimize, OPT_TPB, OPT_SMEM_BYTES));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
    if (per_sm < 1 || per_sm_opt < 1) return fail(B200MVS_ERR_CUDA, "patch-optimisation kernels do not fit on an SM");
    ctx->optimize_grid = per_sm_opt * sms;
    ctx->frontier_grid = per_sm * sms;
    return 0;
}

// JobParams of one reference view at level `scale` that passed check_ref_view (everything except the map pointers)
JobParams make_job(const b200mvs_ctx* ctx, int scale, int ref, const std::vector<int>& gsel)
{
    const HostLevel& L = ctx->views[ref].lv[scale];
    JobParams J;
    std::memset(&J, 0, sizeof(J));
    J.ref_view = ref; J.W = L.w; J.H = L.h; J.n_global = (int)gsel.size();
    for (size_t k = 0; k < gsel.size(); ++k) J.gview[k] = gsel[k];
    J.ki0 = L.invproj[0]; J.ki2 = L.invproj[2]; J.ki4 = L.invproj[4]; J.ki5 = L.invproj[5];
    J.ref_img = L.d_img; J.ref_pitch = L.pitch;
    return J;
}

unsigned ids_to_slots(const std::vector<int>& gsel, const int32_t* ids, int n, bool* ok)
{
    unsigned s = 0xFFFFFFFFu;
    std::vector<int> slots;
    for (int k = 0; k < n; ++k) {
        auto it = std::lower_bound(gsel.begin(), gsel.end(), (int)ids[k]);
        if (it == gsel.end() || *it != ids[k]) { *ok = false; return s; }
        slots.push_back((int)(it - gsel.begin()));
    }
    std::sort(slots.begin(), slots.end());
    for (size_t k = 0; k < slots.size() && k < 4; ++k) s = (s & ~(0xFFu << (8 * k))) | ((unsigned)slots[k] << (8 * k));
    *ok = true;
    return s;
}

} // namespace

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

const char* b200mvs_version(void) { return "b200mvs 0.1 (sm_90a)"; }

void b200mvs_default_settings(b200mvs_settings* s)
{
    if (!s) return;
    s->filter_width = 5; s->min_ncc = 0.3f; s->min_parallax = 10.0f; s->accept_ncc = 0.6f; s->min_refine_diff = 0.001f;
    s->max_iterations = 20; s->nr_recon_neighbors = 4; s->global_vs_max = 20; s->scale = 0; s->use_color_scale = 1;
    for (int i = 0; i < 3; ++i) { s->aabb_min[i] = -3.402823466e+38f; s->aabb_max[i] = 3.402823466e+38f; }
    s->frontier_band = 0.f; s->frontier_topk = 0;
}

const char* b200mvs_last_error(const b200mvs_ctx*) { return last_error.c_str(); }

int b200mvs_create(int device, int n_views, b200mvs_ctx** out)
{
    if (!out || n_views <= 0) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_create: bad arguments");
    *out = nullptr;
    if (device == B200MVS_DEVICE_NONE) {
        // planning context: cameras, features, global view selection (pure host logic); every compute entry point fails
        *out = new b200mvs_ctx(B200MVS_DEVICE_NONE, n_views);
        return 0;
    }
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(B200MVS_ERR_CUDA, "no CUDA device available (%s); b200mvs has no CPU fallback", cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(B200MVS_ERR_INVALID_ARG, "device %d out of range (%d devices)", device, ndev);
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail(B200MVS_ERR_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
    // on a failure the partly made context is destroyed, which frees what it holds
    std::unique_ptr<b200mvs_ctx> ctx(new b200mvs_ctx(device, n_views));
    auto bail = [](const char* what, cudaError_t ce) { return fail(B200MVS_ERR_CUDA, "%s: %s", what, cudaGetErrorString(ce)); };
    cudaStream_t st = nullptr;
    if ((e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    ctx->stream.reset(st);
    if ((e = ctx->d_views.reserve(n_views)) != cudaSuccess) return bail("device allocation (view table)", e);
    if ((e = ctx->d_lut.reserve(256)) != cudaSuccess) return bail("device allocation (sRGB table)", e);
    void* h = nullptr;
    if ((e = cudaMallocHost(&h, sizeof(HostCounters))) != cudaSuccess) return bail("cudaMallocHost", e);
    ctx->h_counters.reset(static_cast<HostCounters*>(h));
    if ((e = cudaHostAlloc(&h, MIRROR_BYTES, cudaHostAllocMapped)) != cudaSuccess) return bail("cudaHostAlloc", e);
    ctx->h_mirror.reset(static_cast<HostMirror*>(h));
    for (Event* ev : {&ctx->ev_begin, &ctx->ev_end, &ctx->ev_copied, &ctx->ev_caller, &ctx->ev_source}) {
        cudaEvent_t made = nullptr;
        if ((e = cudaEventCreate(&made)) != cudaSuccess) return bail("cudaEventCreate", e);
        ev->reset(made);
    }
    // sRGB code value -> linear: the formula documented at mvs_tools.cc:21-29; tests/test_oracle_vs_reference.py::test_srgb_table_matches_reference checks the
    // 256 floats against the reference table.
    float lut[256];
    for (int i = 0; i < 256; ++i) {
        const double x = i / 255.0;
        lut[i] = (float)((i <= 0.04045 * 255.0) ? x / 12.92 : std::pow((x + 0.055) / 1.055, 2.4));
    }
    if ((e = cudaMemcpy(ctx->d_lut.p, lut, sizeof(lut), cudaMemcpyHostToDevice)) != cudaSuccess) return bail("cudaMemcpy(lut)", e);
    *out = ctx.release();
    return 0;
}

void b200mvs_destroy(b200mvs_ctx* ctx)
{
    if (!ctx) return;
    if (ctx->device != B200MVS_DEVICE_NONE) cudaSetDevice(ctx->device);
    delete ctx;
}

} // extern "C"

namespace {

// The next upload staging slot, at least `bytes` large.  With alloc, a pinned host buffer and a device buffer; without, the
// slot's device bytes are only charged to the budget (a device image is read in place, and charging what a host image would
// hold keeps the accounting, evictions and groups of both kinds of source the same).
int next_stage(b200mvs_ctx* ctx, size_t bytes, bool alloc, b200mvs_ctx::Stage** out)
{
    b200mvs_ctx::Stage& S = ctx->stage[ctx->stage_next++ & 1u];
    if (S.busy) { CK(cudaEventSynchronize(S.done.get())); S.busy = false; }   // the transfer that used this slot two uploads ago
    if (S.cap() < bytes || (alloc && !S.dev.p)) {
        // the old slot goes before the larger one is made
        const size_t cap = std::max(S.cap(), bytes);
        S.host.reset();
        S.dev.release();
        dev_uncharge(ctx, S.charged);
        S.charged = 0;
        if (alloc) {
            void* h = nullptr;
            CK(cudaMallocHost(&h, cap));
            S.host.reset(static_cast<uint8_t*>(h));
            CK(S.dev.reserve(cap));
        } else {
            CK(dev_charge(ctx, cap));
            S.charged = cap;
        }
    }
    *out = &S;
    return 0;
}

// The pyramid of registered view `id` from a host image of its size: pinned staging -> device -> build_pyramid
int upload_host(b200mvs_ctx* ctx, int id, const uint8_t* rgb, int channels)
{
    const HostView& v = ctx->views[id];
    const size_t bytes = (size_t)v.w * v.h * channels;
    b200mvs_ctx::Stage* S = nullptr;
    if (int rc = next_stage(ctx, bytes, true, &S)) return rc;
    if (!S->done) {
        cudaEvent_t made = nullptr;
        CK(cudaEventCreateWithFlags(&made, cudaEventDisableTiming));
        S->done.reset(made);
    }
    std::memcpy(S->host.get(), rgb, bytes);                                  // pageable -> pinned; returns the caller's buffer
    CK(cudaMemcpyAsync(S->dev.p, S->host.get(), bytes, cudaMemcpyHostToDevice, ctx->stream.get()));
    const int rc = build_pyramid(ctx, id, b200mvs_undistort::Src{S->dev.p, (int64_t)v.w * channels, 0}, channels, ctx->stream.get());
    CK(cudaEventRecord(S->done.get(), ctx->stream.get()));
    S->busy = true;
    // no synchronisation here: everything that reads the pyramid is ordered behind it on the context's stream
    return rc;
}

// Empty when a device source's image of view `v` may be read; else what is wrong with it
std::string device_image_problem(const b200mvs_device_image& im, const HostView& v, int device)
{
    char buf[256];
    if (im.w != v.w || im.h != v.h || im.channels < 1 || im.channels > 4) {
        snprintf(buf, sizeof(buf), "is %dx%dx%d, registered as %dx%d", im.w, im.h, im.channels, v.w, v.h);
        return buf;
    }
    const bool planar = im.plane_pitch != 0;
    const int64_t min_row = planar ? (int64_t)im.w : (int64_t)im.w * im.channels;
    if (im.row_pitch < min_row || im.plane_pitch < 0) {
        snprintf(buf, sizeof(buf), "has row_pitch %lld and plane_pitch %lld: row_pitch must be at least %lld and plane_pitch not "
                 "negative", (long long)im.row_pitch, (long long)im.plane_pitch, (long long)min_row);
        return buf;
    }
    if (planar && im.plane_pitch / im.h < im.row_pitch) {                   // plane_pitch < h * row_pitch, without overflow
        snprintf(buf, sizeof(buf), "has plane_pitch %lld: its planes overlap, it must be at least h * row_pitch = %d * %lld",
                 (long long)im.plane_pitch, im.h, (long long)im.row_pitch);
        return buf;
    }
    const std::string why = device_buffer_problem(im.data, device, 1);
    return why.empty() ? why : "data " + why;
}

// A device source's image of view `id`: checked, then the pyramid is built from it in place once the fetch's stream has
// produced it.  The caller releases the image after the kernels that read it have completed.
int load_device_image(b200mvs_ctx* ctx, int id, const b200mvs_device_image& im)
{
    const HostView& v = ctx->views[id];
    const std::string why = device_image_problem(im, v, ctx->device);
    if (!why.empty()) return fail(B200MVS_ERR_INVALID_ARG, "device image of view %d %s", id, why.c_str());
    b200mvs_ctx::Stage* S = nullptr;
    if (int rc = next_stage(ctx, (size_t)v.w * v.h * im.channels, false, &S)) return rc;
    CK(cudaEventRecord(ctx->ev_source.get(), static_cast<cudaStream_t>(im.cuda_stream)));
    CK(cudaStreamWaitEvent(ctx->stream.get(), ctx->ev_source.get(), 0));
    return build_pyramid(ctx, id, b200mvs_undistort::Src{im.data, im.row_pitch, im.plane_pitch}, im.channels, ctx->stream.get());
}

// loadColorImage (image_pyramid.cc:56-95) for every listed view whose pyramid is not resident: through the image source on
// a cache miss; without a source the missing image fails the call.
int load_views(b200mvs_ctx* ctx, const std::vector<int>& ids, int* failed_view)
{
    std::vector<int> held;                    // device images fetched: released once the kernels that read them are done
    int rc = 0;
    for (int id : ids) {
        HostView& v = ctx->views[id];
        if (v.has_image) continue;
        int w = 0, h = 0, channels = 0;
        if (ctx->fetch_device) {
            b200mvs_device_image im = {};
            if (ctx->fetch_device(ctx->user, id, &im) != 0 || !im.data) {
                rc = fail(B200MVS_ERR_INVALID_ARG, "color image of view %d could not be loaded", id);
            } else {
                held.push_back(id);
                rc = load_device_image(ctx, id, im);
                w = im.w; h = im.h; channels = im.channels;
            }
        } else {
            b200mvs_image im = {nullptr, 0, 0, 0};
            if (!ctx->fetch || ctx->fetch(ctx->user, id, &im) != 0 || !im.rgb) {
                rc = fail(B200MVS_ERR_INVALID_ARG, "color image of view %d %s", id, ctx->fetch ? "could not be loaded" : "is not loaded");
            } else {
                if (im.w != v.w || im.h != v.h || im.channels < 1 || im.channels > 4)
                    rc = fail(B200MVS_ERR_INVALID_ARG, "image of view %d is %dx%dx%d, registered as %dx%d", id, im.w, im.h, im.channels, v.w, v.h);
                else
                    rc = upload_host(ctx, id, im.rgb, im.channels);
                if (ctx->release) ctx->release(ctx->user, id);                  // the image was copied to pinned staging
                w = im.w; h = im.h; channels = im.channels;
            }
        }
        if (rc) { if (failed_view) *failed_view = id; break; }
        ctx->mem.n_loads++;
        ctx->mem.bytes_loaded += (uint64_t)w * h * channels;
    }
    if (!held.empty()) {
        // one wait for every pyramid built from the caller's memory, then the images go back
        cudaError_t e = cudaEventRecord(ctx->ev_source.get(), ctx->stream.get());
        if (e == cudaSuccess) e = cudaEventSynchronize(ctx->ev_source.get());
        if (ctx->release) for (int id : held) ctx->release(ctx->user, id);
        if (e != cudaSuccess && !rc) rc = fail(B200MVS_ERR_CUDA, "device image source: %s", cudaGetErrorString(e));
    }
    return rc;
}

} // namespace

extern "C" {

int b200mvs_upload_view(b200mvs_ctx* ctx, int id, const uint8_t* rgb, int w, int h, int channels,
                        float flen, float paspect, const float ppoint[2], const float rot[9], const float trans[3])
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    int rc;
    if ((rc = require_device(ctx)) || (rc = check_camera_args(ctx, "b200mvs_upload_view", id, rgb != nullptr, w, h, ppoint, rot, trans))) return rc;
    if (channels < 1 || channels > 4) return fail(B200MVS_ERR_INVALID_ARG, "Image with invalid number of channels");
    CK(cudaSetDevice(ctx->device));
    if ((rc = set_camera(ctx, id, w, h, flen, paspect, ppoint, rot, trans))) return rc;
    return upload_host(ctx, id, rgb, channels);
}

int b200mvs_upload_view_device(b200mvs_ctx* ctx, int id, const uint8_t* rgb_dev, int w, int h,
                               float flen, float paspect, const float ppoint[2], const float rot[9], const float trans[3],
                               void* cuda_stream)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    int rc;
    if ((rc = require_device(ctx)) || (rc = check_camera_args(ctx, "b200mvs_upload_view_device", id, rgb_dev != nullptr, w, h, ppoint, rot, trans)))
        return rc;
    CK(cudaSetDevice(ctx->device));
    if ((rc = set_camera(ctx, id, w, h, flen, paspect, ppoint, rot, trans))) return rc;
    cudaStream_t s = cuda_stream ? (cudaStream_t)cuda_stream : ctx->stream.get();
    rc = build_pyramid(ctx, id, b200mvs_undistort::Src{rgb_dev, (int64_t)w * 3, 0}, 3, s);
    cudaError_t e = cudaStreamSynchronize(s);
    if (!rc && e != cudaSuccess) rc = fail(B200MVS_ERR_CUDA, "upload sync: %s", cudaGetErrorString(e));
    return rc;
}

int b200mvs_set_view_camera(b200mvs_ctx* ctx, int id, int w, int h, float flen, float paspect, const float ppoint[2],
                            const float rot[9], const float trans[3])
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    int rc = check_camera_args(ctx, "b200mvs_set_view_camera", id, true, w, h, ppoint, rot, trans);
    if (rc) return rc;
    if (ctx->device != B200MVS_DEVICE_NONE) CK(cudaSetDevice(ctx->device));
    if ((rc = set_camera(ctx, id, w, h, flen, paspect, ppoint, rot, trans))) return rc;
    // camera only: the image follows when a call needs the view (loadColorImage, dmrecon.cc:78,238-240)
    drop_pyramid(ctx, ctx->views[id]);
    ctx->views[id].valid = true;
    return 0;
}

int b200mvs_set_view_distortion(b200mvs_ctx* ctx, int id, float k2, float k4)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (id < 0 || id >= (int)ctx->views.size() || !std::isfinite(k2) || !std::isfinite(k4))
        return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_set_view_distortion: bad arguments");
    HostView& v = ctx->views[id];
    if (v.k2 == k2 && v.k4 == k4) return 0;
    v.k2 = k2; v.k4 = k4;
    // the resident pyramid was built with the old coefficients: the view is fetched or uploaded again when needed
    if (v.pyr.p) {
        CK(cudaSetDevice(ctx->device));
        drop_pyramid(ctx, v);
    }
    return 0;
}

int b200mvs_set_view_mask(b200mvs_ctx* ctx, int id, const uint8_t* mask, int w, int h)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (id < 0 || id >= (int)ctx->views.size() || (mask && (w < 1 || h < 1)))
        return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_set_view_mask: bad arguments");
    HostView& v = ctx->views[id];
    if (v.mask_dev.p) {
        CK(cudaSetDevice(ctx->device));
        v.mask_dev.release();
    }
    if (!mask) { v.mask.clear(); v.mask.shrink_to_fit(); v.mask_w = v.mask_h = 0; return 0; }
    v.mask.assign(mask, mask + (size_t)w * h);
    v.mask_w = w; v.mask_h = h;
    return 0;
}

int b200mvs_set_view_mask_device(b200mvs_ctx* ctx, int id, const uint8_t* mask_dev, int w, int h, int64_t row_pitch, void* cuda_stream)
{
    static const char* fn = "b200mvs_set_view_mask_device";
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    std::lock_guard<std::mutex> lk(ctx->mtx);
    const int nv = (int)ctx->views.size();
    if (id < 0 || id >= nv) return fail(B200MVS_ERR_INVALID_ARG, "%s: view_id is %d, not in 0..%d", fn, id, nv - 1);
    HostView& v = ctx->views[id];
    if (!mask_dev) {
        if (v.mask_dev.p) { CK(cudaSetDevice(ctx->device)); v.mask_dev.release(); }
        v.mask.clear(); v.mask.shrink_to_fit(); v.mask_w = v.mask_h = 0;
        return 0;
    }
    if (w < 1) return fail(B200MVS_ERR_INVALID_ARG, "%s: w is %d, must be at least 1", fn, w);
    if (h < 1) return fail(B200MVS_ERR_INVALID_ARG, "%s: h is %d, must be at least 1", fn, h);
    if (row_pitch < w) return fail(B200MVS_ERR_INVALID_ARG, "%s: row_pitch is %lld, less than w (%d)", fn, (long long)row_pitch, w);
    if (ctx->device == B200MVS_DEVICE_NONE)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: mask_dev cannot be read by a planning context (B200MVS_DEVICE_NONE), which has no device", fn);
    CK(cudaSetDevice(ctx->device));
    int rc = check_device_buffer(fn, "mask_dev", mask_dev, ctx->device, 1);
    if (rc) return rc;
    // the new block is filled before the old one goes, so a mask that does not fit leaves the previous one in place
    DevBuf<uint8_t> block(ctx);
    if (block.reserve((size_t)w * h) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200MVS_ERR_NO_MEMORY, "%s: a %d x %d mask does not fit the device budget", fn, w, h);
    }
    cudaStream_t st = ctx->stream.get();
    if ((rc = wait_for_stream(ctx->ev_caller.get(), cuda_stream, st))) return rc;
    CK(cudaMemcpy2DAsync(block.p, (size_t)w, mask_dev, (size_t)row_pitch, (size_t)w, (size_t)h, cudaMemcpyDeviceToDevice, st));
    CK(cudaStreamSynchronize(st));
    std::swap(v.mask_dev.p, block.p);
    std::swap(v.mask_dev.cap, block.cap);
    v.mask.clear(); v.mask.shrink_to_fit();
    v.mask_w = w; v.mask_h = h;
    return 0;
}

namespace {

// The checks of every prior call with a prior that do not depend on the context's device
int check_prior_shape(const char* fn, const b200mvs_ctx* ctx, int id, int w, int h, int stride)
{
    const int nv = (int)ctx->views.size();
    if (id < 0 || id >= nv) return fail(B200MVS_ERR_INVALID_ARG, "%s: view_id is %d, not in 0..%d", fn, id, nv - 1);
    if (w < 1) return fail(B200MVS_ERR_INVALID_ARG, "%s: w is %d, must be at least 1", fn, w);
    if (h < 1) return fail(B200MVS_ERR_INVALID_ARG, "%s: h is %d, must be at least 1", fn, h);
    if (stride < 1 || stride > 65535) return fail(B200MVS_ERR_INVALID_ARG, "%s: stride is %d, not in 1..65535", fn, stride);
    return 0;
}

// The checks of both prior calls with a prior: 0 when it may be stored
int check_prior(const char* fn, const b200mvs_ctx* ctx, int id, int w, int h, int stride)
{
    if (int rc = check_prior_shape(fn, ctx, id, w, h, stride)) return rc;
    if (ctx->device == B200MVS_DEVICE_NONE)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: depth cannot be stored by a planning context (B200MVS_DEVICE_NONE), which has no device", fn);
    return 0;
}

// The planes of a prior: depth, dz and view ids, with their bytes per pixel.  src[k] null: plane k is not given.
struct PriorPlanes {
    static constexpr size_t px_bytes[3] = {sizeof(float), sizeof(float2), sizeof(int4)};
    const void* src[3];
    size_t pitch[3];       // bytes from one row to the next
};

// Makes filled blocks view v's prior, in place of all of its old ones (which the blocks then own and free)
void install_prior(HostView& v, DevBuf<float>& depth, DevBuf<float2>& dz, DevBuf<int4>& ids, int w, int h, int stride)
{
    auto take = [](auto& mine, auto& block) { std::swap(mine.p, block.p); std::swap(mine.cap, block.cap); };
    take(v.prior, depth);
    take(v.prior_dz, dz);
    take(v.prior_ids, ids);
    v.prior_w = w; v.prior_h = h; v.prior_stride = stride;
}

// Copies a w x h prior into new blocks of view `id`, which then replace all of its old ones: a plane that is not given
// leaves the view without one.  The new blocks are filled before the old ones go, so a prior that does not fit leaves the
// previous one whole.
int store_prior(const char* fn, b200mvs_ctx* ctx, int id, const PriorPlanes& in, int w, int h, int stride, cudaMemcpyKind kind)
{
    HostView& v = ctx->views[id];
    const size_t n = (size_t)w * h;
    DevBuf<float> depth(ctx);
    DevBuf<float2> dz(ctx);
    DevBuf<int4> ids(ctx);
    if (depth.reserve(n) != cudaSuccess || (in.src[1] && dz.reserve(n) != cudaSuccess) || (in.src[2] && ids.reserve(n) != cudaSuccess)) {
        cudaGetLastError();
        return fail(B200MVS_ERR_NO_MEMORY, "%s: a %d x %d prior does not fit the device budget", fn, w, h);
    }
    void* const dst[3] = {depth.p, dz.p, ids.p};
    cudaStream_t st = ctx->stream.get();
    for (int k = 0; k < 3; ++k) {
        if (!in.src[k]) continue;
        const size_t row = (size_t)w * PriorPlanes::px_bytes[k];
        CK(cudaMemcpy2DAsync(dst[k], row, in.src[k], in.pitch[k], row, (size_t)h, kind, st));
    }
    CK(cudaStreamSynchronize(st));
    install_prior(v, depth, dz, ids, w, h, stride);
    return 0;
}

// NULL prior: view `id` has none from now on
int clear_prior(const char* fn, b200mvs_ctx* ctx, int id)
{
    const int nv = (int)ctx->views.size();
    if (id < 0 || id >= nv) return fail(B200MVS_ERR_INVALID_ARG, "%s: view_id is %d, not in 0..%d", fn, id, nv - 1);
    HostView& v = ctx->views[id];
    if (v.prior.p) {
        CK(cudaSetDevice(ctx->device));
        v.prior.release();
        v.prior_dz.release();
        v.prior_ids.release();
    }
    v.prior_w = v.prior_h = v.prior_stride = 0;
    return 0;
}

// Where a device prior's planes are read: their pitches, the name of the depth pitch argument and the caller's stream
struct DevicePrior { int64_t pitch[3]; const char* depth_pitch_name; void* stream; };

// The one path of the four prior calls.  dev null: the planes are packed rows in host memory.
int set_prior(const char* fn, b200mvs_ctx* ctx, int id, const float* depth, const float* dz, const int32_t* ids, int w, int h,
              int stride, const DevicePrior* dev)
{
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    std::lock_guard<std::mutex> lk(ctx->mtx);
    const char* const names[3] = {dev ? "depth_dev" : "depth", dev ? "dz_dev" : "dz", dev ? "view_ids_dev" : "view_ids"};
    PriorPlanes P = {{depth, dz, ids}, {}};
    if (!depth) {
        for (int k = 1; k < 3; ++k)
            if (P.src[k]) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s is given without a depth map", fn, names[k]);
        return clear_prior(fn, ctx, id);
    }
    if (int rc = check_prior(fn, ctx, id, w, h, stride)) return rc;
    for (int k = 0; k < 3; ++k) P.pitch[k] = (size_t)w * PriorPlanes::px_bytes[k];
    if (dev) {
        const char* const pitch_names[3] = {dev->depth_pitch_name, "dz_pitch", "ids_pitch"};
        for (int k = 0; k < 3; ++k) {
            const long long least = (long long)P.pitch[k], p = (long long)dev->pitch[k];
            if (P.src[k] && (p < least || p % 4))
                return fail(B200MVS_ERR_INVALID_ARG, "%s: %s is %lld, not a multiple of 4 of at least %d w (%lld)", fn,
                            pitch_names[k], p, (int)PriorPlanes::px_bytes[k], least);
            P.pitch[k] = (size_t)p;
        }
    }
    CK(cudaSetDevice(ctx->device));
    if (dev) {
        for (int k = 0; k < 3; ++k)
            if (P.src[k])
                if (int rc = check_device_buffer(fn, names[k], P.src[k], ctx->device, 4)) return rc;
        if (int rc = wait_for_stream(ctx->ev_caller.get(), dev->stream, ctx->stream.get())) return rc;
    }
    return store_prior(fn, ctx, id, P, w, h, stride, dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice);
}

} // namespace

int b200mvs_set_view_prior(b200mvs_ctx* ctx, int id, const float* depth, int w, int h, int stride)
{
    return set_prior("b200mvs_set_view_prior", ctx, id, depth, nullptr, nullptr, w, h, stride, nullptr);
}

int b200mvs_set_view_prior_device(b200mvs_ctx* ctx, int id, const float* depth_dev, int w, int h, int64_t row_pitch, int stride,
                                  void* cuda_stream)
{
    const DevicePrior dev = {{row_pitch, 0, 0}, "row_pitch", cuda_stream};
    return set_prior("b200mvs_set_view_prior_device", ctx, id, depth_dev, nullptr, nullptr, w, h, stride, &dev);
}

int b200mvs_set_view_prior_state(b200mvs_ctx* ctx, int id, const float* depth, const float* dz, const int32_t* ids, int w,
                                 int h, int stride)
{
    return set_prior("b200mvs_set_view_prior_state", ctx, id, depth, dz, ids, w, h, stride, nullptr);
}

int b200mvs_set_view_prior_state_device(b200mvs_ctx* ctx, int id, const float* depth_dev, const float* dz_dev,
                                        const int32_t* ids_dev, int w, int h, int64_t depth_pitch, int64_t dz_pitch,
                                        int64_t ids_pitch, int stride, void* cuda_stream)
{
    const DevicePrior dev = {{depth_pitch, dz_pitch, ids_pitch}, "depth_pitch", cuda_stream};
    return set_prior("b200mvs_set_view_prior_state_device", ctx, id, depth_dev, dz_dev, ids_dev, w, h, stride, &dev);
}

namespace {

static_assert(B200MVS_PRIOR_DISPARITY == PRIOR_DISPARITY && B200MVS_PRIOR_DEPTH == PRIOR_DEPTH &&
              B200MVS_PRIOR_DEPTH_SCALE == PRIOR_DEPTH_SCALE, "prior kinds of include/b200mvs.h and prior_align.cuh");
constexpr size_t ALIGN_FIT_BYTES = 64;          // the fit record's slot in the scratch block
static_assert(sizeof(AlignFit) <= ALIGN_FIT_BYTES, "AlignFit fits its slot");

const char* align_reason(int status)
{
    switch (status) {
    case ALIGN_FEW_OBS: return "fewer than 16 usable feature observations";
    case ALIGN_FLAT: return "the map has no spread at the observations (MAD(d) = 0)";
    case ALIGN_FEW_INLIERS: return "fewer than 16 inliers";
    case ALIGN_SINGULAR: return "the least-squares refit is singular";
    default: return "the scale is not positive, or the scale or shift is not finite";
    }
}

// The one path of b200mvs_set_view_prior_relative[_device]: the observations of the view's features, the fit and the
// apply run on the context's stream, and a fit that may be installed becomes the view's prior.  dev: values are in
// device memory, rows `pitch` bytes apart; else packed host rows, uploaded into the new block and applied there.
int set_prior_relative(const char* fn, b200mvs_ctx* ctx, int id, const float* values, int w, int h, int64_t pitch, int stride,
                       int kind, bool dev, void* cuda_stream, b200mvs_prior_fit* out)
{
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    if (out) *out = b200mvs_prior_fit{};
    std::lock_guard<std::mutex> lk(ctx->mtx);
    const char* field = dev ? "values_dev" : "values";
    if (int rc = check_prior_shape(fn, ctx, id, w, h, stride)) return rc;
    if (!values) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s is NULL", fn, field);
    if (kind < B200MVS_PRIOR_DISPARITY || kind > B200MVS_PRIOR_DEPTH_SCALE)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: kind is %d, not a B200MVS_PRIOR_* kind (0..2)", fn, kind);
    const HostView& v = ctx->views[id];
    if (!v.valid) return fail(B200MVS_ERR_INVALID_ARG, "%s: view_id %d has no camera", fn, id);
    if (ctx->feat_off.size() < 2) return fail(B200MVS_ERR_INVALID_ARG, "%s: the context has no features (b200mvs_set_features)", fn);
    if (dev && (pitch < 4ll * w || pitch % 4))
        return fail(B200MVS_ERR_INVALID_ARG, "%s: row_pitch is %lld, not a multiple of 4 of at least 4 w (%lld)", fn,
                    (long long)pitch, 4ll * w);
    if (ctx->device == B200MVS_DEVICE_NONE)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: %s cannot be read by a planning context (B200MVS_DEVICE_NONE), which has no device", fn, field);
    CK(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream.get();
    if (dev) {
        if (int rc = check_device_buffer(fn, field, values, ctx->device, 4)) return rc;
        if (int rc = wait_for_stream(ctx->ev_caller.get(), cuda_stream, st)) return rc;
    }
    // the view's features, from the inverted index
    const int* fid = ctx->vf_ids.data() + ctx->vf_off[id];
    const unsigned m = (unsigned)(ctx->vf_off[id + 1] - ctx->vf_off[id]);
    std::vector<float> pos(3 * (size_t)m);
    for (unsigned i = 0; i < m; ++i) std::memcpy(&pos[3 * (size_t)i], &ctx->feat_pos[3 * (size_t)fid[i]], 3 * sizeof(float));
    AlignCam cam;
    for (int k = 0; k < 9; ++k) cam.R[k] = v.rot[k];
    for (int k = 0; k < 3; ++k) cam.t[k] = v.trans[k];
    const HostLevel& L0 = v.lv[0];
    cam.ax = L0.proj[0]; cam.ay = L0.proj[4]; cam.cx = L0.proj[2]; cam.cy = L0.proj[5];
    cam.W0 = v.w; cam.H0 = v.h;
    // the new block, then the scratch: observations (16 B each), the fit record and the positions (12 B each)
    DevBuf<float> block(ctx);
    DevBuf<float2> no_dz(ctx);
    DevBuf<int4> no_ids(ctx);
    DevBuf<unsigned char> scratch(ctx);
    const size_t obs_bytes = sizeof(double2) * (size_t)m;
    if (block.reserve((size_t)w * h) != cudaSuccess || scratch.reserve(obs_bytes + ALIGN_FIT_BYTES + 3 * sizeof(float) * (size_t)m) != cudaSuccess) {
        cudaGetLastError();
        return fail(B200MVS_ERR_NO_MEMORY, "%s: a %d x %d prior and the scratch of %u features do not fit the device budget", fn, w, h, m);
    }
    double2* obs = reinterpret_cast<double2*>(scratch.p);
    AlignFit* fit = reinterpret_cast<AlignFit*>(scratch.p + obs_bytes);
    float* pos_dev = reinterpret_cast<float*>(scratch.p + obs_bytes + ALIGN_FIT_BYTES);
    const float* src = values;
    size_t src_pitch = (size_t)pitch;
    if (!dev) {
        src_pitch = (size_t)w * sizeof(float);
        CK(cudaMemcpyAsync(block.p, values, src_pitch * h, cudaMemcpyHostToDevice, st));
        src = block.p;
    }
    if (m) {
        CK(cudaMemcpyAsync(pos_dev, pos.data(), 3 * sizeof(float) * (size_t)m, cudaMemcpyHostToDevice, st));
        k_align_observe<<<(m + 255) / 256, 256, 0, st>>>(pos_dev, m, cam, src, w, h, src_pitch, kind, obs);
    }
    k_align_fit<<<1, ALIGN_FIT_TPB, 0, st>>>(obs, m, kind, fit);
    const dim3 blk(32, 8);
    k_align_apply<<<dim3((w + 31) / 32, (h + 7) / 8), blk, 0, st>>>(src, src_pitch, block.p, w, h, cam, kind, fit);
    CK(cudaGetLastError());
    AlignFit f;
    CK(cudaMemcpyAsync(&f, fit, sizeof(f), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (out) {
        out->n_obs = f.n_obs;
        if (f.status == ALIGN_OK) { out->scale = f.s; out->shift = f.t; out->n_inliers = f.n_in; out->median_rel_err = f.med_rel; }
    }
    if (f.status != ALIGN_OK) return fail(B200MVS_ERR_INVALID_ARG, "%s: the fit failed: %s (%u observations)", fn, align_reason(f.status), f.n_obs);
    install_prior(ctx->views[id], block, no_dz, no_ids, w, h, stride);
    return 0;
}

} // namespace

int b200mvs_set_view_prior_relative(b200mvs_ctx* ctx, int id, const float* values, int w, int h, int stride, int kind,
                                    b200mvs_prior_fit* fit_out)
{
    return set_prior_relative("b200mvs_set_view_prior_relative", ctx, id, values, w, h, 0, stride, kind, false, nullptr, fit_out);
}

int b200mvs_set_view_prior_relative_device(b200mvs_ctx* ctx, int id, const float* values_dev, int w, int h, int64_t row_pitch,
                                           int stride, int kind, void* cuda_stream, b200mvs_prior_fit* fit_out)
{
    return set_prior_relative("b200mvs_set_view_prior_relative_device", ctx, id, values_dev, w, h, row_pitch, stride, kind,
                              true, cuda_stream, fit_out);
}

int b200mvs_set_features(b200mvs_ctx* ctx, int n, const float* pos, const int32_t* off, const int32_t* ids)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (n < 0 || (n > 0 && (!pos || !off || !ids))) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_set_features: bad arguments");
    { std::lock_guard<std::mutex> pl(ctx->plan_mtx); ctx->plans.clear(); }
    ctx->feat_pos.assign(pos, pos + 3 * (size_t)n);
    ctx->feat_off.assign(1, 0);
    ctx->feat_refs.clear();
    for (int i = 0; i < n; ++i) {
        ctx->feat_refs.insert(ctx->feat_refs.end(), ids + off[i], ids + off[i + 1]);
        ctx->feat_off.push_back((int)ctx->feat_refs.size());
    }
    // Feature3D::contains_view_id (bundle.cc:15-21) for every view at once
    std::vector<std::vector<int>> view_feats(ctx->views.size());
    for (int i = 0; i < n; ++i)
        for (int r = ctx->feat_off[i]; r < ctx->feat_off[i + 1]; ++r) {
            const int vid = ctx->feat_refs[r];
            if (vid >= 0 && vid < (int)ctx->views.size()) {
                std::vector<int>& vf = view_feats[vid];
                if (vf.empty() || vf.back() != i) vf.push_back(i);
            }
        }
    ctx->vf_off.assign(1, 0);
    ctx->vf_ids.clear();
    for (const std::vector<int>& vf : view_feats) {
        ctx->vf_ids.insert(ctx->vf_ids.end(), vf.begin(), vf.end());
        ctx->vf_off.push_back((int)ctx->vf_ids.size());
    }
    return 0;
}

int b200mvs_num_levels(b200mvs_ctx* ctx, int id)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (id < 0 || id >= (int)ctx->views.size() || !ctx->views[id].valid) return B200MVS_ERR_INVALID_ARG;
    return (int)ctx->views[id].lv.size();
}

} // extern "C"

namespace {

// b200mvs_get_level (rgb_dev == nullptr) and b200mvs_get_level_device (rgb == nullptr, with the caller's stream): the size
// of the level and, when a buffer is given, its packed RGB bytes, written in place into a device buffer or through a
// staging buffer into a host one
int get_level(b200mvs_ctx* ctx, int id, int level, int* w, int* h, uint8_t* rgb, uint8_t* rgb_dev, void* cuda_stream)
{
    if (id < 0 || id >= (int)ctx->views.size() || !ctx->views[id].valid) return fail(B200MVS_ERR_INVALID_ARG, "invalid view");
    const HostView& v = ctx->views[id];
    if (level < 0 || level >= (int)v.lv.size()) return fail(B200MVS_ERR_INVALID_ARG, "invalid level");
    const HostLevel& L = v.lv[level];
    if (w) *w = L.w;
    if (h) *h = L.h;
    if (!rgb && !rgb_dev) return 0;
    // a planning context has no image and no source: it fails in load_views before any device call
    int rc = 0;
    if (ctx->device != B200MVS_DEVICE_NONE) {
        CK(cudaSetDevice(ctx->device));
        if (rgb_dev && ((rc = check_device_buffer("b200mvs_get_level_device", "rgb_dev", rgb_dev, ctx->device, 1)) ||
                        (rc = wait_for_stream(ctx->ev_caller.get(), cuda_stream, ctx->stream.get()))))
            return rc;
    }
    const PinsOfCall pins(ctx);
    pin_views(ctx, {id});
    if ((rc = load_views(ctx, {id}, nullptr))) return rc;   // an evicted view is fetched again through the source
    const dim3 grid((L.w + 31) / 32, (L.h + 7) / 8), blk(32, 8);
    const cudaStream_t st = ctx->stream.get();
    if (rgb_dev) {
        k_export_rgb<<<grid, blk, 0, st>>>(L.d_img, L.w, L.h, L.pitch, rgb_dev);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(st));
        return 0;
    }
    DevBuf<uint8_t> d(ctx);
    const size_t bytes = (size_t)L.w * L.h * 3;
    CK(d.reserve(bytes));
    k_export_rgb<<<grid, blk, 0, st>>>(L.d_img, L.w, L.h, L.pitch, d.p);
    cudaError_t e = cudaMemcpyAsync(rgb, d.p, bytes, cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(B200MVS_ERR_CUDA, "get_level copy: %s", cudaGetErrorString(e));
    return 0;
}

} // namespace

extern "C" {

int b200mvs_get_level(b200mvs_ctx* ctx, int id, int level, int* w, int* h, uint8_t* rgb)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    return get_level(ctx, id, level, w, h, rgb, nullptr, nullptr);
}

int b200mvs_get_level_device(b200mvs_ctx* ctx, int id, int level, int* w, int* h, uint8_t* rgb_dev, void* cuda_stream)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    return get_level(ctx, id, level, w, h, nullptr, rgb_dev, cuda_stream);
}

int b200mvs_global_view_selection(b200mvs_ctx* ctx, const b200mvs_settings* s, int ref, int32_t* ids_out, int cap)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    int rc;
    if ((rc = check_settings(s)) || (rc = check_ref_view(ctx, s->scale, ref))) return rc;
    if (cap > 0 && !ids_out) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_global_view_selection: ids_out is NULL");
    std::vector<int> sel;
    bool planned = false;
    {
        // a plan prepared by b200mvs_plan_views already holds the selection (it stays there for b200mvs_reconstruct)
        std::lock_guard<std::mutex> pl(ctx->plan_mtx);
        if (const HostPlan* p = find_plan(ctx, *s, ref)) { sel = p->gsel; planned = true; }
    }
    if (!planned) {
        std::vector<PL::PlanView> views;
        sel = global_view_selection(plan_input(ctx, *s, views), s->min_parallax, ref);
    }
    for (int i = 0; i < (int)sel.size() && i < cap; ++i) ids_out[i] = sel[i];
    return (int)sel.size();
}

int b200mvs_set_patch_mode(b200mvs_ctx* ctx, int mode, int64_t thread_min)
{
    if (!ctx || mode < 0 || mode > 2) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    ctx->optimize_mode = mode;
    ctx->thread_min = thread_min;
    return 0;
}

int b200mvs_set_frontier_capacity(b200mvs_ctx* ctx, double entries_per_px, uint64_t min_entries)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (!std::isfinite(entries_per_px) || entries_per_px < 0.0 || entries_per_px > 64.0)
        return fail(B200MVS_ERR_INVALID_ARG, "frontier capacity: entries per pixel must be in [0, 64], got %g", entries_per_px);
    if (min_entries > (1ull << 40) || (entries_per_px == 0.0 && min_entries == 0))
        return fail(B200MVS_ERR_INVALID_ARG, "frontier capacity: min_entries must be at most 2^40, and at least 1 when entries per pixel is 0");
    ctx->frontier_cap.per_px = entries_per_px;
    ctx->frontier_cap.min = min_entries;
    return 0;
}

int b200mvs_frontier_info(b200mvs_ctx* ctx, uint64_t* initial_entries, uint64_t* final_entries, uint64_t* n_resumes)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (initial_entries) *initial_entries = ctx->fr_initial;
    if (final_entries) *final_entries = ctx->fr_final;
    if (n_resumes) *n_resumes = ctx->fr_resumes;
    return 0;
}

int b200mvs_plan_views(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    // Deliberately NOT under ctx->mtx: planning reads only cameras and features and may overlap a running
    // b200mvs_reconstruct of another batch (the caller must not change cameras / features meanwhile).
    int rc = check_settings(s);
    if (rc) return rc;
    if (n_refs < 0 || (n_refs > 0 && !refs)) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_plan_views: bad arguments");
    // entries at s->scale with their plans only: the workspace reads per-view state that changes under ctx->mtx
    Batch B;
    std::vector<int> all(n_refs);
    for (int j = 0; j < n_refs; ++j) {
        if ((rc = check_ref_view(ctx, s->scale, refs[j]))) return rc;
        B.e.push_back(BatchEntry{refs[j], s->scale});
        all[j] = j;
    }
    std::vector<PL::PlanView> views;
    make_plans(plan_input(ctx, *s, views), *s, B, all);
    std::lock_guard<std::mutex> pl(ctx->plan_mtx);
    for (BatchEntry& E : B.e) ctx->plans[E.view] = std::move(E.plan);
    return 0;
}

int b200mvs_optimize_patches(b200mvs_ctx* ctx, const b200mvs_settings* s, int ref, const int32_t* gids, int ng,
                             const b200mvs_patch_in* in, int n, b200mvs_patch_out* out, b200mvs_stats* stats)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    int rc;
    if ((rc = require_device(ctx)) || (rc = check_settings(s)) || (rc = check_ref_view(ctx, s->scale, ref))) return rc;
    if (ng < 1 || ng > MAX_GLOBAL || !gids || n < 0 || (n > 0 && (!in || !out)))
        return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_optimize_patches: bad arguments");
    std::vector<int> gsel(gids, gids + ng);
    if (!std::is_sorted(gsel.begin(), gsel.end())) return fail(B200MVS_ERR_INVALID_ARG, "global ids must be ascending");
    for (int g : gsel) if (g < 0 || g >= (int)ctx->views.size() || !ctx->views[g].valid) return fail(B200MVS_ERR_INVALID_ARG, "invalid global view id");
    CK(cudaSetDevice(ctx->device));
    std::vector<int> need(gsel);
    need.push_back(ref);
    const PinsOfCall pins(ctx);
    pin_views(ctx, need);
    if ((rc = load_views(ctx, need, nullptr))) return rc;
    if (stats) std::memset(stats, 0, sizeof(*stats));
    if (n == 0) return 0;
    if ((rc = sync_view_params(ctx))) return rc;
    const JobParams J = make_job(ctx, s->scale, ref, gsel);
    std::vector<Entry> he(n);
    for (int i = 0; i < n; ++i) {
        bool ok = true;
        if (in[i].n_local < 0 || in[i].n_local > 4) return fail(B200MVS_ERR_INVALID_ARG, "patch %d: n_local out of range", i);
        const unsigned slots = ids_to_slots(gsel, in[i].local_ids, in[i].n_local, &ok);
        if (!ok) return fail(B200MVS_ERR_INVALID_ARG, "patch %d: local view id not in the global set", i);
        // a patch outside the 16-bit range goes to (0xFFFF, 0xFFFF), which the kernel's bounds test rejects
        const bool in_range = in[i].x >= 0 && in[i].y >= 0 && in[i].x <= 0xFFFF && in[i].y <= 0xFFFF;
        he[i] = make_entry(in_range ? pack_xy(in[i].x, in[i].y) : pack_xy(0xFFFF, 0xFFFF), 0, 0, 0.f, in[i].depth, in[i].dz_i,
                           in[i].dz_j, slots);
    }
    // idle workspace goes first when these buffers would not fit next to it
    if (ctx->mem.resident + (uint64_t)n * (sizeof(Entry) + sizeof(PatchOut)) + sizeof(JobParams) + 4096 > budget_limit(ctx))
        release_workspace(ctx);
    WorkspaceInUse in_use(ctx);
    CK(ctx->run_in.reserve(n));
    CK(ctx->run_out.reserve(n));
    CK(ctx->counters.reserve(C_NUM + 8));
    CK(ctx->d_jobs.reserve(1));
    CK(ctx->d_settings.reserve(1));
    const DevSettings ds = to_dev(*s);
    cudaStream_t st = ctx->stream.get();
    CK(cudaMemcpyAsync(ctx->run_in.p, he.data(), sizeof(Entry) * n, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_jobs.p, &J, sizeof(J), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_settings.p, &ds, sizeof(ds), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(ctx->counters.p, 0, sizeof(unsigned long long) * C_NUM, st));
    cudaEvent_t e0 = ctx->ev_begin.get(), e1 = ctx->ev_end.get();
    CK(cudaEventRecord(e0, st));
    {
        int rc2 = prepare_kernels(ctx);
        if (rc2) return rc2;
        const int warps_per_block = OPT_TPB / 32;
        const int grid = std::max(1, std::min((n + warps_per_block - 1) / warps_per_block, ctx->optimize_grid));
        k_optimize<<<grid, OPT_TPB, OPT_SMEM_BYTES, st>>>(ctx->run_in.p, ctx->run_out.p, n, ctx->optimize_mode, ctx->d_settings.p,
                                                          ctx->d_jobs.p, ctx->d_views.p, ctx->d_lut.p, ctx->counters.p);
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(e1, st));
    std::vector<PatchOut> ho(n);
    CK(cudaMemcpyAsync(ho.data(), ctx->run_out.p, sizeof(PatchOut) * n, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(ctx->h_counters->count, ctx->counters.p, sizeof(unsigned long long) * C_NUM, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) {
        const PatchOut& r = ho[i];
        b200mvs_patch_out& o = out[i];
        o.conf = r.conf; o.depth = r.depth; o.dz_i = r.dzI; o.dz_j = r.dzJ;
        o.normal[0] = r.nx; o.normal[1] = r.ny; o.normal[2] = r.nz;
        o.n_local = slots_to_ids(J.gview, J.n_global, r.slots, o.local_ids);
        o.iterations = r.iterations; o.converged = r.flags & 1; o.opti_success = (r.flags >> 1) & 1;
    }
    if (stats) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, e0, e1);
        stats->n_opt = ctx->h_counters->count[C_OPTS];
        stats->n_sample_sets = ctx->h_counters->count[C_SETS];
        stats->ms_patch_kernel = ms; stats->ms_total_device = ms;
        stats->n_patch_launches = 1; stats->n_kernel_launches = 1;
    }
    return 0;
}

} // extern "C"

// ------------------------------------------------------------------------------------------------
// host: batches, groups that fit the device budget, one frontier launch per group
// ------------------------------------------------------------------------------------------------
namespace {

// The first step of building the batch of b200mvs_reconstruct, b200mvs_working_set and b200mvs_plan_batches: the
// settings, then the entries into B.  levels: the pyramid level of each entry (the *_levels entry points), or NULL for
// s->scale everywhere.  An entry is a (view, level) pair, and a call of the *_levels entry points may hold each pair once.
// B.e stays empty when the settings or the arguments fail, before any view is checked.
int check_batch(const b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                b200mvs_progress* progress, Batch& B)
{
    int rc = check_settings(s, !levels);
    if (rc) return rc;
    if (n_refs < 1 || !refs) return fail(B200MVS_ERR_INVALID_ARG, "bad arguments");
    B = Batch{*s, {}, progress};
    for (int j = 0; j < n_refs; ++j) B.e.push_back(BatchEntry{refs[j], levels ? levels[j] : s->scale});
    for (int j = 0; j < n_refs; ++j) {
        const BatchEntry& E = B.e[j];
        B.failed = j;
        if ((rc = check_ref_view(ctx, E.level, E.view))) return rc;
        const HostLevel& L = ctx->views[E.view].lv[E.level];
        if (L.w > 0xFFFF || L.h > 0xFFFF) return fail(B200MVS_ERR_UNSUPPORTED, "reference level larger than 65535 pixels per side");
    }
    B.failed = -1;
    if (levels) {
        std::vector<std::pair<int, int>> pairs(n_refs);
        for (int j = 0; j < n_refs; ++j) pairs[j] = {B.e[j].view, B.e[j].level};
        std::sort(pairs.begin(), pairs.end());
        const auto dup = std::adjacent_find(pairs.begin(), pairs.end());
        if (dup != pairs.end()) {
            B.failed = (int)(std::find_if(B.e.begin(), B.e.end(), [&](const BatchEntry& E) { return E.view == dup->first; }) - B.e.begin());
            return fail(B200MVS_ERR_INVALID_ARG, "view %d appears more than once at level %d", dup->first, dup->second);
        }
    }
    return 0;
}

// The level array of a *_levels entry point `fn`, which must not be NULL
int check_levels(const char* fn, const int32_t* levels, int32_t* failed_view)
{
    if (failed_view) *failed_view = -1;
    return levels ? 0 : fail(B200MVS_ERR_INVALID_ARG, "%s: levels is NULL", fn);
}

// ---- the host phase on the device (plan_device.cuh) ----
constexpr int PLAN_TPB = 256;
struct BlockSync { __device__ void operator()() const { __syncthreads(); } };

__global__ void __launch_bounds__(PLAN_TPB) k_plan_views(const b200mvs_plan::PlanInput in, const b200mvs_plan::PlanJob* __restrict__ jobs,
                                                         uint32_t* ws, uint32_t* out)
{
    b200mvs_plan::PlanBlock B;
    B.bind(&in, &jobs[blockIdx.x], ws, out);
    b200mvs_plan::plan_view(B, (int)threadIdx.x, (int)blockDim.x, BlockSync{});
}

inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// Plans B.e[j] for j in `todo` on the device: one CTA per reference view, one launch per chunk of views that fits the
// budget next to the shared inputs.  The views it cannot plan stay in `todo` for host threads: all of them when the
// factor table would exceed its cap (min_parallax above about 41 degrees), and any view whose workspace does not fit on
// its own.  Every allocation goes through the accounted allocator and is freed before it returns.
int plan_on_device(b200mvs_ctx* ctx, const b200mvs_settings& s, const PL::PlanInput& in, Batch& B, std::vector<int>& todo)
{
    const uint64_t n_table = PL::table_entries(in.dot_skip);
    if (todo.empty() || n_table == 0) return 0;
    CK(cudaSetDevice(ctx->device));
    const int nv = in.nv, nf = in.nf;
    if (ctx->plx_table.size() != n_table || ctx->plx_table_mp != s.min_parallax) {
        ctx->plx_table.resize(n_table);
        PL::fill_table(ctx->plx_table.data(), n_table, in.dot_skip, s.min_parallax);
        ctx->plx_table_mp = s.min_parallax;
    }
    size_t max_vf = 0;
    for (int v = 0; v < nv; ++v) max_vf = std::max(max_vf, (size_t)(in.vf_off[v + 1] - in.vf_off[v]));
    // the input's arrays as they are, then the factor table
    const std::pair<const void*, size_t> parts[] = {{in.views, nv * sizeof(PL::PlanView)}, {in.feat_pos, 3 * (size_t)nf * 4},
                                                    {in.feat_off, ((size_t)nf + 1) * 4}, {in.feat_refs, (size_t)in.feat_off[nf] * 4},
                                                    {in.vf_off, ((size_t)nv + 1) * 4}, {in.vf_ids, (size_t)in.vf_off[nv] * 4},
                                                    {ctx->plx_table.data(), ctx->plx_table.size() * 4}};
    size_t in_bytes = 0;
    for (const auto& q : parts) in_bytes += align256(q.second);
    // one reference view: its workspace (bounded by the refs of its features) and its results (the seeds bounded by the
    // features of the view and of globalVSMax views with the most features)
    struct Sized { int j; PL::PlanJob job; size_t bytes; };
    std::vector<Sized> jobs;
    for (int j : todo) {
        const int ref = B.e[j].view;
        PL::PlanJob J = {};
        J.ref = ref;
        J.F = in.vf_off[ref + 1] - in.vf_off[ref];
        for (int t = in.vf_off[ref]; t < in.vf_off[ref + 1]; ++t) J.E += (uint64_t)(in.feat_off[in.vf_ids[t] + 1] - in.feat_off[in.vf_ids[t]]);
        J.seed_cap = std::min<uint64_t>((uint64_t)nf, (uint64_t)J.F + (uint64_t)s.global_vs_max * max_vf);
        const uint64_t words = PL::job_layout(J.F, J.E, nv, nf).words + PL::out_words(J.seed_cap) + sizeof(PL::PlanJob) / 4;
        jobs.push_back(Sized{j, J, (size_t)words * 4});
    }
    // what the call may hold: the budget's headroom (pyramids of unpinned views can be evicted); without a budget, half
    // the free device memory
    if (ctx->mem.budget && ctx->mem.resident + in_bytes + jobs[0].bytes > ctx->mem.budget) release_workspace(ctx);
    uint64_t avail = headroom(ctx, 0);
    if (!ctx->mem.budget) {
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        avail = free_b / 2;
    }
    if (in_bytes >= avail) return 0;
    avail -= in_bytes;
    DevBuf<char> d_in(ctx);
    CK(d_in.reserve(in_bytes));
    cudaStream_t st = ctx->stream.get();
    PL::PlanInput d = in;              // the same input with the device copies of its arrays
    {
        const void* dptr[7];
        size_t o = 0;
        for (int k = 0; k < 7; ++k) {
            dptr[k] = d_in.p + o;
            if (parts[k].second) CK(cudaMemcpyAsync(d_in.p + o, parts[k].first, parts[k].second, cudaMemcpyHostToDevice, st));
            o += align256(parts[k].second);
        }
        d.views = static_cast<const PL::PlanView*>(dptr[0]);
        d.feat_pos = static_cast<const float*>(dptr[1]);
        d.feat_off = static_cast<const int*>(dptr[2]); d.feat_refs = static_cast<const int*>(dptr[3]);
        d.vf_off = static_cast<const int*>(dptr[4]); d.vf_ids = static_cast<const int*>(dptr[5]);
        d.table = static_cast<const float*>(dptr[6]);
    }
    std::vector<char> done(B.e.size(), 0);
    b200mvs_plan_info& info = ctx->plan_info;
    size_t k0 = 0;
    while (k0 < jobs.size()) {
        // the next chunk: consecutive views while they fit; a view that does not fit on its own is left to the host
        if (jobs[k0].bytes > avail) { ++k0; continue; }
        size_t k1 = k0, bytes = 0;
        while (k1 < jobs.size() && jobs[k1].bytes <= avail - bytes) bytes += jobs[k1++].bytes;
        const size_t n = k1 - k0;
        uint64_t ws_words = 0, out_words = 0;
        std::vector<PL::PlanJob> hj(n);
        for (size_t k = 0; k < n; ++k) {
            hj[k] = jobs[k0 + k].job;
            hj[k].ws = ws_words; ws_words += PL::job_layout(hj[k].F, hj[k].E, nv, nf).words;
            hj[k].out = out_words; out_words += PL::out_words(hj[k].seed_cap);
        }
        const size_t jobs_bytes = align256(n * sizeof(PL::PlanJob));
        // the chunk's workspace and results, freed in reverse order before the next chunk
        DevBuf<char> d_ws(ctx), d_out(ctx);
        CK(d_ws.reserve(align256(ws_words * 4)));
        CK(d_out.reserve(jobs_bytes + out_words * 4));
        info.peak_bytes = std::max<uint64_t>(info.peak_bytes, in_bytes + align256(ws_words * 4) + jobs_bytes + out_words * 4);
        uint32_t* d_res = reinterpret_cast<uint32_t*>(d_out.p + jobs_bytes);
        CK(cudaMemcpyAsync(d_out.p, hj.data(), n * sizeof(PL::PlanJob), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(d_res, 0, out_words * 4, st));
        cudaEvent_t e0 = ctx->ev_begin.get(), e1 = ctx->ev_end.get();
        CK(cudaEventRecord(e0, st));
        k_plan_views<<<(unsigned)n, PLAN_TPB, 0, st>>>(d, reinterpret_cast<const PL::PlanJob*>(d_out.p), reinterpret_cast<uint32_t*>(d_ws.p), d_res);
        CK(cudaGetLastError());
        CK(cudaEventRecord(e1, st));
        std::vector<uint32_t> res(out_words);
        CK(cudaMemcpyAsync(res.data(), d_res, out_words * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        info.ms_device += ms;
        for (size_t k = 0; k < n; ++k) {
            const uint32_t* r = &res[hj[k].out];
            const int j = jobs[k0 + k].j;
            HostPlan& p = B.e[j].plan;
            p.settings = s;
            p.gsel.assign(reinterpret_cast<const int*>(r + PL::OUT_SEL), reinterpret_cast<const int*>(r + PL::OUT_SEL) + r[0]);
            done[j] = 1;
            info.n_device++;
            if (p.gsel.empty()) continue;
            if (B.progress) B.progress[j].status = 2;
            const PL::SeedOut* so = reinterpret_cast<const PL::SeedOut*>(r + PL::OUT_HEAD);
            p.seeds.assign(so, so + r[1]);
        }
        k0 = k1;
    }
    todo.erase(std::remove_if(todo.begin(), todo.end(), [&](int j) { return done[j] != 0; }), todo.end());
    return 0;
}

// The second step of building a batch: analyzeFeatures + globalViewSelection + seed list per entry (dmrecon.cc:179-292)
// into its plan, then its workspace and needed views.  A plan prepared ahead (b200mvs_plan_views, possibly while the
// previous batch was running) serves an entry whose settings at its level are the plan's; the other entries are planned
// once per distinct level, each with the planning input of that level, as a call at that level alone.  A view whose
// selection is empty fails the call.
// `recon`: a reconstruction consumes the prepared plans it uses, may plan the others on the device (plan_on_device) and
// records its planning in ctx->plan_info; the inspection calls read prepared plans and plan on host threads.
int plan_batch(b200mvs_ctx* ctx, Batch& B, bool recon)
{
    const auto t0 = std::chrono::steady_clock::now();
    const int n_refs = (int)B.e.size();
    std::map<int, std::vector<int>> todo;            // the entries without a prepared plan, by level
    {
        const std::time_t t_start = std::time(nullptr);
        std::lock_guard<std::mutex> pl(ctx->plan_mtx);
        for (int j = 0; j < n_refs; ++j) {
            BatchEntry& E = B.e[j];
            if (B.progress) { B.progress[j].status = 1; B.progress[j].start_time = (uint64_t)t_start; B.progress[j].filled = 0; B.progress[j].queue_size = 0; }
            HostPlan* p = find_plan(ctx, at_level(B.s, E.level), E.view);
            if (!p) { todo[E.level].push_back(j); continue; }
            if (recon) { E.plan = std::move(*p); ctx->plans.erase(E.view); ctx->plan_info.n_prepared++; }
            else E.plan = *p;
            if (B.progress) B.progress[j].status = 2;
        }
    }
    for (auto& [level, todo_l] : todo) {
        const b200mvs_settings sl = at_level(B.s, level);
        std::vector<PL::PlanView> views;
        const PL::PlanInput in = plan_input(ctx, sl, views);
        if (recon) {
            if (int rc = plan_on_device(ctx, sl, in, B, todo_l)) return rc;
            ctx->plan_info.n_host += todo_l.size();
        }
        make_plans(in, sl, B, todo_l);
    }
    if (recon) ctx->plan_info.ms_plan = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    for (int j = 0; j < n_refs; ++j) {
        BatchEntry& E = B.e[j];
        if (E.plan.gsel.empty()) { B.failed = j; return fail(B200MVS_ERR_GLOBAL_VS, "Global View Selection failed"); }
        const HostLevel& L = ctx->views[E.view].lv[E.level];
        E.ws = Workspace(B.s, ctx->frontier_cap);
        E.ws.px = (size_t)L.w * L.h;
        E.ws.tiles = (size_t)((L.w + 15) / 16) * ((L.h + 15) / 16);
        E.ws.seeds = E.plan.seeds.size() + prior_bound(ctx->views[E.view], E.level);
        E.ws.jobs = 1;
        E.need = E.plan.gsel;                    // ascending; the reference view is never selected
        E.need.insert(std::upper_bound(E.need.begin(), E.need.end(), E.view), E.view);
    }
    return 0;
}

// the views whose pyramids the entries js need, ascending
std::vector<int> views_of(const Batch& B, const std::vector<int>& js)
{
    std::vector<int> v;
    for (int j : js) v.insert(v.end(), B.e[j].need.begin(), B.e[j].need.end());
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    return v;
}

// b200mvs_working_set of the entries js: the pyramids they need, each once, and their workspace
uint64_t working_set_bytes(b200mvs_ctx* ctx, const Batch& B, const std::vector<int>& js)
{
    uint64_t pyr = 0;
    for (int v : views_of(B, js)) pyr += pyramid_bytes(ctx->views[v]);
    Workspace w(B.s, ctx->frontier_cap);
    for (int j : js) w.add(B.e[j].ws);
    return pyr + workspace_bytes(ctx, w);
}

// b200mvs_plan_batches: greedy, deterministic grouping (see the header) of the entries of B.  Returns the number of groups.
int plan_groups(b200mvs_ctx* ctx, Batch& B, uint64_t available, std::vector<int>& group_of)
{
    const int n = (int)B.e.size();
    std::vector<uint64_t> pyr_of(ctx->views.size(), 0);
    for (size_t v = 0; v < ctx->views.size(); ++v) if (ctx->views[v].valid) pyr_of[v] = pyramid_bytes(ctx->views[v]);
    group_of.assign(n, -1);
    std::vector<char> in_group(ctx->views.size(), 0);
    int n_groups = 0;
    for (int first = 0; first < n; ++first) {
        if (group_of[first] >= 0) continue;
        std::fill(in_group.begin(), in_group.end(), 0);
        Workspace gw(B.s, ctx->frontier_cap);
        uint64_t pyr = 0;
        int size = 0;
        auto added = [&](int j) { uint64_t a = 0; for (int v : B.e[j].need) if (!in_group[v]) a += pyr_of[v]; return a; };
        auto fits = [&](int j, uint64_t a) { Workspace t = gw; t.add(B.e[j].ws); return pyr + a + workspace_bytes(ctx, t) <= available; };
        auto take = [&](int j, uint64_t a) { group_of[j] = n_groups; gw.add(B.e[j].ws); pyr += a; for (int v : B.e[j].need) in_group[v] = 1; ++size; };
        const uint64_t a0 = added(first);
        if (!fits(first, a0)) {
            B.failed = first;
            Workspace t = gw; t.add(B.e[first].ws);
            return fail(B200MVS_ERR_NO_MEMORY, "view %d needs %llu device bytes on its own, %llu are available", B.e[first].view,
                        (unsigned long long)(a0 + workspace_bytes(ctx, t)), (unsigned long long)available);
        }
        take(first, a0);
        while (size < MAX_GROUP_VIEWS) {
            int best = -1;
            uint64_t best_add = 0;
            for (int j = first + 1; j < n; ++j) {
                if (group_of[j] >= 0) continue;
                const uint64_t a = added(j);
                if (best >= 0 && a >= best_add) continue;
                if (fits(j, a)) { best = j; best_add = a; }
            }
            if (best < 0) break;
            take(best, best_add);
        }
        ++n_groups;
    }
    return n_groups;
}

// After a launch stopped with ST_GROW (host copy `c` of its control block): grows the frontier arrays from `cap` to
// max(2 x cap, c.need) entries - fewer when the budget allows fewer, never fewer than c.need - and copies what the resumed
// round still reads: the carried entries of list[1 - p] and the winners, results and `written` flags of the round.  The
// dead arrays (the consumed list[p], the other run list) are freed first, so the accounted bytes never exceed the final size.
int grow_frontier(b200mvs_ctx* ctx, const FrontierCtl& c, FrontierParams& P, size_t& cap, uint64_t reserve)
{
    const uint64_t need = c.need;
    const uint64_t room = headroom(ctx, reserve);   // the pyramids the group does not need may be evicted
    auto extra = [&](uint64_t n) {              // accounted bytes the frontier arrays add at n entries
        uint64_t b = 0;
        for_each_frontier_array(ctx, [&](auto& buf) { if (n > buf.cap) b += (n - buf.cap) * sizeof(*buf.p); });
        return b;
    };
    uint64_t n = std::max<uint64_t>(need, 2 * (uint64_t)cap);
    if (extra(n) > room) {
        uint64_t lo = cap, hi = n;               // extra(lo) = 0 <= room < extra(hi)
        while (hi - lo > 1) { const uint64_t mid = lo + (hi - lo) / 2; (extra(mid) <= room ? lo : hi) = mid; }
        if (lo < need)
            return fail(B200MVS_ERR_OVERFLOW, "frontier overflow: the next round needs %llu entries, the device budget allows %llu",
                        (unsigned long long)need, (unsigned long long)lo);
        n = lo;
    }
    const int p = c.resume_p;
    DevBuf<Entry>& live_list = p ? ctx->ent_a : ctx->ent_b;              // list[1 - p]
    DevBuf<Entry>& dead_list = p ? ctx->ent_b : ctx->ent_a;
    DevBuf<Entry>& live_run = c.resume_sorted ? ctx->run_sorted : ctx->run_in;
    DevBuf<Entry>& dead_run = c.resume_sorted ? ctx->run_in : ctx->run_sorted;
    const size_t n_run = (size_t)c.resume_nrun, carried = (size_t)c.nlist[1 - p];
    cudaStream_t st = ctx->stream.get();
    if (dead_list.cap < n) dead_list.release();
    if (dead_run.cap < n) dead_run.release();
    cudaError_t e = ctx->written.grow(n, n_run, st);
    if (e == cudaSuccess) e = ctx->run_out.grow(n, n_run, st);
    if (e == cudaSuccess) e = live_list.grow(n, carried, st);
    if (e == cudaSuccess) e = live_run.grow(n, n_run, st);
    if (e == cudaSuccess) e = dead_list.reserve(n);
    if (e == cudaSuccess) e = dead_run.reserve(n);
    if (e != cudaSuccess)
        return fail(B200MVS_ERR_OVERFLOW, "frontier overflow: the next round needs %llu entries, growing to %llu failed: %s",
                    (unsigned long long)need, (unsigned long long)n, cudaGetErrorString(e));
    P.list[0] = ctx->ent_a.p; P.list[1] = ctx->ent_b.p;
    P.run = ctx->run_in.p; P.run2 = ctx->run_sorted.p; P.res = ctx->run_out.p; P.written = ctx->written.p;
    P.cap = n;
    cap = (size_t)n;
    return 0;
}

// Removes from each entry's seeds those on a background pixel of its view's reconstruction mask at the entry's level, in
// place.  Host masks are read on the host; the seeds of every entry with a device mask are looked up by one
// k_seed_background launch.  The entries' workspaces keep counting every planned seed.
int seed_background(b200mvs_ctx* ctx, Batch& B)
{
    std::vector<SeedMask> views;
    std::vector<int4> seeds;
    for (BatchEntry& E : B.e) {
        const HostView& v = ctx->views[E.view];
        const HostLevel& L = v.lv[E.level];
        std::vector<PL::SeedOut>& q = E.plan.seeds;
        if (!v.mask.empty()) {
            q.erase(std::remove_if(q.begin(), q.end(), [&](const PL::SeedOut& p) { return background(v, L.w, L.h, p.x, p.y); }), q.end());
        } else if (v.mask_dev.p && !q.empty()) {
            for (const PL::SeedOut& p : q) seeds.push_back(make_int4(p.x, p.y, (int)views.size(), 0));
            views.push_back(SeedMask{v.mask_dev.p, v.mask_w, v.mask_h, L.w, L.h});
        }
    }
    if (seeds.empty()) return 0;
    DevBuf<SeedMask> d_views(ctx);
    DevBuf<int4> d_seeds(ctx);
    DevBuf<unsigned char> d_bg(ctx);
    CK(d_views.reserve(views.size()));
    CK(d_seeds.reserve(seeds.size()));
    CK(d_bg.reserve(seeds.size()));
    cudaStream_t st = ctx->stream.get();
    CK(cudaMemcpyAsync(d_views.p, views.data(), sizeof(SeedMask) * views.size(), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(d_seeds.p, seeds.data(), sizeof(int4) * seeds.size(), cudaMemcpyHostToDevice, st));
    k_seed_background<<<(unsigned)((seeds.size() + 255) / 256), 256, 0, st>>>(d_views.p, d_seeds.p, seeds.size(), d_bg.p);
    CK(cudaGetLastError());
    std::vector<unsigned char> flags(seeds.size());
    CK(cudaMemcpyAsync(flags.data(), d_bg.p, flags.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const unsigned char* bg = flags.data();
    for (BatchEntry& E : B.e) {
        if (!ctx->views[E.view].mask_dev.p) continue;          // a view has at most one kind of mask
        std::vector<PL::SeedOut>& q = E.plan.seeds;
        size_t n = 0;
        for (size_t i = 0; i < q.size(); ++i) if (!bg[i]) q[n++] = q[i];
        bg += q.size();
        q.resize(n);
    }
    return 0;
}

// The seed round's seeds are counted in an int (FrontierParams::n_seeds) and seed_key keeps a 32-bit index: a launch of the
// entries js holds at most INT_MAX feature seeds and prior candidate bounds.  Else B200MVS_ERR_INVALID_ARG, failing the
// last entry counted.
int check_seed_limit(Batch& B, const std::vector<int>& js)
{
    uint64_t n = 0;
    for (int j : js) {
        n += B.e[j].ws.seeds;
        if (n > (uint64_t)INT_MAX) {
            B.failed = j;
            return fail(B200MVS_ERR_INVALID_ARG, "a launch with view %d has %llu feature seeds and prior candidates, more than %d",
                        B.e[j].view, (unsigned long long)n, INT_MAX);
        }
    }
    return 0;
}

// Where a reconstruction's maps go: the caller's buffers (buffer_sink) or a point set.  Right after a group's launch,
// unless the whole group was cancelled, each view j gets its width and height in sizes[j] (when set) and, unless it was
// cancelled, take(j, job) runs while the group's maps and pyramids are resident.  take may allocate up to bytes(w, h)
// device bytes for a map of w x h pixels through the accounted allocator; every group's plan keeps that much free for
// the largest map of the batch.
struct MapSink {
    std::function<uint64_t(int w, int h)> bytes;
    std::function<int(int j, const JobParams& job)> take;
    b200mvs_maps* sizes = nullptr;
};

// One frontier launch over the entries B.e[j], j in js (at most MAX_GROUP_VIEWS): makes room for the pyramids they need
// within the budget (`reserve` bytes kept free for the sink), loads the missing ones, runs, hands the maps to `sink`.
// Accumulates `stats`; marks the entries that ended cancelled in `view_cancelled`.
int run_group(b200mvs_ctx* ctx, Batch& B, const std::vector<int>& js, const MapSink* sink, uint64_t reserve,
              b200mvs_stats* stats, std::vector<char>& view_cancelled)
{
    b200mvs_progress* progress = B.progress;
    // `if (progress.cancelled) return` at the head of every stage (dmrecon.cc:100-104,336): a group whose views were all
    // cancelled before it starts loads nothing and never runs
    if (progress && std::all_of(js.begin(), js.end(), [&](int j) { return progress[j].cancelled != 0; })) {
        for (int j : js) { progress[j].status = 5; view_cancelled[j] = 1; }
        return 0;
    }
    int rc = 0;
    const int n_refs = (int)js.size();
    cudaStream_t st = ctx->stream.get();
    std::memset(ctx->h_counters.get(), 0, sizeof(HostCounters));
    Workspace W(B.s, ctx->frontier_cap);
    for (int j : js) W.add(B.e[j].ws);
    WorkspaceInUse in_use(ctx);

    // make room: drop workspace larger than this group needs when the budget requires it, evict the pyramids the group does
    // not need (least recently used first), then load what it lacks
    const std::vector<int> need = views_of(B, js);
    pin_views(ctx, need);
    uint64_t missing = 0;
    for (int v : need) if (!ctx->views[v].has_image) missing += pyramid_bytes(ctx->views[v]);
    const uint64_t fixed = fixed_bytes(ctx);
    auto over = [&](uint64_t ws) { return fixed + ctx->pyr_resident + missing + ws + reserve > budget_limit(ctx); };
    if (over(workspace_grown_bytes(ctx, W))) shrink_workspace(ctx, W);
    const uint64_t ws = workspace_grown_bytes(ctx, W);
    while (over(ws) && evict_lru(ctx)) {}
    int32_t fv = -1;
    if ((rc = load_views(ctx, need, &fv))) {
        for (int j : js)
            if (std::binary_search(B.e[j].need.begin(), B.e[j].need.end(), (int)fv)) { B.failed = j; break; }
        return rc;
    }
    if ((rc = sync_view_params(ctx))) return rc;

    std::vector<JobParams> jobs(n_refs);
    std::vector<Entry> seeds;
    size_t total_px = 0, n_tiles = 0;
    std::vector<size_t> px_off(n_refs);
    bool masked = false;                   // a view of the group has a reconstruction mask
    for (int k = 0; k < n_refs; ++k) {
        const BatchEntry& E = B.e[js[k]];
        jobs[k] = make_job(ctx, E.level, E.view, E.plan.gsel);
        px_off[k] = total_px;
        total_px += (size_t)jobs[k].W * jobs[k].H;
        jobs[k].tiles_x = (jobs[k].W + 15) / 16;
        jobs[k].tile_base = (long long)n_tiles;
        n_tiles += (size_t)jobs[k].tiles_x * ((jobs[k].H + 15) / 16);
        masked = masked || ctx->views[E.view].masked();
        for (const PL::SeedOut& q : E.plan.seeds) {
            // a seed outside the image fails in the PatchSampler ctor (patch_sampler.cc:47-50); keep it so that the
            // processed count matches, the kernel rejects it by the same bounds test
            const int x = std::min(std::max(q.x, -1), 0xFFFE), y = std::min(std::max(q.y, -1), 0xFFFE);
            seeds.push_back(make_entry(pack_xy(x & 0xFFFF, y & 0xFFFF), k, 4, 0.f, q.depth, 0.f, 0.f, 0xFFFFFFFFu));
        }
    }

    // ---- device buffers: the sizes of b200mvs_working_set ----
    {
        cudaError_t e = cudaSuccess;
        for_each_workspace(ctx, W, [&](auto& buf, size_t n) { if (e == cudaSuccess) e = buf.reserve(n); });
        if (e != cudaSuccess)
            return fail(B200MVS_ERR_CUDA, "workspace of %llu bytes for %d reference views: %s",
                        (unsigned long long)workspace_bytes(ctx, W), n_refs, cudaGetErrorString(e));
    }
    unsigned char* base = ctx->maps.p;
    // sel first (8-byte alignment), then the float maps
    float* const conf = reinterpret_cast<float*>(base + total_px * 8) + total_px;
    const unsigned mask_blocks = (unsigned)((total_px + 255) / 256);
    {
        unsigned long long* sel = reinterpret_cast<unsigned long long*>(base);
        float* depth = conf - total_px;
        float* dz = conf + total_px;
        float* normal = dz + 2 * total_px;
        unsigned* slots = reinterpret_cast<unsigned*>(normal + 3 * total_px);
        for (int k = 0; k < n_refs; ++k) {
            jobs[k].sel = sel + px_off[k];
            jobs[k].depth = depth + px_off[k];
            jobs[k].conf = conf + px_off[k];
            jobs[k].dz = dz + 2 * px_off[k];
            jobs[k].normal = normal + 3 * px_off[k];
            jobs[k].slots = slots + px_off[k];
        }
        CK(cudaMemsetAsync(base, 0, total_px * (MAP_BYTES_PER_PX - 4), st));               // sel, depth, conf, dz, normal = 0
        CK(cudaMemsetAsync(slots, 0xFF, total_px * 4, st));
        if (masked) {
            // the background bytes of the masked views travel in the zeroed normal maps (12 bytes per pixel, one used),
            // so a mask adds no memory to the batch; k_mask_background zeroes them again.  A host mask is resampled on the
            // host and uploaded, a device mask is resampled in place by k_mark_background.
            unsigned char* bg_dev = reinterpret_cast<unsigned char*>(normal);
            std::vector<unsigned char> bg;
            for (int k = 0; k < n_refs; ++k) {
                const HostView& rv = ctx->views[B.e[js[k]].view];
                if (rv.mask_dev.p) {
                    const dim3 blk(32, 8), grd((jobs[k].W + 31) / 32, (jobs[k].H + 7) / 8);
                    k_mark_background<<<grd, blk, 0, st>>>(rv.mask_dev.p, rv.mask_w, rv.mask_h, jobs[k].W, jobs[k].H, bg_dev + px_off[k]);
                    CK(cudaGetLastError());
                    continue;
                }
                if (rv.mask.empty()) continue;
                bg.resize((size_t)jobs[k].W * jobs[k].H);
                mark_background(rv, jobs[k].W, jobs[k].H, bg.data());
                // pageable source: the call returns once `bg` has been read, so it may be refilled
                CK(cudaMemcpyAsync(bg_dev + px_off[k], bg.data(), bg.size(), cudaMemcpyHostToDevice, st));
            }
            k_mask_background<<<mask_blocks, 256, 0, st>>>(conf, bg_dev, total_px);
            CK(cudaGetLastError());
        }
    }
    size_t cap = W.cap();
    const bool thresholded = W.thresholded;
    CK(cudaMemsetAsync(ctx->tile_cnt.p, 0, sizeof(unsigned) * n_tiles, st));
    CK(ctx->d_settings.reserve(1));
    CK(ctx->ctl.reserve(1));
    CK(cudaMemsetAsync(ctx->job_run.p, 0, sizeof(unsigned long long) * n_refs, st));
    const DevSettings ds = to_dev(B.s);
    CK(cudaMemcpyAsync(ctx->d_jobs.p, jobs.data(), sizeof(JobParams) * n_refs, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(ctx->d_settings.p, &ds, sizeof(ds), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(ctx->counters.p, 0, sizeof(unsigned long long) * (C_NUM + n_refs), st));
    CK(cudaMemsetAsync(ctx->ctl.p, 0, sizeof(FrontierCtl), st));
    if (thresholded) CK(cudaMemsetAsync(ctx->hist.p, 0, sizeof(unsigned) * (size_t)n_refs * HIST_PER_JOB, st));
    if (!seeds.empty()) CK(cudaMemcpyAsync(ctx->run_in.p, seeds.data(), sizeof(Entry) * seeds.size(), cudaMemcpyHostToDevice, st));
    HostMirror* mirror = ctx->h_mirror.get();
    std::memset(mirror, 0, sizeof(HostMirror) + (sizeof(unsigned long long) + sizeof(int)) * n_refs);
    volatile unsigned long long* m_filled = reinterpret_cast<volatile unsigned long long*>(mirror + 1);
    volatile int* m_cancel_job = reinterpret_cast<volatile int*>(m_filled + n_refs);
    CK(cudaMemsetAsync(ctx->job_cancel.p, 0, sizeof(int) * n_refs, st));
    // the prior seeds follow the feature seeds in run_in; the launch reads their number back once.  Their cursor is
    // counters[C_TICKET], the ticket of k_optimize, which the frontier kernels do not use: it is zeroed again after.
    size_t n_prior = 0;
    if (std::any_of(js.begin(), js.end(), [&](int j) { return ctx->views[B.e[j].view].prior.p != nullptr; })) {
        unsigned long long* cursor = ctx->counters.p + C_TICKET;
        for (int k = 0; k < n_refs; ++k) {
            const HostView& rv = ctx->views[B.e[js[k]].view];
            const size_t n = prior_bound(rv, B.e[js[k]].level);
            if (n == 0) continue;
            k_prior_seeds<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(rv.prior.p, rv.prior_dz.p, rv.prior_ids.p, rv.prior_w,
                rv.prior_h, rv.prior_stride, prior_cells(jobs[k].W, rv.prior_stride), n, jobs[k], B.s.nr_recon_neighbors, k,
                ctx->run_in.p + seeds.size(), cursor);
            CK(cudaGetLastError());
        }
        unsigned long long* h_count = &ctx->h_counters->count[C_TICKET];
        CK(cudaMemcpyAsync(h_count, cursor, sizeof(*h_count), cudaMemcpyDeviceToHost, st));
        CK(cudaMemsetAsync(cursor, 0, sizeof(*cursor), st));
        CK(cudaStreamSynchronize(st));
        n_prior = (size_t)*h_count;
        if (stats) stats->n_seeds_processed += n_prior;
    }

    FrontierParams P;
    P.list[0] = ctx->ent_a.p; P.list[1] = ctx->ent_b.p;
    P.run = ctx->run_in.p; P.res = ctx->run_out.p; P.written = ctx->written.p;
    P.run2 = ctx->run_sorted.p; P.tile_cnt = ctx->tile_cnt.p; P.tile_off = ctx->tile_off.p;
    P.n_tiles = (long long)n_tiles;
    P.cap = cap; P.n_seeds = (int)(seeds.size() + n_prior); P.n_jobs = n_refs;
    P.st = ctx->d_settings.p; P.jobs = ctx->d_jobs.p; P.views = ctx->d_views.p; P.lut = ctx->d_lut.p;
    P.counters = ctx->counters.p; P.ctl = ctx->ctl.p; P.hist = ctx->hist.p; P.thr_bin = ctx->thr_bin.p;
    P.host = mirror; P.host_filled = m_filled; P.host_cancel_job = m_cancel_job; P.job_cancel = ctx->job_cancel.p; P.job_run = ctx->job_run.p;
    P.thread_min = ctx->thread_min >= 0 ? ctx->thread_min : OPT_THREAD_MIN;
    P.band_bins = B.s.frontier_band > 0.f ? std::max(1, (int)(B.s.frontier_band * (float)HIST_FINE)) : 0;
    P.topk = (int)std::min<uint32_t>(B.s.frontier_topk, 1u << 30);
    P.first_list = 1;

    // views cancelled before the launch never start
    std::vector<char> job_cancelled(n_refs, 0);
    if (progress) for (int k = 0; k < n_refs; ++k) if (progress[js[k]].cancelled) { job_cancelled[k] = 1; m_cancel_job[k] = 1; }
    // ---- one cooperative launch: seeds + all frontier rounds (DESIGN.md "Frontier schedule"); when the frontier arrays
    // have to grow, the stopped round is finished by k_frontier_resume and a new launch goes on from the round after it ----
    if ((rc = prepare_kernels(ctx))) return rc;
    ctx->fr_initial = std::max<uint64_t>(ctx->fr_initial, cap);
    FrontierCtl* h_ctl = &ctx->h_counters->ctl;
    float ms_all = 0.f;
    uint64_t n_launches = 0, n_resumes = 0;
    for (;;) {
        cudaEvent_t ev_begin = ctx->ev_begin.get(), ev_end = ctx->ev_end.get();
        CK(cudaEventRecord(ev_begin, st));
        {
            void* args[] = {(void*)&P};
            if (n_resumes > 0) {
                const unsigned long long n_run = h_ctl->resume_nrun;
                k_frontier_resume<<<(unsigned)std::max<unsigned long long>(1ull, (n_run + 255) / 256), 256, 0, st>>>(P);
                CK(cudaGetLastError());
            }
            CK(cudaLaunchCooperativeKernel((const void*)k_frontier, dim3(ctx->frontier_grid), dim3(OPT_TPB), args, OPT_SMEM_BYTES, st));
        }
        CK(cudaEventRecord(ev_end, st));
        CK(cudaMemcpyAsync(ctx->h_counters->count, ctx->counters.p, sizeof(unsigned long long) * (C_NUM + n_refs), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(h_ctl, ctx->ctl.p, sizeof(FrontierCtl), cudaMemcpyDeviceToHost, st));
        cudaEvent_t ev_copied = ctx->ev_copied.get();
        CK(cudaEventRecord(ev_copied, st));
        // While the kernel runs the host only relays: progress out (Progress::filled / queueSize, fancy_progress_printer.cc:84-91)
        // and cancel requests in (imageoperations.cc:177-184): a cancelled view's queue is dropped at the next round, the other
        // views of the batch go on; when every view is cancelled the kernel stops.
        if (progress) {
            for (;;) {
                const cudaError_t q = cudaEventQuery(ev_copied);
                if (q == cudaSuccess) break;
                if (q != cudaErrorNotReady) return fail(B200MVS_ERR_CUDA, "frontier kernel: %s", cudaGetErrorString(q));
                const unsigned long long qs = mirror->queue;
                int n_c = 0;
                for (int k = 0; k < n_refs; ++k) {
                    b200mvs_progress& pg = progress[js[k]];
                    if (pg.cancelled) { job_cancelled[k] = 1; m_cancel_job[k] = 1; }
                    if (job_cancelled[k]) { ++n_c; continue; }
                    pg.status = 3;
                    pg.filled = m_filled[k];
                    pg.queue_size = qs;
                }
                if (n_c == n_refs) mirror->cancel = 1;
                std::this_thread::sleep_for(std::chrono::microseconds(200));
            }
        }
        CK(cudaStreamSynchronize(st));
        ++n_launches;
        float ms = 0.f;
        cudaEventElapsedTime(&ms, ev_begin, ev_end);
        ms_all += ms;
        // a batch whose views are all cancelled is not resumed: it ends cancelled like a kernel that stopped by itself
        if (h_ctl->stop != ST_GROW || mirror->cancel) break;
        if ((rc = grow_frontier(ctx, *h_ctl, P, cap, reserve))) return rc;
        ++n_resumes;
        ctx->fr_resumes++;
        P.first_list = h_ctl->resume_p ^ 1;
        P.n_seeds = 0;
    }
    ctx->fr_final = std::max<uint64_t>(ctx->fr_final, cap);
    if (masked) {
        k_unmask_background<<<mask_blocks, 256, 0, st>>>(conf, total_px);
        CK(cudaGetLastError());
    }
    if (progress) for (int k = 0; k < n_refs; ++k) if (progress[js[k]].cancelled) job_cancelled[k] = 1;
    const bool cancelled = h_ctl->stop == ST_CANCELLED || std::all_of(job_cancelled.begin(), job_cancelled.end(), [](char c) { return c != 0; });
    if (ctx->h_counters->count[C_OVERFLOW] || h_ctl->stop == ST_OVERFLOW)
        return fail(B200MVS_ERR_OVERFLOW, "frontier buffer overflow (capacity %zu entries)", cap);
    if (stats) stats->n_seeds_success += ctx->h_counters->count[C_SEED_OK];

    // ---- results ----
    if (sink && !cancelled)
        for (int k = 0; k < n_refs; ++k) {
            const int j = js[k];
            if (sink->sizes) { sink->sizes[j].width = jobs[k].W; sink->sizes[j].height = jobs[k].H; }
            if (job_cancelled[k]) continue;                  // RECON_CANCELLED: nothing is saved (dmrecon.cc:100-104)
            if (progress) progress[j].status = 4;
            if ((rc = sink->take(j, jobs[k]))) { B.failed = j; return rc; }
        }
    CK(cudaStreamSynchronize(st));
    uint64_t filled = 0;
    for (int k = 0; k < n_refs; ++k) {
        const int j = js[k];
        filled += ctx->h_counters->count[C_NUM + k];
        if (cancelled || job_cancelled[k]) view_cancelled[j] = 1;
        if (progress) { progress[j].filled = ctx->h_counters->count[C_NUM + k]; progress[j].queue_size = 0; progress[j].status = (cancelled || job_cancelled[k]) ? 5 : 0; }
    }
    if (stats) {
        stats->n_opt += ctx->h_counters->count[C_OPTS];
        stats->n_sample_sets += ctx->h_counters->count[C_SETS];
        stats->n_rounds += h_ctl->rounds;
        stats->n_filled += filled;
        stats->n_entries_peak = std::max<uint64_t>(stats->n_entries_peak, h_ctl->peak);
        stats->n_patch_launches += n_launches;
        stats->n_kernel_launches += n_launches + n_resumes;
        // the optimise phases inside the persistent kernel, by %globaltimer of CTA 0 between the grid barriers
        double ns_all = 0.0;
        for (int k = 0; k < PH_NUM; ++k) ns_all += (double)h_ctl->ns[k];
        const double ns_opt = (double)h_ctl->ns[PH_OPT] + (double)h_ctl->ns[PH_SEED] + (double)h_ctl->ns[PH_OPT_THREAD];
        stats->ms_patch_kernel += ms_all;
        stats->ms_total_device += ms_all;
        stats->ms_optimise_phases += ns_all > 0.0 ? ms_all * ns_opt / ns_all : 0.0;
        stats->n_grid_barriers += h_ctl->barriers;
        stats->ms_optimise_thread_phases += ns_all > 0.0 ? ms_all * (double)h_ctl->ns[PH_OPT_THREAD] / ns_all : 0.0;
        stats->ms_sort_phases += ns_all > 0.0 ? ms_all * (double)h_ctl->ns[PH_SORT] / ns_all : 0.0;
    }
    return 0;
}

// The start of every reconstruction, before anything is planned: without a budget the whole batch is one launch (with
// one, the limit applies per group), and the call's statistics, frontier and planning records start from zero.  The host
// entry points begin before they check their entries, b200mvs_reconstruct[_levels]_device after its buffer checks.
int begin_reconstruction(b200mvs_ctx* ctx, int n_refs, b200mvs_stats* stats)
{
    if (!ctx->mem.budget && n_refs > MAX_GROUP_VIEWS) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_reconstruct: bad arguments");
    if (stats) std::memset(stats, 0, sizeof(*stats));
    ctx->fr_initial = ctx->fr_final = ctx->fr_resumes = 0;
    ctx->plan_info = b200mvs_plan_info{};
    return 0;
}

// The reconstruction of the checked batch B, with the context locked and a device: each entry's maps go to the sink after
// its group's launch, and no group plans into the sink's bytes for the largest map of the batch; without a sink they stay
// on the device, one group only.
int run_batch(b200mvs_ctx* ctx, Batch& B, const MapSink* sink, b200mvs_stats* stats)
{
    const int n_refs = (int)B.e.size();
    const PinsOfCall pins(ctx);                  // each group pins the views it needs (run_group)
    int rc = plan_batch(ctx, B, true);
    if (rc) return rc;
    for (int j = 0; j < n_refs; ++j)
        if ((rc = check_seed_limit(B, {j}))) return rc;
    // an image that is missing and cannot be fetched fails the call before anything runs
    if (!has_source(ctx))
        for (int j = 0; j < n_refs; ++j) {
            if (!ctx->views[B.e[j].view].has_image) { B.failed = j; return fail(B200MVS_ERR_INVALID_ARG, "color image of view %d is not loaded", B.e[j].view); }
            for (int g : B.e[j].plan.gsel)
                if (!ctx->views[g].has_image) { B.failed = j; return fail(B200MVS_ERR_INVALID_ARG, "color image of view %d (selected neighbour of view %d) is not loaded", g, B.e[j].view); }
        }
    CK(cudaSetDevice(ctx->device));
    if ((rc = seed_background(ctx, B))) return rc;
    if (stats) for (const BatchEntry& E : B.e) stats->n_seeds_processed += E.plan.seeds.size();

    // ---- groups that fit the budget, one frontier launch each ----
    uint64_t reserve = 0;
    if (sink)
        for (const BatchEntry& E : B.e) {
            const HostLevel& L = ctx->views[E.view].lv[E.level];
            reserve = std::max(reserve, sink->bytes(L.w, L.h));
        }
    const uint64_t fixed = fixed_bytes(ctx), limit = budget_limit(ctx);
    std::vector<int> group_of;
    const int n_groups = plan_groups(ctx, B, limit > fixed + reserve ? limit - fixed - reserve : 0, group_of);
    if (n_groups < 0) return n_groups;
    if (!sink && n_groups > 1)
        return fail(B200MVS_ERR_INVALID_ARG, "maps == NULL keeps the results on the device, but the budget splits the batch into %d launches", n_groups);
    ctx->mem.n_groups = (uint64_t)n_groups;
    std::vector<std::vector<int>> group_js(n_groups);
    for (int j = 0; j < n_refs; ++j) group_js[group_of[j]].push_back(j);
    for (const std::vector<int>& js : group_js)
        if ((rc = check_seed_limit(B, js))) return rc;
    std::vector<char> view_cancelled(n_refs, 0);
    for (const std::vector<int>& js : group_js) {
        if ((rc = run_group(ctx, B, js, sink, reserve, stats, view_cancelled))) return rc;
    }
    if (std::all_of(view_cancelled.begin(), view_cancelled.end(), [](char c) { return c != 0; }))
        return fail(B200MVS_ERR_CANCELLED, "reconstruction cancelled");
    return 0;
}

// A reconstruction of b200mvs_reconstruct[_levels] or b200mvs_pset_add_reconstruction[_levels], with the context locked
// and a device.  levels: the level of each entry, or NULL for s->scale everywhere (check_batch).
int reconstruct(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                const MapSink* sink, b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view)
{
    int rc = begin_reconstruction(ctx, n_refs, stats);
    if (rc) return rc;
    Batch B;
    if (!(rc = check_batch(ctx, s, n_refs, refs, levels, progress, B))) rc = run_batch(ctx, B, sink, stats);
    return B.report(rc, failed_view);
}

// The sink into the caller's buffers `maps` (host memory, or with on_device the context's device): copies on ctx->stream,
// view ids decoded on the host or by k_slots_to_ids.  The buffers are not the context's, so it reserves no budget.
MapSink buffer_sink(b200mvs_ctx* ctx, b200mvs_maps* maps, bool on_device)
{
    MapSink sink;
    sink.sizes = maps;
    sink.bytes = [](int, int) { return (uint64_t)0; };
    sink.take = [ctx, maps, on_device, hslots = std::vector<unsigned>()](int j, const JobParams& J) mutable {
        const b200mvs_maps& m = maps[j];
        const size_t np = (size_t)J.W * J.H;
        const cudaStream_t st = ctx->stream.get();
        const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
        if (m.depth) CK(cudaMemcpyAsync(m.depth, J.depth, np * 4, kind, st));
        if (m.conf) CK(cudaMemcpyAsync(m.conf, J.conf, np * 4, kind, st));
        if (m.dz) CK(cudaMemcpyAsync(m.dz, J.dz, np * 8, kind, st));
        if (m.normal) CK(cudaMemcpyAsync(m.normal, J.normal, np * 12, kind, st));
        if (m.view_ids && on_device) {
            k_slots_to_ids<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(J, m.view_ids, reinterpret_cast<uintptr_t>(m.view_ids) % 16 == 0);
            CK(cudaGetLastError());
        } else if (m.view_ids) {
            hslots.resize(np);
            CK(cudaMemcpyAsync(hslots.data(), J.slots, np * 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            for (size_t p = 0; p < np; ++p) slots_to_ids(J.gview, J.n_global, hslots[p], m.view_ids + 4 * p);
        }
        return 0;
    };
    return sink;
}

// The C ABI's reconstructions, for the entry point named `fn`: levels is NULL for b200mvs_reconstruct,
// b200mvs_reconstruct_device and b200mvs_pset_add_reconstruction, and the level of each entry for their *_levels forms.
int reconstruct_host(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                     b200mvs_maps* maps, b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view)
{
    std::lock_guard<std::mutex> lk(ctx->mtx);
    int rc = require_device(ctx);
    if (rc) return rc;
    if (!maps) return reconstruct(ctx, s, n_refs, refs, levels, nullptr, progress, stats, failed_view);
    const MapSink sink = buffer_sink(ctx, maps, false);
    return reconstruct(ctx, s, n_refs, refs, levels, &sink, progress, stats, failed_view);
}

int reconstruct_device(const char* fn, b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs,
                       const int32_t* levels, b200mvs_maps* maps_dev, void* cuda_stream, b200mvs_progress* progress,
                       b200mvs_stats* stats, int32_t* failed_view)
{
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (!maps_dev) return fail(B200MVS_ERR_INVALID_ARG, "%s: maps_dev is NULL", fn);
    Batch B;
    int rc = check_batch(ctx, s, n_refs, refs, levels, progress, B);
    if (rc && B.e.empty()) return rc;            // a settings or argument error names no view: failed_view is left as it was
    auto run = [&]() {
        if ((rc = require_device(ctx))) return rc;
        // every buffer is checked before anything runs
        CK(cudaSetDevice(ctx->device));
        for (int j = 0; j < n_refs; ++j) {
            const b200mvs_maps& m = maps_dev[j];
            auto what = [&](const char* field) { return "maps_dev[" + std::to_string(j) + "]." + field + " (view " + std::to_string(refs[j]) + ")"; };
            if (!m.depth) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s is NULL", fn, what("depth").c_str());
            const std::pair<const void*, const char*> bufs[] = {{m.depth, "depth"}, {m.conf, "conf"}, {m.dz, "dz"}, {m.normal, "normal"},
                                                                {m.view_ids, "view_ids"}};
            for (const auto& b : bufs)
                if (b.first && (rc = check_device_buffer(fn, what(b.second), b.first, ctx->device, 4))) return rc;
        }
        if ((rc = wait_for_stream(ctx->ev_caller.get(), cuda_stream, ctx->stream.get()))) return rc;
        if ((rc = begin_reconstruction(ctx, n_refs, stats))) return rc;
        const MapSink sink = buffer_sink(ctx, maps_dev, true);
        return run_batch(ctx, B, &sink, stats);
    };
    return B.report(rc ? rc : run(), failed_view);
}

int pset_add_reconstruction(const char* fn, b200mvs_pset* ps, b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs,
                            const int32_t* refs, const int32_t* levels, b200mvs_progress* progress, b200mvs_stats* stats,
                            int32_t* failed_view, b200mvs_pset_view* views_out)
{
    namespace PD = b200mvs_pset_dev;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (failed_view) *failed_view = -1;
    if (ctx->device == B200MVS_DEVICE_NONE)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: a planning context (B200MVS_DEVICE_NONE) cannot reconstruct", fn);
    if (int rc = PD::check(ps, ctx->device)) return rc;
    // the handle's workspace lives in the context's budget for the duration of the call
    const PD::Allocator A{ctx, [](void* c, void** p, size_t n) { return dev_alloc(static_cast<b200mvs_ctx*>(c), p, n); },
                          [](void* c, void* p, size_t n) { dev_free(static_cast<b200mvs_ctx*>(c), p, n); }};
    std::vector<PD::Block> blocks(std::max(n_refs, 0));
    MapSink sink;
    sink.bytes = [&](int w, int h) { return PD::workspace_bytes(ps, w, h); };
    sink.take = [&](int j, const JobParams& J) {
        // the camera the view was registered with: scene2pset forms the calibration from it and the map's size; the colours
        // are the job's reference level, the level of the entry
        const HostView& v = ctx->views[refs[j]];
        b200mvs_pset_camera cam;
        cam.flen = v.flen; cam.paspect = v.paspect; cam.ppoint[0] = v.pp[0]; cam.ppoint[1] = v.pp[1];
        std::memcpy(cam.rot, v.rot, sizeof(cam.rot));
        std::memcpy(cam.trans, v.trans, sizeof(cam.trans));
        const int rc = PD::extract(ps, refs[j], J.depth, J.W, J.H, J.ref_img, J.ref_pitch, cam, blocks[j]);
        return rc ? fail(rc, "view %d: %s", refs[j], last_error.c_str()) : 0;
    };
    struct UsingAllocator {
        b200mvs_pset* ps;
        UsingAllocator(b200mvs_pset* p, const PD::Allocator* a) : ps(p) { PD::use_allocator(ps, a); }
        ~UsingAllocator() { PD::use_allocator(ps, nullptr); }
    };
    int rc;
    {
        const UsingAllocator using_ctx(ps, &A);
        rc = reconstruct(ctx, s, n_refs, refs, levels, &sink, progress, stats, failed_view);
    }
    if (rc) { PD::discard(ps); return rc; }
    return PD::commit(ps, blocks, views_out);
}

// b200mvs_working_set and b200mvs_plan_batches (group_of_ref != NULL), with levels as for reconstruct_host
int working_set(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels, uint64_t* bytes)
{
    std::lock_guard<std::mutex> lk(ctx->mtx);
    Batch B;
    int rc = check_batch(ctx, s, n_refs, refs, levels, nullptr, B);
    if (rc || (rc = plan_batch(ctx, B, false))) return rc;
    std::vector<int> js(n_refs);
    for (int j = 0; j < n_refs; ++j) js[j] = j;
    *bytes = working_set_bytes(ctx, B, js);
    return 0;
}

int plan_batches(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                 uint64_t available, int32_t* group_of_ref, int32_t* failed_view)
{
    std::lock_guard<std::mutex> lk(ctx->mtx);
    Batch B;
    std::vector<int> group_of;
    int rc = check_batch(ctx, s, n_refs, refs, levels, nullptr, B);
    if (!rc) rc = plan_batch(ctx, B, false);
    if (!rc && (rc = plan_groups(ctx, B, available, group_of)) > 0) std::copy(group_of.begin(), group_of.end(), group_of_ref);
    return B.report(rc, failed_view);           // rc: the number of groups, or the error
}

} // namespace

extern "C" {

int b200mvs_reconstruct(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs,
                        b200mvs_maps* maps, b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    return reconstruct_host(ctx, s, n_refs, refs, nullptr, maps, progress, stats, failed_view);
}

int b200mvs_reconstruct_levels(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                               b200mvs_maps* maps, b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    if (int rc = check_levels("b200mvs_reconstruct_levels", levels, failed_view)) return rc;
    return reconstruct_host(ctx, s, n_refs, refs, levels, maps, progress, stats, failed_view);
}

int b200mvs_reconstruct_device(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, b200mvs_maps* maps_dev,
                               void* cuda_stream, b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view)
{
    static const char* fn = "b200mvs_reconstruct_device";
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    return reconstruct_device(fn, ctx, s, n_refs, refs, nullptr, maps_dev, cuda_stream, progress, stats, failed_view);
}

int b200mvs_reconstruct_levels_device(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs,
                                      const int32_t* levels, b200mvs_maps* maps_dev, void* cuda_stream, b200mvs_progress* progress,
                                      b200mvs_stats* stats, int32_t* failed_view)
{
    static const char* fn = "b200mvs_reconstruct_levels_device";
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    if (int rc = check_levels(fn, levels, failed_view)) return rc;
    return reconstruct_device(fn, ctx, s, n_refs, refs, levels, maps_dev, cuda_stream, progress, stats, failed_view);
}

int b200mvs_pset_add_reconstruction(b200mvs_pset* ps, b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs,
                                    b200mvs_progress* progress, b200mvs_stats* stats, int32_t* failed_view, b200mvs_pset_view* views_out)
{
    static const char* fn = "b200mvs_pset_add_reconstruction";
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    return pset_add_reconstruction(fn, ps, ctx, s, n_refs, refs, nullptr, progress, stats, failed_view, views_out);
}

int b200mvs_pset_add_reconstruction_levels(b200mvs_pset* ps, b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs,
                                           const int32_t* refs, const int32_t* levels, b200mvs_progress* progress,
                                           b200mvs_stats* stats, int32_t* failed_view, b200mvs_pset_view* views_out)
{
    static const char* fn = "b200mvs_pset_add_reconstruction_levels";
    if (!ctx) return fail(B200MVS_ERR_INVALID_ARG, "%s: null context", fn);
    if (int rc = check_levels(fn, levels, failed_view)) return rc;
    return pset_add_reconstruction(fn, ps, ctx, s, n_refs, refs, levels, progress, stats, failed_view, views_out);
}

int b200mvs_working_set(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, uint64_t* bytes)
{
    if (!ctx || !bytes) return B200MVS_ERR_INVALID_ARG;
    return working_set(ctx, s, n_refs, refs, nullptr, bytes);
}

int b200mvs_working_set_levels(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                               uint64_t* bytes)
{
    if (!ctx || !bytes) return B200MVS_ERR_INVALID_ARG;
    if (int rc = check_levels("b200mvs_working_set_levels", levels, nullptr)) return rc;
    return working_set(ctx, s, n_refs, refs, levels, bytes);
}

int b200mvs_plan_batches(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, uint64_t available,
                         int32_t* group_of_ref, int32_t* failed_view)
{
    if (!ctx || !group_of_ref) return B200MVS_ERR_INVALID_ARG;
    return plan_batches(ctx, s, n_refs, refs, nullptr, available, group_of_ref, failed_view);
}

int b200mvs_plan_batches_levels(b200mvs_ctx* ctx, const b200mvs_settings* s, int n_refs, const int32_t* refs, const int32_t* levels,
                                uint64_t available, int32_t* group_of_ref, int32_t* failed_view)
{
    if (!ctx || !group_of_ref) return B200MVS_ERR_INVALID_ARG;
    if (int rc = check_levels("b200mvs_plan_batches_levels", levels, failed_view)) return rc;
    return plan_batches(ctx, s, n_refs, refs, levels, available, group_of_ref, failed_view);
}

} // extern "C"

namespace {

// Installs the context's one image source (host or device; both NULL removes it) with its budget
int set_source(b200mvs_ctx* ctx, b200mvs_fetch_fn fetch, b200mvs_device_fetch_fn fetch_device, b200mvs_release_fn release,
               void* user, uint64_t budget_bytes)
{
    if (!ctx) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    if (int rc = require_device(ctx)) return rc;
    CK(cudaSetDevice(ctx->device));
    if (!fetch && !fetch_device) {
        ctx->fetch = nullptr; ctx->fetch_device = nullptr; ctx->release = nullptr; ctx->user = nullptr; ctx->mem.budget = 0;
        return 0;
    }
    if (budget_bytes == 0) {
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        budget_bytes = (uint64_t)((double)free_b * 0.9);
    }
    ctx->fetch = fetch; ctx->fetch_device = fetch_device; ctx->release = release; ctx->user = user;
    ctx->mem.budget = budget_bytes;
    make_room(ctx, 0);                 // idle workspace and then pyramids go until the resident bytes fit
    ctx->mem.peak = ctx->mem.resident;
    return 0;
}

} // namespace

extern "C" {

int b200mvs_set_image_source(b200mvs_ctx* ctx, b200mvs_fetch_fn fetch, b200mvs_release_fn release, void* user, uint64_t budget_bytes)
{
    return set_source(ctx, fetch, nullptr, release, user, budget_bytes);
}

int b200mvs_set_image_source_device(b200mvs_ctx* ctx, b200mvs_device_fetch_fn fetch, b200mvs_release_fn release, void* user,
                                    uint64_t budget_bytes)
{
    return set_source(ctx, nullptr, fetch, release, user, budget_bytes);
}

int b200mvs_plan_stats(b200mvs_ctx* ctx, b200mvs_plan_info* out)
{
    if (!ctx || !out) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    *out = ctx->plan_info;
    return 0;
}

int b200mvs_memory_stats(b200mvs_ctx* ctx, b200mvs_memory* out)
{
    if (!ctx || !out) return B200MVS_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> lk(ctx->mtx);
    *out = ctx->mem;
    out->fixed = fixed_bytes(ctx);
    return 0;
}

} // extern "C"
