// Drop-in replacement for the reference's libmve_dmrecon.a: the class mvs::DMRecon with the reference's OWN header
// (libs/dmrecon/dmrecon.h:40-68, included from the reference tree at build time - nothing is copied into this repo),
// implemented as a thin host shim over the C ABI of libb200mvs.so (include/b200mvs.h).
//
// apps/dmrecon/dmrecon.cc and fancy_progress_printer.* compile and link UNCHANGED against this (shim/Makefile):
//   mvs::DMRecon recon(scene, settings); recon.start(); recon.getProgress(); recon.getRefViewNr();
// Everything below the boundary that is I/O stays the reference's (mve::Scene / mve::View / mve::Bundle, libmve.a).
//
// What the shim does, mirroring dmrecon.cc:
//   ctor  (dmrecon.cc:30-87)   same argument validation and exception types/messages; width/height of the scaled image
//   start (dmrecon.cc:90-172)  views + bundle -> b200mvs context (cached per scene like ImagePyramidCache,
//                              image_pyramid.cc:99-132), b200mvs_reconstruct, results attached with View::set_image
//                              under the reference's embedding names (depth-L<s>, dz-L<s>, conf-L<s>, undist-L<s>),
//                              writePlyFile / plyPath through the reference's own save_ply_view, same log lines, Progress
//                              updated live while the kernel runs, cancellation of a running view -> RECON_CANCELLED
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <iostream>
#include <map>
#include <memory>
#include <mutex>
#include <sstream>
#include <string>
#include <stdexcept>
#include <thread>
#include <vector>

#include "dmrecon/dmrecon.h"
#include "dmrecon/settings.h"
#include "mve/image.h"
#include "mve/image_tools.h"
#include "mve/mesh_io_ply.h"
#include "util/file_system.h"
#include "util/string_utils.h"

#include "b200mvs.h"

namespace {

// One device context per (scene, embedding) AND per GPU, shared by all DMRecon objects of the process - the reference
// shares its image pyramids the same way through ImagePyramidCache's statics (image_pyramid.cc:157-160).
//
// The reference driver runs DMRecon::start() concurrently from OpenMP threads (apps/dmrecon/dmrecon.cc:285).  Here the
// concurrent calls are (i) spread round-robin over the GPUs named by B200MVS_DEVICES (default: device B200MVS_DEVICE or
// 0) and (ii) per GPU COMBINED: every caller only ENQUEUES its request; one of them becomes the leader, waits a short
// collection window for the other threads of the OpenMP team to arrive, then does for the whole batch what each DMRecon
// does for itself in the reference - global view selection - and submits ONE b200mvs_reconstruct in which all views
// advance together; the library loads the colour images the batch needs and splits it into launches that fit the device
// budget.  While the kernel runs a
// relay thread copies the live progress into every caller's mvs::Progress and forwards cancel requests.
struct Request {
    int32_t ref = 0;
    b200mvs_settings settings;
    b200mvs_maps maps;
    mvs::Progress* progress = nullptr;      // the caller's DMRecon::progress (read by progress printers / UMVE while we run)
    std::string embedding;
    bool quiet = true;
    b200mvs_stats stats;
    std::vector<int32_t> gvs;
    int rc = 0;
    std::string err;
    bool done = false;
};

struct DeviceCtx {
    std::mutex mtx;                 // protects everything below
    std::condition_variable cv;
    int device = 0;
    mve::Scene::Ptr scene;
    std::string embedding;
    b200mvs_ctx* ctx = nullptr;
    std::map<int, mve::ByteImage::Ptr> held;   // images the library fetched and has not released yet (image source)
    bool features_set = false;
    bool cameras_set = false;
    std::vector<char> masks_set;    // views whose B200MVS_RECON_MASK embedding has been read
    std::vector<char> priors_set;   // views whose B200MVS_PRIOR embedding has been read
    bool leader_active = false;
    int planners = 0;               // callers that run their global view selection right now and will enqueue next
    std::vector<Request*> pending;
    uint64_t arrivals = 0;          // bumped by every enqueue: the leader's collection window watches it
    size_t last_batch = 0;          // size of the previous batch = how many callers to expect
    ~DeviceCtx() { if (ctx) b200mvs_destroy(ctx); }
};

std::mutex g_mtx;
std::vector<std::unique_ptr<DeviceCtx>> g_devices;
std::atomic<unsigned> g_next(0);
std::mutex g_cout;

std::vector<int> device_list()
{
    std::vector<int> out;
    if (const char* e = std::getenv("B200MVS_DEVICES")) {
        std::string s(e);
        size_t pos = 0;
        while (pos < s.size()) {
            size_t q = s.find(',', pos);
            if (q == std::string::npos) q = s.size();
            if (q > pos) out.push_back(std::atoi(s.substr(pos, q - pos).c_str()));
            pos = q + 1;
        }
    }
    if (out.empty()) {
        const char* e = std::getenv("B200MVS_DEVICE");
        out.push_back(e ? std::atoi(e) : 0);
    }
    return out;
}

DeviceCtx& pick_device_ctx()
{
    std::lock_guard<std::mutex> lk(g_mtx);
    if (g_devices.empty())
        for (int d : device_list()) { g_devices.emplace_back(new DeviceCtx()); g_devices.back()->device = d; }
    return *g_devices[g_next.fetch_add(1) % g_devices.size()];
}

void throw_for(int rc, const std::string& msg)
{
    if (rc == B200MVS_ERR_INVALID_ARG || rc == B200MVS_ERR_UNSUPPORTED) throw std::invalid_argument(msg);
    throw std::runtime_error(msg);     // B200MVS_ERR_GLOBAL_VS ("Global View Selection failed"), CUDA errors, overflow
}

// Requests whose settings differ at most in the scale run in one b200mvs_reconstruct_levels call, each at its own scale
// (--max-pixels gives views of different sizes different scales, apps/dmrecon/dmrecon.cc:89-111,299-302)
bool same_settings_but_scale(b200mvs_settings a, b200mvs_settings b)
{
    a.scale = b.scale = 0;
    return std::memcmp(&a, &b, sizeof(a)) == 0;
}

// Image source of a device context: the library loads the colour images a batch needs (loadColorImage, dmrecon.cc:78,
// 238-240) and evicts pyramids to stay within the device budget (ImagePyramidCache::cleanup, image_pyramid.cc:134-155).
// Called with the library's context lock held, by whichever thread runs the library call.
int fetch_image(void* user, int32_t id, b200mvs_image* out)
{
    DeviceCtx& D = *static_cast<DeviceCtx*>(user);
    try {
        mve::View::Ptr v = D.scene->get_views()[id];
        mve::ByteImage::Ptr img = v->get_byte_image(D.embedding);
        if (img == nullptr) return 1;
        D.held[id] = img;
        out->rgb = img->get_data_pointer();
        out->w = img->width(); out->h = img->height(); out->channels = img->channels();
        return 0;
    } catch (std::exception&) {
        return 1;
    }
}

void release_image(void* user, int32_t id)
{
    DeviceCtx& D = *static_cast<DeviceCtx*>(user);
    D.held.erase(id);
    D.scene->get_views()[id]->cache_cleanup();
}

// B200MVS_UNDISTORT=1: the images read (-i, default `undistorted`) are distorted photos, undistorted on the device with each
// view's camera.radial_distortion (b200mvs_set_view_distortion); unset or 0, they are used as they are.
bool undistort_images()
{
    const char* e = std::getenv("B200MVS_UNDISTORT");
    return e != nullptr && std::strcmp(e, "0") != 0 && *e != '\0';
}

// B200MVS_RECON_MASK=<embedding>: each reference view's one-channel image of that embedding is its reconstruction mask
// (b200mvs_set_view_mask, 0 = background); unset or empty, views are reconstructed whole.
const char* recon_mask_embedding()
{
    const char* e = std::getenv("B200MVS_RECON_MASK");
    return e != nullptr && *e != '\0' ? e : nullptr;
}

// Reads view `id`'s mask embedding into the context.  A view without it, or with more than one channel, is reconstructed
// unmasked, with the message scene2pset prints when it skips such a view (apps/scene2pset/scene2pset.cc:419-430).
void set_recon_mask(b200mvs_ctx* ctx, mve::View::Ptr view, int id, const char* embedding)
{
    mve::ByteImage::Ptr mask = view->get_byte_image(embedding);
    const char* problem = mask == nullptr ? "Mask not found for image \"" : mask->channels() != 1 ? "Expected 1-channel mask for image \"" : nullptr;
    if (problem) {
        std::lock_guard<std::mutex> lk(g_cout);
        std::cout << problem << view->get_name() << "\", skipping." << std::endl;
        return;
    }
    const int rc = b200mvs_set_view_mask(ctx, id, mask->get_data_pointer(), mask->width(), mask->height());
    if (rc != 0) throw_for(rc, b200mvs_last_error(ctx));
}

// B200MVS_PRIOR=<embedding>,<stride>: each reference view's one-channel float image of that embedding is its prior depth
// map (b200mvs_set_view_prior), seeded every <stride> pixels; unset or empty, views grow from the features alone.  For
// example B200MVS_PRIOR=depth-L2,4 with -s1 grows each level-1 map from the level-2 map of an earlier -s2 run as well.
// B200MVS_PRIOR_DZ=<embedding>, read only with B200MVS_PRIOR: the view's two-channel float image of that embedding is the
// prior's dz (b200mvs_set_view_prior_state), e.g. dz-L2 of an -s2 --keep-dz run, so each prior seed starts from the
// coarser map's slope as well.  dmrecon saves no view ids, so a prior from its files carries depth and dz only.
// B200MVS_PRIOR_MONO=<embedding>,<stride>,<kind>, not with B200MVS_PRIOR: the one-channel float image of that embedding
// is a map known up to a transform, such as a monocular network's output, of kind disparity, depth or depth_scale
// (b200mvs_set_view_prior_relative).  The view's features fix the transform, and one line per view reports it.
struct PriorSpec { std::string embedding, dz_embedding; int stride = 0; int kind = -1; };
bool prior_mono_spec(PriorSpec& out)
{
    const char* e = std::getenv("B200MVS_PRIOR_MONO");
    if (e == nullptr || *e == '\0') return false;
    const std::string v(e);
    const char* p = std::getenv("B200MVS_PRIOR");
    if (p != nullptr && *p != '\0') throw std::invalid_argument("B200MVS_PRIOR_MONO and B200MVS_PRIOR cannot both be set");
    const size_t c1 = v.find(','), c2 = c1 == std::string::npos ? c1 : v.find(',', c1 + 1);
    const std::string kind = c2 == std::string::npos ? "" : v.substr(c2 + 1);
    char* end = nullptr;
    const long stride = c2 == std::string::npos ? 0 : std::strtol(v.c_str() + c1 + 1, &end, 10);
    out.kind = kind == "disparity" ? B200MVS_PRIOR_DISPARITY : kind == "depth" ? B200MVS_PRIOR_DEPTH :
               kind == "depth_scale" ? B200MVS_PRIOR_DEPTH_SCALE : -1;
    if (c2 == std::string::npos || c1 == 0 || end == v.c_str() + c1 + 1 || end != v.c_str() + c2 || stride < 1 ||
        stride > 65535 || out.kind < 0)
        throw std::invalid_argument("B200MVS_PRIOR_MONO: expected <embedding>,<stride>,<kind> with a stride in 1..65535 "
                                    "and a kind of disparity, depth or depth_scale, not: " + v);
    out.embedding = v.substr(0, c1);
    out.stride = (int)stride;
    return true;
}

bool prior_spec(PriorSpec& out)
{
    if (prior_mono_spec(out)) return true;
    const char* e = std::getenv("B200MVS_PRIOR");
    if (e == nullptr || *e == '\0') return false;
    const std::string v(e);
    const size_t comma = v.rfind(',');
    char* end = nullptr;
    const long stride = comma == std::string::npos ? 0 : std::strtol(v.c_str() + comma + 1, &end, 10);
    if (comma == std::string::npos || comma == 0 || end == v.c_str() + comma + 1 || *end != '\0' || stride < 1 || stride > 65535)
        throw std::invalid_argument("B200MVS_PRIOR: expected <embedding>,<stride> with a stride in 1..65535, not: " + v);
    out.embedding = v.substr(0, comma);
    out.stride = (int)stride;
    const char* dz = std::getenv("B200MVS_PRIOR_DZ");
    out.dz_embedding = dz == nullptr ? "" : dz;
    return true;
}

// Reads view `id`'s prior embedding into the context.  A view without it, or with one that is not a one-channel float
// image, is reconstructed from its features alone.  A dz embedding that is missing, not a two-channel float image or of
// another size than the depth leaves the view a depth-only prior.
void set_prior(b200mvs_ctx* ctx, mve::View::Ptr view, int id, const PriorSpec& p)
{
    mve::ImageBase::Ptr img = view->get_image(p.embedding);
    const char* problem = img == nullptr ? "Prior not found for image \"" :
        img->get_type() != mve::IMAGE_TYPE_FLOAT || img->channels() != 1 ? "Expected 1-channel float prior for image \"" : nullptr;
    if (problem) {
        std::lock_guard<std::mutex> lk(g_cout);
        std::cout << problem << view->get_name() << "\", skipping." << std::endl;
        return;
    }
    const mve::FloatImage::Ptr depth = std::dynamic_pointer_cast<mve::FloatImage>(img);
    if (p.kind >= 0) {
        b200mvs_prior_fit fit;
        const int rc = b200mvs_set_view_prior_relative(ctx, id, depth->get_data_pointer(), depth->width(), depth->height(),
                                                       p.stride, p.kind, &fit);
        if (rc != 0 && rc != B200MVS_ERR_INVALID_ARG) throw_for(rc, b200mvs_last_error(ctx));
        char line[256];
        if (rc == 0)
            std::snprintf(line, sizeof(line), "Prior fit for image \"%s\": s %.6g t %.6g, %u of %u inliers",
                          view->get_name().c_str(), fit.scale, fit.shift, fit.n_inliers, fit.n_obs);
        else   // a fit that fails leaves the view without a prior
            std::snprintf(line, sizeof(line), "Prior fit failed for image \"%s\" (%s), skipping.", view->get_name().c_str(),
                          b200mvs_last_error(ctx));
        std::lock_guard<std::mutex> lk(g_cout);
        std::cout << line << std::endl;
        return;
    }
    const float* dz = nullptr;
    mve::ImageBase::Ptr dz_img;
    if (!p.dz_embedding.empty()) {
        dz_img = view->get_image(p.dz_embedding);
        problem = dz_img == nullptr ? "Prior dz not found for image \"" :
            dz_img->get_type() != mve::IMAGE_TYPE_FLOAT || dz_img->channels() != 2 ? "Expected 2-channel float prior dz for image \"" :
            dz_img->width() != depth->width() || dz_img->height() != depth->height() ? "Prior dz differs in size from the depth for image \"" :
            nullptr;
        if (problem) {
            std::lock_guard<std::mutex> lk(g_cout);
            std::cout << problem << view->get_name() << "\", using the depth alone." << std::endl;
        } else {
            dz = std::dynamic_pointer_cast<mve::FloatImage>(dz_img)->get_data_pointer();
        }
    }
    const int rc = b200mvs_set_view_prior_state(ctx, id, depth->get_data_pointer(), dz, nullptr, depth->width(),
                                                depth->height(), p.stride);
    if (rc != 0) throw_for(rc, b200mvs_last_error(ctx));
}

// Device budget of a context: B200MVS_DEVICE_BUDGET_MB, or 0 = 90 % of the free device memory (include/b200mvs.h).
uint64_t device_budget()
{
    const char* e = std::getenv("B200MVS_DEVICE_BUDGET_MB");
    return e ? (uint64_t)std::strtoull(e, nullptr, 10) << 20 : 0;
}

// Initial frontier capacity of a context: B200MVS_FRONTIER_CAPACITY=<entries_per_px>[,<min_entries>] (include/b200mvs.h),
// min_entries 65536 when omitted; unset = the library's default.
void set_frontier_capacity(b200mvs_ctx* ctx)
{
    const char* e = std::getenv("B200MVS_FRONTIER_CAPACITY");
    if (!e) return;
    char* end = nullptr;
    const double per_px = std::strtod(e, &end);
    uint64_t min_entries = 65536;
    if (end == e) throw std::invalid_argument(std::string("B200MVS_FRONTIER_CAPACITY: not a number: ") + e);
    if (*end == ',') min_entries = (uint64_t)std::strtoull(end + 1, nullptr, 10);
    if (b200mvs_set_frontier_capacity(ctx, per_px, min_entries) != 0) throw std::invalid_argument(b200mvs_last_error(ctx));
}

// Global view selection of one request (dmrecon.cc:211-241), done by the batch leader.  The colour images are loaded by
// the library through the image source when the batch runs.
void prepare_request(DeviceCtx& D, Request& r)
{
    r.progress->status = mvs::RECON_GLOBALVS;
    int32_t ids[B200MVS_MAX_GLOBAL_VIEWS];
    const int n = b200mvs_global_view_selection(D.ctx, &r.settings, r.ref, ids, B200MVS_MAX_GLOBAL_VIEWS);
    if (n < 0) { r.rc = n; r.err = b200mvs_last_error(D.ctx); return; }
    if (n == 0) { r.rc = B200MVS_ERR_GLOBAL_VS; r.err = "Global View Selection failed"; return; }
    r.gvs.assign(ids, ids + n);
    if (!r.quiet) {
        std::lock_guard<std::mutex> lk(g_cout);
        std::cout << "Global View Selection:";
        for (int i = 0; i < n; ++i) std::cout << " " << ids[i];
        std::cout << std::endl << "Loading color images..." << std::endl;
    }
    r.progress->status = mvs::RECON_FEATURES;
}

// Runs one batch on the device context (called by the leader WITHOUT holding D.mtx).
void run_batch(DeviceCtx& D, std::vector<Request*> batch)
{
    for (Request* r : batch) prepare_request(D, *r);
    // requests that failed in preparation or were cancelled meanwhile leave the batch with their own result
    std::vector<Request*> live;
    for (Request* r : batch) {
        if (r->rc != 0) continue;
        if (r->progress->cancelled) { r->rc = B200MVS_ERR_CANCELLED; continue; }
        live.push_back(r);
    }
    while (!live.empty()) {
        const size_t n = live.size();
        std::vector<int32_t> refs(n), levels(n);
        std::vector<b200mvs_maps> maps(n);
        std::vector<b200mvs_progress> prog(n);
        std::memset(prog.data(), 0, sizeof(b200mvs_progress) * n);
        for (size_t i = 0; i < n; ++i) {
            refs[i] = live[i]->ref; levels[i] = live[i]->settings.scale; maps[i] = live[i]->maps;
            live[i]->progress->status = mvs::RECON_QUEUE;
        }
        // relay: live progress out, cancel requests in (Progress is read/written without locks in the reference too,
        // fancy_progress_printer.cc:84-91, apps/umve/viewinspect/imageoperations.cc:177-184)
        std::atomic<bool> stop(false);
        std::thread relay([&]() {
            while (!stop.load()) {
                for (size_t i = 0; i < n; ++i) {
                    live[i]->progress->filled = prog[i].filled;
                    live[i]->progress->queueSize = prog[i].queue_size;
                    if (live[i]->progress->cancelled) prog[i].cancelled = 1;
                }
                std::this_thread::sleep_for(std::chrono::milliseconds(2));
            }
        });
        b200mvs_stats stats;
        int32_t failed = -1;
        const int rc = b200mvs_reconstruct_levels(D.ctx, &live[0]->settings, (int)n, refs.data(), levels.data(), maps.data(),
                                                  prog.data(), &stats, &failed);
        stop = true;
        relay.join();
        if (rc == 0 || rc == B200MVS_ERR_CANCELLED) {
            for (size_t i = 0; i < n; ++i) {
                // a cancelled view ends as RECON_CANCELLED; the other views of the batch keep their results
                const bool cancelled = rc == B200MVS_ERR_CANCELLED || prog[i].status == 5;
                live[i]->rc = cancelled ? B200MVS_ERR_CANCELLED : 0;
                live[i]->progress->filled = prog[i].filled;
                live[i]->maps = maps[i]; live[i]->stats = stats;
                live[i]->err = cancelled ? "reconstruction cancelled" : "";
            }
            return;
        }
        // one view made the call fail: give it its error, retry the others
        const std::string msg = b200mvs_last_error(D.ctx);
        bool removed = false;
        for (size_t i = 0; i < live.size(); ++i) {
            if (failed >= 0 && live[i]->ref != failed) continue;
            live[i]->rc = rc; live[i]->err = msg;
            if (failed >= 0) { live.erase(live.begin() + i); removed = true; break; }
        }
        if (failed < 0 || !removed) return;      // error not attributable to one view: every request got it
    }
}

} // namespace

MVS_NAMESPACE_BEGIN

DMRecon::DMRecon(mve::Scene::Ptr _scene, Settings const& _settings)
    : scene(_scene)
    , settings(_settings)
{
    mve::Scene::ViewList const& mve_views(scene->get_views());
    if (settings.refViewNr >= mve_views.size())
        throw std::invalid_argument("Master view index out of bounds");
    if (settings.scale < 0.f)
        throw std::invalid_argument("Invalid scale factor");
    if (settings.imageEmbedding.empty())
        throw std::invalid_argument("Invalid image embedding");
    try {
        this->bundle = this->scene->get_bundle();
    } catch (std::exception& e) {
        throw std::runtime_error(std::string("Error reading bundle file: ") + e.what());
    }
    mve::View::Ptr refV = mve_views[settings.refViewNr];
    if (refV == nullptr || !refV->is_camera_valid()
        || !refV->has_image(settings.imageEmbedding, mve::IMAGE_TYPE_UINT8))
        throw std::invalid_argument("Invalid master view");
    // size of pyramid level `scale` ((w+1)/2 per level, image_pyramid.cc:46-47)
    mve::View::ImageProxy const* proxy = refV->get_image_proxy(settings.imageEmbedding);
    int w = proxy->width, h = proxy->height;
    for (int l = 0; l < settings.scale; ++l) { w = (w + 1) / 2; h = (h + 1) / 2; }
    this->width = w;
    this->height = h;
    if (!settings.quiet)
        std::cout << "scaled image size: " << this->width << " x " << this->height << std::endl;
}

void
DMRecon::start()
{
    progress.start_time = std::time(nullptr);
    mve::Scene::ViewList const& mve_views(scene->get_views());
    DeviceCtx& D = pick_device_ctx();
    std::unique_lock<std::mutex> lock(D.mtx);

    /* (Re)create the device context for this scene; cameras and features are registered once per context. */
    if (D.ctx == nullptr || D.scene != scene || D.embedding != settings.imageEmbedding) {
        while (D.leader_active || D.planners > 0) D.cv.wait(lock);
        if (D.ctx) { b200mvs_destroy(D.ctx); D.ctx = nullptr; }
        int rc = b200mvs_create(D.device, (int)mve_views.size(), &D.ctx);
        if (rc != 0) throw std::runtime_error(b200mvs_last_error(nullptr));
        D.scene = scene;
        D.embedding = settings.imageEmbedding;
        D.held.clear();
        D.masks_set.assign(mve_views.size(), 0);
        D.priors_set.assign(mve_views.size(), 0);
        rc = b200mvs_set_image_source(D.ctx, fetch_image, release_image, &D, device_budget());
        if (rc != 0) throw std::runtime_error(b200mvs_last_error(D.ctx));
        set_frontier_capacity(D.ctx);
        D.features_set = false;
        D.cameras_set = false;
    }
    b200mvs_ctx* ctx = D.ctx;

    /* Views: the same validity test as dmrecon.cc:62-71.  Every valid view gets its camera registered
       (SingleView::create); colour images are loaded by the library through the context's image source, only for the
       master views and their selected neighbours (loadColorImage, dmrecon.cc:78,238-240), and evicted when the device
       budget needs the room. */
    progress.status = RECON_FEATURES;
    if (!D.cameras_set) {
        while (D.leader_active || D.planners > 0) D.cv.wait(lock);
        for (std::size_t i = 0; i < mve_views.size(); ++i) {
            mve::View::Ptr v = mve_views[i];
            if (v == nullptr || !v->is_camera_valid() || !v->has_image(settings.imageEmbedding, mve::IMAGE_TYPE_UINT8))
                continue;
            mve::View::ImageProxy const* proxy = v->get_image_proxy(settings.imageEmbedding);
            mve::CameraInfo const& cam = v->get_camera();
            int rc = b200mvs_set_view_camera(ctx, (int)i, proxy->width, proxy->height, cam.flen, cam.paspect, cam.ppoint,
                cam.rot, cam.trans);
            /* B200MVS_UNDISTORT=1: the embedding holds the distorted photo; undistort it with the view's
               camera.radial_distortion as sfmrecon does (sfmrecon.cc:425-437) */
            if (rc == 0 && undistort_images())
                rc = b200mvs_set_view_distortion(ctx, (int)i, cam.dist[0], cam.dist[1]);
            if (rc != 0) throw_for(rc, b200mvs_last_error(ctx));
        }
        D.cameras_set = true;
    }
    if (!D.features_set) {
        mve::Bundle::Features const& features = bundle->get_features();
        std::vector<float> pos(features.size() * 3);
        std::vector<int32_t> off(features.size() + 1, 0), ids;
        for (std::size_t i = 0; i < features.size(); ++i) {
            std::memcpy(&pos[3 * i], features[i].pos, 3 * sizeof(float));
            for (std::size_t j = 0; j < features[i].refs.size(); ++j) ids.push_back(features[i].refs[j].view_id);
            off[i + 1] = (int32_t)ids.size();
        }
        while (D.leader_active || D.planners > 0) D.cv.wait(lock);
        int rc = b200mvs_set_features(ctx, (int)features.size(), pos.data(), off.data(), ids.data());
        if (rc != 0) throw_for(rc, b200mvs_last_error(ctx));
        D.features_set = true;
    }
    if (progress.cancelled) { progress.status = RECON_CANCELLED; return; }

    /* Settings: POD part of mvs::Settings, field for field. */
    b200mvs_settings s;
    b200mvs_default_settings(&s);
    s.filter_width = settings.filterWidth;
    s.min_ncc = settings.minNCC;
    s.min_parallax = settings.minParallax;
    s.accept_ncc = settings.acceptNCC;
    s.min_refine_diff = settings.minRefineDiff;
    s.max_iterations = settings.maxIterations;
    s.nr_recon_neighbors = settings.nrReconNeighbors;
    s.global_vs_max = settings.globalVSMax;
    s.scale = settings.scale;
    s.use_color_scale = settings.useColorScale ? 1 : 0;
    for (int i = 0; i < 3; ++i) { s.aabb_min[i] = settings.aabbMin[i]; s.aabb_max[i] = settings.aabbMax[i]; }
    if (const char* e = std::getenv("B200MVS_FRONTIER_TOPK")) s.frontier_topk = (uint32_t)std::atoi(e);   // engine knobs, include/b200mvs.h
    if (const char* e = std::getenv("B200MVS_FRONTIER_BAND")) s.frontier_band = (float)std::atof(e);

    /* Result images, allocated like SingleView::prepareMasterView (single_view.cc:78-81). */
    mve::FloatImage::Ptr depthImg = mve::FloatImage::create(width, height, 1);
    mve::FloatImage::Ptr dzImg = mve::FloatImage::create(width, height, 2);
    mve::FloatImage::Ptr confImg = mve::FloatImage::create(width, height, 1);
    Request req;
    req.ref = (int32_t)settings.refViewNr;
    req.settings = s;
    req.progress = &progress;
    req.embedding = settings.imageEmbedding;
    req.quiet = settings.quiet;
    std::memset(&req.maps, 0, sizeof(req.maps));
    req.maps.depth = depthImg->get_data_pointer();
    req.maps.dz = dzImg->get_data_pointer();
    req.maps.conf = confImg->get_data_pointer();
    std::memset(&req.stats, 0, sizeof(req.stats));

    /* Global view selection + seed list (dmrecon.cc:96-98,211-292) on the CALLER's thread, like the reference, where every
       DMRecon of the OpenMP team does its own: in parallel over the team and while the GPU still runs the previous batch.
       The result is parked in the context (b200mvs_plan_views); the leader's b200mvs_global_view_selection and
       b200mvs_reconstruct pick it up instead of computing it again. */
    progress.status = RECON_GLOBALVS;
    const char* mask_embedding = recon_mask_embedding();
    const bool read_mask = mask_embedding != nullptr && !D.masks_set[req.ref];
    if (read_mask) D.masks_set[req.ref] = 1;
    PriorSpec prior;
    const bool read_prior = prior_spec(prior) && !D.priors_set[req.ref];
    if (read_prior) D.priors_set[req.ref] = 1;
    D.planners++;
    lock.unlock();
    try {
        if (read_mask) set_recon_mask(ctx, mve_views[req.ref], req.ref, mask_embedding);
        if (read_prior) set_prior(ctx, mve_views[req.ref], req.ref, prior);
    } catch (...) {
        lock.lock();
        D.planners--;
        D.cv.notify_all();
        throw;
    }
    b200mvs_plan_views(ctx, &s, 1, &req.ref);        // a failure shows up again, with its message, in the leader's call
    lock.lock();
    D.planners--;
    if (progress.cancelled) { D.cv.notify_all(); progress.status = RECON_CANCELLED; return; }

    /* Submit.  Whoever finds no leader becomes one and runs batches until the queue is empty. */
    D.pending.push_back(&req);
    D.arrivals++;
    D.cv.notify_all();
    if (!D.leader_active) {
        D.leader_active = true;
        while (!D.pending.empty()) {
            /* Collection window: the other threads of the caller's OpenMP team reach this point within microseconds to
               milliseconds of each other (they all finished the previous batch together).  Callers that are computing
               their view selection right now (D.planners) are certain to arrive: wait for them (at most 250 ms).  Beyond
               that: until as many requests as the previous batch had are here, or nothing new has arrived for 3 ms, at
               most 30 ms. */
            const auto t_open = std::chrono::steady_clock::now();
            uint64_t seen = D.arrivals;
            for (;;) {
                if (D.planners == 0 && D.last_batch > 1 && D.pending.size() >= D.last_batch) break;
                const bool woke = D.cv.wait_for(lock, std::chrono::milliseconds(3), [&]() { return D.arrivals != seen; });
                if (!woke && D.planners == 0) break;
                seen = D.arrivals;
                if (std::chrono::steady_clock::now() - t_open > std::chrono::milliseconds(D.planners > 0 ? 250 : 30)) break;
            }
            // one batch: the requests that share the first one's settings up to the scale and its embedding, each
            // (view, scale) once
            std::vector<Request*> batch;
            std::vector<Request*> rest;
            for (Request* r : D.pending) {
                const bool joins = batch.empty() ||
                    (same_settings_but_scale(r->settings, batch[0]->settings) && r->embedding == batch[0]->embedding &&
                     std::none_of(batch.begin(), batch.end(), [&](const Request* q) { return q->ref == r->ref && q->settings.scale == r->settings.scale; }));
                (joins ? batch : rest).push_back(r);
            }
            D.pending.swap(rest);
            D.last_batch = batch.size();
            lock.unlock();
            run_batch(D, batch);
            lock.lock();
            for (Request* r : batch) r->done = true;
            D.cv.notify_all();
        }
        D.leader_active = false;
        D.cv.notify_all();
    }
    while (!req.done) D.cv.wait(lock);
    lock.unlock();

    const b200mvs_stats& stats = req.stats;
    const int rc0 = req.rc;
    progress.queueSize = 0;
    if (rc0 == B200MVS_ERR_CANCELLED || progress.cancelled) { progress.status = RECON_CANCELLED; return; }
    if (rc0 != 0) throw_for(rc0, req.err);
    if (!settings.quiet) {
        std::ostringstream line;       // one write: the OpenMP threads of the driver print concurrently
        line << "Reconstructed view " << settings.refViewNr << " (batch of all views in flight: " << stats.n_seeds_processed
             << " features processed, " << stats.n_seeds_success << " succeeded optimization, " << stats.n_rounds
             << " frontier rounds)." << std::endl;
        std::lock_guard<std::mutex> lk(g_cout);
        std::cout << line.str() << std::flush;
    }

    progress.status = RECON_SAVING;
    mve::View::Ptr view = mve_views[settings.refViewNr];
    mve::ByteImage::Ptr scaled;
    if (settings.scale != 0 || settings.writePlyFile) {
        // level `scale` of the reference view as the device built it (bit-exact with the reference's pyramid)
        scaled = mve::ByteImage::create(width, height, 3);
        int w = 0, h = 0;
        int rc = b200mvs_get_level(ctx, (int)settings.refViewNr, settings.scale, &w, &h, scaled->get_data_pointer());
        if (rc != 0) throw_for(rc, b200mvs_last_error(ctx));
    }
    if (settings.writePlyFile) {
        // SingleView::saveReconAsPly (single_view.cc:123-138) through the same libmve writers
        if (settings.plyPath.empty()) throw std::invalid_argument("Empty path");
        std::string fname = "mvs-" + util::string::get_filled(settings.refViewNr, 4) + "-L" + util::string::get((float)settings.scale);
        if (!settings.quiet)
            std::cout << "Saving ply file as " << settings.plyPath << "/" << fname << ".ply" << std::endl;
        if (!util::fs::dir_exists(settings.plyPath.c_str())) util::fs::mkdir(settings.plyPath.c_str());
        mve::geom::save_ply_view(util::fs::join_path(settings.plyPath, fname + ".ply"), view->get_camera(), depthImg, confImg, scaled);
        mve::geom::save_xf_file(util::fs::join_path(settings.plyPath, fname + ".xf"), view->get_camera());
    }
    std::string name("depth-L");
    name += util::string::get(settings.scale);
    view->set_image(depthImg, name);
    if (settings.keepDzMap) {
        name = "dz-L";
        name += util::string::get(settings.scale);
        view->set_image(dzImg, name);
    }
    if (settings.keepConfidenceMap) {
        name = "conf-L";
        name += util::string::get(settings.scale);
        view->set_image(confImg, name);
    }
    if (settings.scale != 0) {
        name = "undist-L";
        name += util::string::get(settings.scale);
        view->set_image(scaled, name);
    }
    progress.status = RECON_IDLE;
    {
        int nrPix = this->width * this->height;
        float percent = (float) progress.filled / (float) nrPix;
        if (!settings.quiet)
            std::cout << "Filled " << progress.filled << " pixels, i.e. "
                      << util::string::get_fixed(percent * 100.f, 1) << " %." << std::endl;
    }
    size_t mvs_time = std::time(nullptr) - progress.start_time;
    if (!settings.quiet)
        std::cout << "MVS took " << mvs_time << " seconds." << std::endl;
}

MVS_NAMESPACE_END
