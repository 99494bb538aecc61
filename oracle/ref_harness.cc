/* TEST INFRASTRUCTURE - NOT PRODUCT CODE.
 *
 * Our own driver around the UNMODIFIED reference classes (linked from oracle/_ref/libmve_dmrecon.a,
 * libmve.a, libmve_util.a, built by oracle/Makefile from /root/reference).  It never re-implements the
 * algorithm; it only calls the reference's public interface:
 *
 *   ref_harness patches SCENE REF SCALE NRN IN.bin OUT.bin
 *       Mints per-patch golden vectors: builds the SingleViews like DMRecon's ctor (dmrecon.cc:62-79),
 *       runs analyzeFeatures' loop (dmrecon.cc:179-208) + mvs::GlobalViewSelection, then one
 *       mvs::PatchOptimization (ctor + doAutoOptimization + computeConfidence, exactly the three calls of
 *       dmrecon.cc:293-296 / :374-377) per record of IN.bin and writes the results to OUT.bin.
 *       Record layouts = mvs_oracle_patch_in / mvs_oracle_patch_out of oracle/mvs_oracle.h.
 *
 *   ref_harness timed SCENE SCALE NRN SECONDS STEPS VIEW [VIEW...]
 *       CPU baseline: STEPS times, runs mvs::DMRecon(scene, settings).start() for the listed views, one thread per view
 *       (the reference's own parallelism, apps/dmrecon/dmrecon.cc:285); the clock starts when every view has reached
 *       processQueue (Progress::status == RECON_QUEUE), Progress::cancelled is set SECONDS later (the reference's
 *       cooperative cancel, dmrecon.cc:353); prints one JSON line per step with the pixels filled inside the clocked
 *       interval and its length.  SECONDS <= 0 runs to completion.
 */
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "dmrecon/dmrecon.h"
#include "dmrecon/global_view_selection.h"
#include "dmrecon/patch_optimization.h"
#include "dmrecon/settings.h"
#include "dmrecon/single_view.h"
#include "math/octree_tools.h"
#include "mve/depthmap.h"
#include "mve/mesh.h"
#include "mve/mesh_info.h"
#include "mve/scene.h"

#include "mvs_oracle.h"

static int run_patches(int argc, char** argv)
{
    if (argc != 8) { std::fprintf(stderr, "usage: ref_harness patches SCENE REF SCALE NRN IN OUT\n"); return 2; }
    mve::Scene::Ptr scene = mve::Scene::create(argv[2]);
    mvs::Settings settings;
    settings.refViewNr = std::atoi(argv[3]);
    settings.scale = std::atoi(argv[4]);
    settings.nrReconNeighbors = std::atoi(argv[5]);
    settings.quiet = true;
    mve::Bundle::ConstPtr bundle = scene->get_bundle();
    mve::Scene::ViewList const& mve_views(scene->get_views());
    std::vector<mvs::SingleView::Ptr> views(mve_views.size());
    for (std::size_t i = 0; i < mve_views.size(); ++i) {
        if (mve_views[i] == nullptr || !mve_views[i]->is_camera_valid()
            || !mve_views[i]->has_image(settings.imageEmbedding, mve::IMAGE_TYPE_UINT8))
            continue;
        views[i] = mvs::SingleView::create(scene, mve_views[i], settings.imageEmbedding);
    }
    mvs::SingleView::Ptr refV = views[settings.refViewNr];
    refV->loadColorImage(settings.scale);
    refV->prepareMasterView(settings.scale);
    mve::Bundle::Features const& features = bundle->get_features();
    for (std::size_t i = 0; i < features.size(); ++i) {
        if (!features[i].contains_view_id(settings.refViewNr)) continue;
        math::Vec3f featurePos(features[i].pos);
        if (!refV->pointInFrustum(featurePos)) continue;
        if (!math::geom::point_box_overlap(featurePos, settings.aabbMin, settings.aabbMax)) continue;
        for (std::size_t j = 0; j < features[i].refs.size(); ++j) {
            int view_id = features[i].refs[j].view_id;
            if (view_id < 0 || view_id >= static_cast<int>(views.size()) || views[view_id] == nullptr) continue;
            if (views[view_id]->pointInFrustum(featurePos)) views[view_id]->addFeature(i);
        }
    }
    mvs::GlobalViewSelection globalVS(views, features, settings);
    globalVS.performVS();
    mvs::IndexSet neighViews = globalVS.getSelectedIDs();
    std::printf("Global View Selection:");
    for (std::size_t id : neighViews) std::printf(" %zu", id);
    std::printf("\n");
    for (std::size_t id : neighViews) views[id]->loadColorImage(0);

    std::ifstream in(argv[6], std::ios::binary);
    std::vector<char> buf((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    const std::size_t n = buf.size() / sizeof(mvs_oracle_patch_in);
    const mvs_oracle_patch_in* pin = reinterpret_cast<const mvs_oracle_patch_in*>(buf.data());
    std::vector<mvs_oracle_patch_out> pout(n);
    for (std::size_t i = 0; i < n; ++i) {
        mvs::IndexSet local;
        for (int k = 0; k < pin[i].n_local; ++k) local.insert(pin[i].local_ids[k]);
        mvs_oracle_patch_out& o = pout[i];
        std::memset(&o, 0, sizeof(o));
        for (int k = 0; k < 4; ++k) o.local_ids[k] = -1;
        mvs::PatchOptimization patch(views, settings, pin[i].x, pin[i].y, pin[i].depth, pin[i].dz_i, pin[i].dz_j,
            neighViews, local);
        patch.doAutoOptimization();
        o.conf = patch.computeConfidence();
        o.depth = patch.getDepth();
        o.dz_i = patch.getDzI();
        o.dz_j = patch.getDzJ();
        if (o.conf > 0.f) {
            math::Vec3f nrm = patch.getNormal();
            o.normal[0] = nrm[0]; o.normal[1] = nrm[1]; o.normal[2] = nrm[2];
        }
        int k = 0;
        for (std::size_t id : patch.getLocalViewIDs()) { if (k < 4) o.local_ids[k] = (int)id; ++k; }
        o.n_local = k;
        o.iterations = -1;           /* Status is private in the reference */
        o.converged = o.conf != 0.f; /* computeConfidence returns 0 unless converged (patch_optimization.cc:117) */
        o.opti_success = -1;
    }
    std::ofstream out(argv[7], std::ios::binary);
    out.write(reinterpret_cast<const char*>(pout.data()), (std::streamsize)(n * sizeof(mvs_oracle_patch_out)));
    return 0;
}

static int run_timed(int argc, char** argv)
{
    if (argc < 8) { std::fprintf(stderr, "usage: ref_harness timed SCENE SCALE NRN SECONDS STEPS VIEW...\n"); return 2; }
    mve::Scene::Ptr scene = mve::Scene::create(argv[2]);
    const int scale = std::atoi(argv[3]);
    const int nrn = std::atoi(argv[4]);
    const double seconds = std::atof(argv[5]);
    const int steps = std::max(1, std::atoi(argv[6]));
    std::vector<int> ids;
    for (int i = 7; i < argc; ++i) ids.push_back(std::atoi(argv[i]));
    scene->get_bundle();
    /* touch the input images first so that no step measures file I/O */
    for (int id : ids) scene->get_views()[id]->get_byte_image("undistorted");
    for (int step = 0; step < steps; ++step) {
        std::vector<mvs::DMRecon*> recons(ids.size(), nullptr);
        std::vector<std::size_t> filled(ids.size(), 0);
        std::vector<int> state(ids.size(), 0);       /* 0 setting up, 1 running, 2 finished, 3 failed */
        std::vector<int> done(ids.size(), 0);
        std::atomic<int> running((int)ids.size());
        std::mutex mtx;
        std::vector<std::thread> th;
        for (std::size_t k = 0; k < ids.size(); ++k) {
            th.emplace_back([&, k]() {
                try {
                    mvs::Settings settings;
                    settings.refViewNr = ids[k];
                    settings.scale = scale;
                    settings.nrReconNeighbors = nrn;
                    settings.quiet = true;
                    settings.keepDzMap = true;
                    settings.keepConfidenceMap = true;
                    mvs::DMRecon recon(scene, settings);
                    { std::lock_guard<std::mutex> lk(mtx); recons[k] = &recon; state[k] = 1; }
                    recon.start();
                    std::lock_guard<std::mutex> lk(mtx);
                    filled[k] = recon.getProgress().filled;
                    done[k] = recon.getProgress().cancelled ? 0 : 1;
                    recons[k] = nullptr;
                    state[k] = 2;
                } catch (std::exception& e) {
                    std::fprintf(stderr, "view %d failed: %s\n", ids[k], e.what());
                    std::lock_guard<std::mutex> lk(mtx);
                    recons[k] = nullptr;
                    state[k] = 3;
                }
                running--;
            });
        }
        /* The clock starts when EVERY view has reached processQueue (RECON_QUEUE): SingleView creation, image pyramids
         * (serialised by the reference's global ImagePyramidCache mutex, image_pyramid.cc:102,137), global view selection
         * and the seed features are set-up, not the region growing this metric is about. */
        auto sum_filled = [&]() {
            std::size_t t = 0;
            for (std::size_t k = 0; k < ids.size(); ++k) t += recons[k] ? recons[k]->getProgress().filled : filled[k];
            return t;
        };
        std::size_t filled0 = 0;
        auto t_setup = std::chrono::steady_clock::now();
        for (;;) {
            std::this_thread::sleep_for(std::chrono::milliseconds(5));
            std::lock_guard<std::mutex> lk(mtx);
            bool all = true;
            for (std::size_t k = 0; k < ids.size(); ++k) {
                if (state[k] == 0) all = false;
                else if (state[k] == 1 && recons[k] && recons[k]->getProgress().status < mvs::RECON_QUEUE) all = false;
            }
            if (all) { filled0 = sum_filled(); break; }
        }
        auto t0 = std::chrono::steady_clock::now();
        const double setup_s = std::chrono::duration<double>(t0 - t_setup).count();
        std::size_t filled1 = 0;
        for (;;) {
            std::this_thread::sleep_for(std::chrono::milliseconds(5));
            const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            if ((seconds > 0 && el >= seconds) || running.load() == 0) {
                std::lock_guard<std::mutex> lk(mtx);
                filled1 = sum_filled();
                for (std::size_t k = 0; k < ids.size(); ++k) if (recons[k]) recons[k]->getProgress().cancelled = true;
                break;
            }
        }
        const double el = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        for (auto& t : th) t.join();
        int complete = 0;
        for (std::size_t k = 0; k < ids.size(); ++k) complete += done[k];
        std::printf("{\"filled\": %zu, \"seconds\": %.6f, \"views\": %zu, \"views_completed\": %d, \"threads\": %zu, "
                    "\"filled_before_clock\": %zu, \"setup_seconds\": %.3f}\n",
                    filled1 - filled0, el, ids.size(), complete, ids.size(), filled0, setup_s);
        std::fflush(stdout);
    }
    return 0;
}

/* Depth-map consumers of the reference (libs/mve/depthmap.cc) on raw little-endian buffers:
 *   ref_harness dmops cleanup W H THRES in.f32 out.f32
 *   ref_harness dmops confclean W H in.f32 conf.f32 out.f32
 *   ref_harness dmops triangulate W H DD in.f32 COLOR.u8|- CCH  i0 .. i8  OUTPREFIX [CONF_ITER [SCALE_FACTOR]]
 *       -> OUTPREFIX.vids (uint32 W*H), .verts (float32 V*3, camera coordinates), .faces (uint32 F*3), .colors (float32 V*4),
 *          .normals (V*3), .confs (V, depthmap_mesh_confidences(mesh, CONF_ITER), default 4; empty for 0),
 *          .scales (V, scene2pset's scale values x SCALE_FACTOR, default 2.5) */
static std::vector<char> read_all(const char* path)
{
    std::ifstream in(path, std::ios::binary);
    return std::vector<char>((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}
static void write_all(const std::string& path, const void* p, std::size_t n)
{
    std::ofstream out(path, std::ios::binary);
    out.write(reinterpret_cast<const char*>(p), (std::streamsize)n);
}
static int run_dmops(int argc, char** argv)
{
    if (argc < 6) return 2;
    const std::string op = argv[2];
    const int W = std::atoi(argv[3]), H = std::atoi(argv[4]);
    auto load_float = [&](const char* path) {
        mve::FloatImage::Ptr img = mve::FloatImage::create(W, H, 1);
        std::vector<char> raw = read_all(path);
        std::memcpy(img->get_data_pointer(), raw.data(), std::min(raw.size(), (std::size_t)W * H * 4));
        return img;
    };
    if (op == "cleanup" && argc >= 8) {
        mve::FloatImage::Ptr dm = load_float(argv[6]);
        mve::FloatImage::Ptr out = mve::image::depthmap_cleanup(dm, std::atoll(argv[5]));
        write_all(argv[7], out->get_data_pointer(), (std::size_t)W * H * 4);
        return 0;
    }
    if (op == "confclean" && argc >= 8) {
        mve::FloatImage::Ptr dm = load_float(argv[5]);
        mve::FloatImage::Ptr cm = load_float(argv[6]);
        mve::image::depthmap_confidence_clean(dm, cm);
        write_all(argv[7], dm->get_data_pointer(), (std::size_t)W * H * 4);
        return 0;
    }
    if (op == "triangulate" && argc >= 19) {
        const float dd = (float)std::atof(argv[5]);
        mve::FloatImage::Ptr dm = load_float(argv[6]);
        mve::ByteImage::Ptr ci;
        const int cch = std::atoi(argv[8]);
        if (std::string(argv[7]) != "-") {
            ci = mve::ByteImage::create(W, H, cch);
            std::vector<char> raw = read_all(argv[7]);
            std::memcpy(ci->get_data_pointer(), raw.data(), std::min(raw.size(), (std::size_t)W * H * cch));
        }
        math::Matrix3f invproj;
        for (int i = 0; i < 9; ++i) invproj[i] = (float)std::atof(argv[9 + i]);
        mve::Image<unsigned int> vids;
        /* the colour overload returns before handing out the vertex ids when there is no colour image (depthmap.cc:340-341) */
        mve::TriangleMesh::Ptr mesh = ci != nullptr ? mve::geom::depthmap_triangulate(dm, ci, invproj, dd, &vids)
                                                    : mve::geom::depthmap_triangulate(dm, invproj, dd, &vids);
        const std::string prefix = argv[18];
        const int conf_iter = argc > 19 ? std::atoi(argv[19]) : 4;
        const float scale_factor = argc > 20 ? (float)std::atof(argv[20]) : 2.5f;
        write_all(prefix + ".vids", vids.get_data_pointer(), (std::size_t)W * H * 4);
        write_all(prefix + ".verts", mesh->get_vertices().data(), mesh->get_vertices().size() * 12);
        write_all(prefix + ".faces", mesh->get_faces().data(), mesh->get_faces().size() * 4);
        write_all(prefix + ".colors", mesh->get_vertex_colors().data(), mesh->get_vertex_colors().size() * 16);
        /* the rest of the per-view work of apps/scene2pset (scene2pset.cc:316-358): normals, boundary confidences, scale */
        mesh->ensure_normals();
        write_all(prefix + ".normals", mesh->get_vertex_normals().data(), mesh->get_vertex_normals().size() * 12);
        mve::geom::depthmap_mesh_confidences(mesh, conf_iter);
        write_all(prefix + ".confs", mesh->get_vertex_confidences().data(), mesh->get_vertex_confidences().size() * 4);
        {
            mve::TriangleMesh::VertexList const& mverts(mesh->get_vertices());
            std::vector<float> mvscale(mverts.size(), 0.0f);
            mve::MeshInfo mesh_info(mesh);
            for (std::size_t j = 0; j < mesh_info.size(); ++j) {
                mve::MeshInfo::VertexInfo const& vinf = mesh_info[j];
                for (std::size_t k = 0; k < vinf.verts.size(); ++k)
                    mvscale[j] += (mverts[j] - mverts[vinf.verts[k]]).norm();
                mvscale[j] /= static_cast<float>(vinf.verts.size());
                mvscale[j] *= scale_factor;
            }
            write_all(prefix + ".scales", mvscale.data(), mvscale.size() * 4);
        }
        return 0;
    }
    return 2;
}

int main(int argc, char** argv)
{
    if (argc >= 3 && std::strcmp(argv[1], "dmops") == 0) return run_dmops(argc, argv);
    if (argc >= 2 && std::strcmp(argv[1], "patches") == 0) return run_patches(argc, argv);
    if (argc >= 2 && std::strcmp(argv[1], "timed") == 0) return run_timed(argc, argv);
    std::fprintf(stderr, "usage: ref_harness patches|timed ...\n");
    return 2;
}
