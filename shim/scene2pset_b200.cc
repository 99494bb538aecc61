// scene2pset_b200: a drop-in for MVE's scene2pset that builds the whole-scene point set on the GPU.
//
// Same command line and output files as apps/scene2pset: the scene is read and the mesh written through the reference's
// own libmve.a (mve::Scene / mve::View, save_ply_mesh with the same SavePLYOptions, save_mesh for other extensions), the
// correspondence CSVs in the same format.  Every view's triangulation, normals, confidences, scales, fill fraction,
// bounding box and the silhouette-mask clipping run in libb200mvs.so behind the b200mvs_pset_* C ABI (include/b200mvs.h).
// The points come in the scene's view order (the reference appends views in the order its OpenMP threads finish them,
// which is the view order on one thread).
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "mve/image.h"
#include "mve/mesh.h"
#include "mve/mesh_io.h"
#include "mve/mesh_io_ply.h"
#include "mve/scene.h"
#include "mve/view.h"
#include "util/arguments.h"
#include "util/string_utils.h"

#include "b200mvs.h"

namespace {

struct Options {
    std::string scene_dir, out;
    std::string depth = "depth-L0", image = "undistorted", mask, aabb;
    bool normals = false, scale = false, conf = false, poisson = false, correspondence = false;
    float min_fraction = 0.0f, scale_factor = 2.5f;
    std::vector<int> ids;
};

[[noreturn]] void die(std::string const& what)
{
    std::cerr << "Error: " << what << std::endl;
    std::exit(EXIT_FAILURE);
}

void check(int rc, char const* call)
{
    if (rc < 0) die(std::string(call) + ": " + b200mvs_depthmap_last_error());
}

bool ends_with(std::string const& s, std::string const& tail)
{
    return s.size() >= tail.size() && s.compare(s.size() - tail.size(), tail.size(), tail) == 0;
}

b200mvs_pset_camera camera_of(mve::CameraInfo const& c)
{
    b200mvs_pset_camera pc;
    pc.flen = c.flen;
    pc.paspect = c.paspect;
    std::memcpy(pc.ppoint, c.ppoint, sizeof(pc.ppoint));
    std::memcpy(pc.rot, c.rot, sizeof(pc.rot));
    std::memcpy(pc.trans, c.trans, sizeof(pc.trans));
    return pc;
}

Options parse(int argc, char** argv)
{
    util::Arguments args;
    args.set_exit_on_error(true);
    args.set_nonopt_minnum(2);
    args.set_nonopt_maxnum(2);
    args.set_helptext_indent(25);
    args.set_usage("Usage: scene2pset_b200 [ OPTS ] SCENE_DIR MESH_OUT");
    args.set_description("Turns the depth maps of an MVE scene into one point set in world coordinates, on the GPU. "
        "Accepts the options of MVE's scene2pset and writes the same files.");
    args.add_option('d', "depthmap", true, "Depth map embedding [depth-L0]");
    args.add_option('i', "image", true, "Colour image embedding [undistorted]");
    args.add_option('n', "with-normals", false, "Write a normal per point (PLY only)");
    args.add_option('s', "with-scale", false, "Write a scale value per point (PLY only)");
    args.add_option('c', "with-conf", false, "Write a confidence per point (PLY only)");
    args.add_option('m', "mask", true, "Silhouette mask embedding; points a mask marks 0 are removed []");
    args.add_option('v', "views", true, "IDs of the views to use [all]");
    args.add_option('b', "bounding-box", true, "Keep points inside this box: minx,miny,minz,maxx,maxy,maxz");
    args.add_option('f', "min-fraction", true, "Skip views with a smaller fraction of valid depths [0.0]");
    args.add_option('p', "poisson-normals", false, "Multiply each normal by its confidence");
    args.add_option('S', "scale-factor", true, "Multiplier of the scale values [2.5]");
    args.add_option('C', "correspondence", false, "Write point-to-pixel correspondences (without -m and -b only)");
    args.add_option('F', "fssr", true, "Output for FSSR at scale ARG: sets -n -s -c and the embeddings of that scale");
    args.parse(argc, argv);

    Options o;
    o.scene_dir = args.get_nth_nonopt(0);
    o.out = args.get_nth_nonopt(1);
    while (util::ArgResult const* a = args.next_result()) {
        if (a->opt == nullptr) continue;
        switch (a->opt->sopt) {
            case 'd': o.depth = a->arg; break;
            case 'i': o.image = a->arg; break;
            case 'n': o.normals = true; break;
            case 's': o.scale = true; break;
            case 'c': o.conf = true; break;
            case 'm': o.mask = a->arg; break;
            case 'v': args.get_ids_from_string(a->arg, &o.ids); break;
            case 'b': o.aabb = a->arg; break;
            case 'f': o.min_fraction = a->get_arg<float>(); break;
            case 'p': o.poisson = true; break;
            case 'S': o.scale_factor = a->get_arg<float>(); break;
            case 'C': o.correspondence = true; break;
            case 'F': {
                int const s = a->get_arg<int>();
                o.normals = o.scale = o.conf = true;
                o.depth = "depth-L" + util::string::get<int>(s);
                o.image = s == 0 ? std::string("undistorted") : "undist-L" + util::string::get<int>(s);
                break;
            }
            default: die("unknown option");
        }
    }
    // point formats without scale or confidence; -p needs confidences again
    if (ends_with(o.out, ".npts") || ends_with(o.out, ".bnpts")) { o.normals = true; o.scale = false; o.conf = false; }
    if (o.poisson) { o.normals = true; o.conf = true; }
    return o;
}

void write_correspondence(Options const& o, std::vector<uint32_t> const& xy, std::vector<b200mvs_pset_corr_view> const& views)
{
    std::ofstream data(o.out + "_correspondence-data.csv");
    std::ofstream meta(o.out + "_correspondence-metadata.csv");
    if (!data.good() || !meta.good()) die("Could not open correspondence file(s).");
    std::ostringstream s;
    s << "x, y\n";
    for (std::size_t i = 0; i + 1 < xy.size(); i += 2) s << xy[i] << ", " << xy[i + 1] << "\n";
    data << s.str();
    meta << "View_ID, Width, Height, First_Vertex_Index\n";
    for (b200mvs_pset_corr_view const& v : views)
        meta << v.view_id << ", " << v.width << ", " << v.height << ", " << v.first_index << "\n";
}

} // namespace

int main(int argc, char** argv)
{
    Options o = parse(argc, argv);

    b200mvs_pset_options po;
    std::memset(&po, 0, sizeof(po));
    po.with_normals = o.normals;
    po.with_conf = o.conf;
    po.with_scale = o.scale;
    po.poisson_normals = o.poisson;
    po.correspondence = o.correspondence && o.aabb.empty() && o.mask.empty();
    po.min_valid_fraction = o.min_fraction;
    po.scale_factor = o.scale_factor;
    po.dd_factor = 5.0f;              // mve::geom::DD_FACTOR_DEFAULT
    po.conf_iterations = 4;
    if (!o.aabb.empty()) {
        std::vector<std::string> tok;
        std::stringstream ss(o.aabb);
        for (std::string t; std::getline(ss, t, ',');) tok.push_back(t);
        if (tok.size() != 6) die("Invalid AABB given");
        for (int i = 0; i < 3; ++i) {
            po.aabb_min[i] = util::string::convert<float>(tok[i]);
            po.aabb_max[i] = util::string::convert<float>(tok[i + 3]);
        }
        po.use_aabb = 1;
        std::cout << "Using AABB: (" << po.aabb_min[0] << " " << po.aabb_min[1] << " " << po.aabb_min[2] << ") / ("
                  << po.aabb_max[0] << " " << po.aabb_max[1] << " " << po.aabb_max[2] << ")" << std::endl;
    }
    std::cout << "Using depthmap \"" << o.depth << "\" and color image \"" << o.image << "\"" << std::endl;

    int device = 0;
    if (char const* e = std::getenv("B200MVS_DEVICE")) device = std::atoi(e);
    b200mvs_pset* ps = nullptr;
    check(b200mvs_pset_create(device, &po, &ps), "b200mvs_pset_create");

    mve::Scene::Ptr scene = mve::Scene::create(o.scene_dir);
    mve::Scene::ViewList& views = scene->get_views();
    for (std::size_t i = 0; i < views.size(); ++i) {
        mve::View::Ptr view = views[i];
        if (view == nullptr) continue;
        int const id = view->get_id();
        if (!o.ids.empty() && std::find(o.ids.begin(), o.ids.end(), id) == o.ids.end()) continue;
        mve::CameraInfo const& cam = view->get_camera();
        if (cam.flen == 0.0f) continue;
        mve::FloatImage::Ptr dm = view->get_float_image(o.depth);
        if (dm == nullptr) continue;
        if (dm->channels() != 1) die("depth map \"" + o.depth + "\" of view \"" + view->get_name() + "\" has more than one channel");
        mve::ByteImage::Ptr ci;
        if (!o.image.empty()) ci = view->get_byte_image(o.image);
        if (ci != nullptr && (ci->width() != dm->width() || ci->height() != dm->height()))
            die("Color image dimension mismatch");
        b200mvs_pset_camera const pc = camera_of(cam);
        b200mvs_pset_view r;
        check(b200mvs_pset_add_view(ps, id, dm->get_data_pointer(), dm->width(), dm->height(),
                                    ci ? ci->get_data_pointer() : nullptr, ci ? ci->channels() : 0, &pc, &r),
              "b200mvs_pset_add_view");
        if (!r.added)
            std::cout << "View " << view->get_name() << ": Fill status " << util::string::get_fixed(r.fraction * 100.0f, 2)
                      << "%, skipping." << std::endl;
        else
            std::cout << "Processing view \"" << view->get_name() << "\"" << (ci != nullptr ? " (with colors)" : "") << "..." << std::endl;
        dm.reset();
        ci.reset();
        view->cache_cleanup();
    }

    if (!o.mask.empty()) {
        std::cout << "Filtering points using silhouette masks..." << std::endl;
        std::vector<mve::ByteImage::Ptr> keep;
        std::vector<uint8_t const*> ptrs;
        std::vector<int32_t> ws, hs;
        std::vector<b200mvs_pset_camera> cams;
        for (std::size_t i = 0; i < views.size(); ++i) {
            mve::View::Ptr view = views[i];
            if (view == nullptr || view->get_camera().flen == 0.0f) continue;
            mve::ByteImage::Ptr mask = view->get_byte_image(o.mask);
            if (mask == nullptr) { std::cout << "Mask not found for image \"" << view->get_name() << "\", skipping." << std::endl; continue; }
            if (mask->channels() != 1) { std::cout << "Expected 1-channel mask for image \"" << view->get_name() << "\", skipping." << std::endl; continue; }
            std::cout << "Processing mask for \"" << view->get_name() << "\"..." << std::endl;
            keep.push_back(mask);
            ptrs.push_back(mask->get_data_pointer());
            ws.push_back(mask->width());
            hs.push_back(mask->height());
            cams.push_back(camera_of(view->get_camera()));
            view->cache_cleanup();
        }
        uint64_t filtered = 0;
        check(b200mvs_pset_clip_masks(ps, (int)ptrs.size(), ptrs.data(), ws.data(), hs.data(), cams.data(), &filtered),
              "b200mvs_pset_clip_masks");
        std::cout << "Filtered a total of " << filtered << " points." << std::endl;
    }

    b200mvs_pset_info info;
    check(b200mvs_pset_get_info(ps, &info), "b200mvs_pset_get_info");
    mve::TriangleMesh::Ptr pset = mve::TriangleMesh::create();
    mve::TriangleMesh::VertexList& verts = pset->get_vertices();
    verts.resize(info.n_points);
    pset->get_vertex_colors().resize(info.n_colors);
    float* normals = nullptr;
    float* values = nullptr;
    float* confs = nullptr;
    if (o.normals) pset->get_vertex_normals().resize(info.n_points);
    if (o.scale) pset->get_vertex_values().resize(info.n_points);
    if (o.conf) pset->get_vertex_confidences().resize(info.n_points);
    // pointers into the mesh's lists, taken only from lists that have entries
    if (info.n_points) {
        if (o.normals) normals = pset->get_vertex_normals().front().begin();
        if (o.scale) values = pset->get_vertex_values().data();
        if (o.conf) confs = pset->get_vertex_confidences().data();
    }
    check(b200mvs_pset_read(ps, info.n_points ? verts.front().begin() : nullptr, normals,
                            info.n_colors ? pset->get_vertex_colors().front().begin() : nullptr, values, confs),
          "b200mvs_pset_read");
    std::vector<uint32_t> corr_xy;
    std::vector<b200mvs_pset_corr_view> corr_views;
    if (po.correspondence) {
        corr_xy.resize(2 * info.n_points);
        corr_views.resize(info.n_views);
        check(b200mvs_pset_read_correspondence(ps, corr_xy.data(), corr_views.data()), "b200mvs_pset_read_correspondence");
    }
    if (std::getenv("B200MVS_PSET_STATS"))
        std::cout << "b200mvs_pset: peak device bytes " << info.peak_device_bytes << ", device ms: pointset " << info.ms_pointset
                  << ", filter " << info.ms_filter << ", mask " << info.ms_mask << std::endl;
    b200mvs_pset_destroy(ps);

    std::cout << "Writing final point set (" << verts.size() << " points)..." << std::endl;
    if (ends_with(o.out, ".ply")) {
        mve::geom::SavePLYOptions opts;
        opts.write_vertex_normals = o.normals;
        opts.write_vertex_values = o.scale;
        opts.write_vertex_confidences = o.conf;
        mve::geom::save_ply_mesh(pset, o.out, opts);
    } else {
        mve::geom::save_mesh(pset, o.out);
    }
    if (po.correspondence) write_correspondence(o, corr_xy, corr_views);
    return EXIT_SUCCESS;
}
