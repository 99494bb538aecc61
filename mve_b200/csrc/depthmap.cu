// Depth-map consumers that run right after dmrecon (SURVEY.md 8f rank 2 and 3), on the device:
//   * mve::image::depthmap_confidence_clean and depthmap_cleanup (libs/mve/depthmap.cc:25-131)
//   * mve::geom::depthmap_triangulate with pixel_3dpos / pixel_footprint (libs/mve/depthmap.cc:136-375), the per-view work of
//     apps/scene2pset (scene2pset.cc:264-328): vertex ids, vertices, colours and faces in EXACTLY the reference's order.
// All of these are streaming kernels over the maps of a batch; the results are bit-exact for the integer parts (masks, component
// sizes, vertex ids, faces) and for the float parts that are pure per-pixel functions evaluated in the reference's operation
// order with IEEE operations (__fmul_rn / __fadd_rn; __fmaf_rn only where the reference build itself contracts and the
// result decides a face: pixel_footprint).
#include "../../include/b200mvs.h"
#include "pset_device.cuh"
#include "host_common.cuh"

#include <cub/device/device_scan.cuh>
#include <cuda/std/functional>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>

using namespace b200mvs_host;

namespace {

// ---- depthmap_confidence_clean and depthmap_cleanup over a batch of maps ----
// One launch covers every map of a batch (cleanup: of a chunk, DmBatch), DM_BLOCK threads per block.  Each map's pixels
// start on a block boundary, and a block reads its map from a block -> map table built on the host, so no thread searches
// the map list.  The host entry points run the same kernels on a batch of one staged map.
constexpr unsigned DM_BLOCK = 256;
// Cleanup and triangulation take the maps of a batch in chunks: the longest run of consecutive maps whose pixels total at
// most DM_CHUNK_PIXELS, a larger map being a chunk of its own.  A chunk's labels then fit 32 bits, its (vertices << 32)
// | faces scan is exact, and the workspace is sized to the largest chunk.
constexpr uint64_t DM_CHUNK_PIXELS = 1ull << 28;
struct DmMap {
    const float* dm;              // depth read
    float* out;                   // depth written: cleanup's out, confidence_clean's depth (== dm)
    const float* cm;              // confidence_clean: the confidence map
    unsigned long long thres;     // cleanup: the map's threshold, converted to size_t as the reference compares it
    unsigned w, h, n;             // n = w * h <= 0xFFFFFFF0
    unsigned label0;              // cleanup: label of the map's first pixel, its offset in the chunk's pixels
    unsigned block0;              // the map's first block in its launch
};
// The map of the calling block and the pixel of the calling thread in it (>= M.n: none); Map is DmMap or TriMap
template <class Map>
__device__ __forceinline__ const Map& map_of(const Map* __restrict__ maps, const unsigned* __restrict__ block_map, unsigned& i)
{
    const Map& M = maps[block_map[blockIdx.x]];
    i = (blockIdx.x - M.block0) * DM_BLOCK + threadIdx.x;
    return M;
}

// depthmap_confidence_clean (depthmap.cc:118-131)
__global__ void k_conf_clean(const DmMap* __restrict__ maps, const unsigned* __restrict__ block_map)
{
    unsigned i;
    const DmMap& M = map_of(maps, block_map, i);
    if (i < M.n && M.cm[i] <= 0.0f) M.out[i] = 0.0f;
}

// ---- depthmap_cleanup (depthmap.cc:25-113): 4-connected components of dm != 0, components smaller than thres are erased ----
// Union-find over the pixels of a chunk: a pixel's label is its index in the chunk's maps laid end to end.  Every pixel
// links to its right and lower neighbour in its own map (atomicMin on roots), so no component crosses a map boundary; the
// roots are then flattened, counted, and small components zeroed with their map's threshold.  Component sizes are exact,
// so the result equals the reference's region growing bit for bit.
__device__ __forceinline__ unsigned uf_find(const unsigned* parent, unsigned i)
{
    unsigned p = parent[i];
    while (p != i) { i = p; p = parent[i]; }
    return i;
}
__device__ __forceinline__ void uf_union(unsigned* parent, unsigned a, unsigned b)
{
    for (;;) {
        a = uf_find(parent, a);
        b = uf_find(parent, b);
        if (a == b) return;
        if (a < b) { const unsigned t = a; a = b; b = t; }      // a > b: hang a below b
        const unsigned old = atomicMin(&parent[a], b);
        if (old == a) return;
        a = old;                                                // somebody re-rooted a meanwhile: continue from there
    }
}
// every label of a chunk its own root, with no pixels counted
__global__ void k_cc_init(unsigned* __restrict__ parent, unsigned* __restrict__ count, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    parent[i] = (unsigned)i;
    count[i] = 0u;
}
__global__ void k_cc_link(const DmMap* __restrict__ maps, const unsigned* __restrict__ block_map, unsigned* __restrict__ parent)
{
    unsigned i;
    const DmMap& M = map_of(maps, block_map, i);
    if (i >= M.n) return;
    const float* dm = M.dm;
    if (dm[i] == 0.0f) return;
    const unsigned y = i / M.w, x = i - y * M.w, l = M.label0 + i;
    if (x + 1 < M.w && dm[i + 1] != 0.0f) uf_union(parent, l, l + 1);
    if (y + 1 < M.h && dm[(size_t)i + M.w] != 0.0f) uf_union(parent, l, l + M.w);
}
// flatten and count
__global__ void k_cc_count(const DmMap* __restrict__ maps, const unsigned* __restrict__ block_map, unsigned* __restrict__ parent,
                           unsigned* __restrict__ count)
{
    unsigned i;
    const DmMap& M = map_of(maps, block_map, i);
    if (i >= M.n || M.dm[i] == 0.0f) return;
    const unsigned l = M.label0 + i, r = uf_find(parent, l);
    parent[l] = r;
    atomicAdd(&count[r], 1u);
}
// out may be dm: a thread reads and writes its own pixel only, and the earlier phases are complete
__global__ void k_cc_erase(const DmMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned* __restrict__ parent,
                           const unsigned* __restrict__ count)
{
    unsigned i;
    const DmMap& M = map_of(maps, block_map, i);
    if (i >= M.n) return;
    const float d = M.dm[i];
    M.out[i] = (d != 0.0f && (unsigned long long)count[parent[M.label0 + i]] < M.thres) ? 0.0f : d;
}

// ---- depthmap_triangulate and the per-vertex attributes over a batch of maps ----
// As the cleanup kernels: one launch covers every map of a chunk (TriBatch), DM_BLOCK threads per block and a thread per
// pixel, each map starting on a block boundary, and a block reads its map from the block -> map table.  The chunk's
// workspace (codes, counts and their scan, confidence rings) holds its maps' pixels end to end, map by map from px0;
// one exclusive scan over the chunk's counts gives every pixel its first vertex and face, and each map subtracts the
// scan at its own px0, so its ids start at 0.  The host entry points and a point-set handle run a batch of one map.
struct InvProj { float m[9]; };
// A colour image on the device: channel k of pixel (x, y) at p[(y * pitch + x) * stride + k]
struct Color {
    const uint8_t* p = nullptr;
    int ch = 0, stride = 0, pitch = 0;
};
struct TriMap {
    const float* dm;
    unsigned w, h, n;             // n = w * h
    unsigned px0;                 // the map's first pixel in its chunk's workspace
    unsigned block0;              // the map's first block in its launch
    int filled;                   // 0: only counted; the kernels after the scan skip the map
    InvProj P;
    int has_ctw;
    float ctw[16];                // 4x4 row-major camera-to-world when has_ctw
    Color color;                  // read when colors != NULL
    unsigned* vids;               // w * h vertex ids
    float* verts;                 // per vertex, never NULL in a filled map: k_tri_vertices writes every vertex
    float *colors, *normals, *scales, *confs;             // per vertex, NULL: not wanted
    unsigned* faces;              // NULL: not wanted
};

// pixel_3dpos / pixel_footprint (depthmap.cc:136-156): ray = invproj * (x + .5, y + .5, 1), math::Matrix::mult accumulates
// from zero, left to right.
__device__ __forceinline__ void pixel_ray(const InvProj& P, int x, int y, float& rx, float& ry, float& rz)
{
    const float vx = (float)x + 0.5f, vy = (float)y + 0.5f, vz = 1.0f;
    rx = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(P.m[0], vx)), __fmul_rn(P.m[1], vy)), __fmul_rn(P.m[2], vz));
    ry = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(P.m[3], vx)), __fmul_rn(P.m[4], vy)), __fmul_rn(P.m[5], vz));
    rz = __fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(P.m[6], vx)), __fmul_rn(P.m[7], vy)), __fmul_rn(P.m[8], vz));
}
__device__ __forceinline__ float vec_norm(float x, float y, float z)
{
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(x, x)), __fmul_rn(y, y)), __fmul_rn(z, z)));
}
// The footprint decides which faces exist, so it repeats the reference build's own arithmetic to the bit: with its flags
// (-O3 -funsafe-math-optimizations on an FMA target) g++ contracts the ray and the squared norm of pixel_footprint into
// rx = fma(m0, vx, fma(m1, vy, m2)), ry = fma(m3, vx, fma(m4, vy, m5)), rz = fma(m7, vy, fma(m6, vx, m8)) and
// |r|^2 = fma(rz, rz, rx*rx + ry*ry), then divides (m0 * depth) by the square root.
__device__ __forceinline__ float pixel_footprint(const InvProj& P, int x, int y, float depth)
{
    const float vx = (float)x + 0.5f, vy = (float)y + 0.5f;
    const float rx = __fmaf_rn(P.m[0], vx, __fmaf_rn(P.m[1], vy, P.m[2]));
    const float ry = __fmaf_rn(P.m[3], vx, __fmaf_rn(P.m[4], vy, P.m[5]));
    const float rz = __fmaf_rn(P.m[7], vy, __fmaf_rn(P.m[6], vx, P.m[8]));
    const float sq = __fmaf_rn(rz, rz, __fadd_rn(__fmul_rn(rx, rx), __fmul_rn(ry, ry)));
    return __fdiv_rn(__fmul_rn(P.m[0], depth), __fsqrt_rn(sq));
}

// corner j of the 2x2 block at i: pixel i + (j % 2) + width * (j / 2); the four candidate triangles (depthmap.cc:247-250)
__constant__ int c_tris[4][3] = {{0, 2, 1}, {0, 3, 1}, {0, 2, 3}, {1, 2, 3}};

// dd_diag is the diagonal factor `dd_factor *= MATH_SQRT2` of depthmap.cc:198: a float times a double literal, so the
// reference rounds the product through double.  The host computes it once (b200mvs_depthmap_pointset).
__device__ __forceinline__ bool is_depthdisc(const float* widths, const float* depths, float dd_factor, float dd_diag, int i1, int i2)
{
    int i_min = i1, i_max = i2;
    if (depths[i2] < depths[i1]) { i_min = i2; i_max = i1; }
    const float dd = i1 + i2 == 3 ? dd_diag : dd_factor;
    return __fadd_rn(depths[i_max], -depths[i_min]) > __fmul_rn(widths[i_min], dd);
}

// Which triangles the block at (x, y) issues (depthmap.cc:229-301): low nibble first triangle (1..4, 0 none), high nibble second.
__device__ __forceinline__ unsigned block_code(const float* __restrict__ dm, int w, int h, int x, int y, const InvProj& P, float dd_factor,
                                               float dd_diag)
{
    if (x < 0 || y < 0 || x >= w - 1 || y >= h - 1) return 0u;
    const size_t i = (size_t)y * w + x;
    const float depths[4] = {dm[i], dm[i + 1], dm[i + w], dm[i + w + 1]};
    int mask = 0, pixels = 0;
    for (int j = 0; j < 4; ++j) if (depths[j] > 0.0f) { mask |= 1 << j; ++pixels; }
    if (pixels < 3) return 0u;
    int tri[2] = {0, 0};
    switch (mask) {
        case 7: tri[0] = 1; break;
        case 11: tri[0] = 2; break;
        case 13: tri[0] = 3; break;
        case 14: tri[0] = 4; break;
        case 15: {
            const float d1 = fabsf(__fadd_rn(depths[0], -depths[3])), d2 = fabsf(__fadd_rn(depths[1], -depths[2]));
            if (d1 < d2) { tri[0] = 2; tri[1] = 3; } else { tri[0] = 1; tri[1] = 4; }
            break;
        }
        default: return 0u;
    }
    if (dd_factor > 0.0f) {
        float widths[4] = {0.f, 0.f, 0.f, 0.f};
        for (int j = 0; j < 4; ++j) if (depths[j] != 0.0f) widths[j] = pixel_footprint(P, x + (j % 2), y + (j / 2), depths[j]);
        for (int j = 0; j < 2 && tri[j] != 0; ++j) {
            const int* tv = c_tris[tri[j] - 1];
            if (is_depthdisc(widths, depths, dd_factor, dd_diag, tv[0], tv[1])) tri[j] = 0;
            if (is_depthdisc(widths, depths, dd_factor, dd_diag, tv[1], tv[2])) tri[j] = 0;
            if (is_depthdisc(widths, depths, dd_factor, dd_diag, tv[2], tv[0])) tri[j] = 0;
        }
    }
    return (unsigned)tri[0] | ((unsigned)tri[1] << 4);
}
__device__ __forceinline__ bool code_uses(unsigned code, int corner)
{
    for (int j = 0; j < 2; ++j) {
        const int t = (code >> (4 * j)) & 0xF;
        if (!t) continue;
        const int* tv = c_tris[t - 1];
        if (tv[0] == corner || tv[1] == corner || tv[2] == corner) return true;
    }
    return false;
}

// The map of the calling block, the pixel (x, y) of the calling thread in it; false when the thread has none
__device__ __forceinline__ bool tri_pixel(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const TriMap*& M,
                                          unsigned& i, int& x, int& y)
{
    M = &map_of(maps, block_map, i);
    if (i >= M->n) return false;
    y = (int)(i / M->w);
    x = (int)(i - (unsigned)y * M->w);
    return true;
}

__global__ void k_tri_codes(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, float dd_factor, float dd_diag,
                            unsigned char* __restrict__ codes)
{
    const TriMap* M; unsigned i; int x, y;
    if (!tri_pixel(maps, block_map, M, i, x, y)) return;
    codes[(size_t)M->px0 + i] = (unsigned char)block_code(M->dm, (int)M->w, (int)M->h, x, y, M->P, dd_factor, dd_diag);
}

// The reference numbers a vertex when a triangle references its pixel for the first time, blocks in raster order
// (dm_make_triangle, depthmap.cc:160-183).  A pixel p = (px, py) can be referenced by the blocks (px-1, py-1) [as corner 3],
// (px, py-1) [corner 2], (px-1, py) [corner 1], (px, py) [corner 0], visited in this order: the first of them that uses the
// corner OWNS the vertex.  Per block: how many vertices it owns (high word) and how many faces it issues (low word); one
// exclusive scan over the blocks in raster order then gives every block its first vertex id and its first face.
__device__ __forceinline__ bool owns(const unsigned char* __restrict__ codes, int w, int h, int bx, int by, int corner)
{
    // pixel of `corner` of block (bx, by); earlier blocks (in raster order) that could reference the same pixel
    const int px = bx + (corner & 1), py = by + (corner >> 1);
    // candidates in visiting order: (px-1,py-1) c3, (px,py-1) c2, (px-1,py) c1, (px,py) c0; stop at (bx, by)
    const int cx[4] = {px - 1, px, px - 1, px}, cy[4] = {py - 1, py - 1, py, py}, cc[4] = {3, 2, 1, 0};
    for (int k = 0; k < 4; ++k) {
        if (cx[k] == bx && cy[k] == by) return true;              // nobody before us used it
        if (cx[k] < 0 || cy[k] < 0 || cx[k] >= w - 1 || cy[k] >= h - 1) continue;
        if (code_uses(codes[(size_t)cy[k] * w + cx[k]], cc[k])) return false;
    }
    return true;
}
__global__ void k_tri_counts(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned char* __restrict__ chunk_codes,
                             unsigned long long* __restrict__ counts)
{
    const TriMap* M; unsigned i; int x, y;
    if (!tri_pixel(maps, block_map, M, i, x, y)) return;
    const unsigned char* codes = chunk_codes + M->px0;
    const int w = (int)M->w, h = (int)M->h;
    const unsigned code = codes[i];
    unsigned nv = 0u, nf = 0u, seen = 0u;
    for (int j = 0; j < 2; ++j) {
        const int t = (code >> (4 * j)) & 0xF;
        if (!t) continue;
        ++nf;
        for (int q = 0; q < 3; ++q) {
            const int c = c_tris[t - 1][q];
            if (seen & (1u << c)) continue;
            seen |= 1u << c;
            if (owns(codes, w, h, x, y, c)) ++nv;
        }
    }
    counts[(size_t)M->px0 + i] = ((unsigned long long)nv << 32) | nf;
}
// Each map of a chunk's (vertices << 32) | faces: the scan at its end less the scan at its start
__global__ void k_tri_totals(const TriMap* __restrict__ maps, unsigned n_maps, const unsigned long long* __restrict__ offsets,
                             unsigned long long* __restrict__ totals)
{
    const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_maps) return;
    const TriMap& M = maps[j];
    totals[j] = offsets[(size_t)M.px0 + M.n] - offsets[M.px0];
}
// no vertex yet at any pixel of a filled map
__global__ void k_tri_clear(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map)
{
    unsigned i;
    const TriMap& M = map_of(maps, block_map, i);
    if (i < M.n && M.filled) M.vids[i] = 0xFFFFFFFFu;
}
__global__ void k_tri_vertices(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned char* __restrict__ chunk_codes,
                               const unsigned long long* __restrict__ offsets)
{
    const TriMap* M; unsigned i; int x, y;
    if (!tri_pixel(maps, block_map, M, i, x, y) || !M->filled) return;
    const unsigned char* codes = chunk_codes + M->px0;
    const int w = (int)M->w, h = (int)M->h;
    const InvProj& P = M->P;
    const float* ctw = M->has_ctw ? M->ctw : nullptr;
    unsigned* vids = M->vids;
    float *verts = M->verts, *colors = M->colors;
    const unsigned code = codes[i];
    unsigned id = (unsigned)((offsets[(size_t)M->px0 + i] - offsets[M->px0]) >> 32), seen = 0u;
    for (int j = 0; j < 2; ++j) {
        const int t = (code >> (4 * j)) & 0xF;
        if (!t) continue;
        for (int q = 0; q < 3; ++q) {
            const int c = c_tris[t - 1][q];
            if (seen & (1u << c)) continue;
            seen |= 1u << c;
            if (!owns(codes, w, h, x, y, c)) continue;
            const int px = x + (c & 1), py = y + (c >> 1);
            const size_t pi = (size_t)py * w + px;
            vids[pi] = id;
            // pixel_3dpos: ray.normalized() * depth (depthmap.cc:149-156)
            float rx, ry, rz;
            pixel_ray(P, px, py, rx, ry, rz);
            const float nrm = vec_norm(rx, ry, rz), d = M->dm[pi];
            float vx = __fmul_rn(__fdiv_rn(rx, nrm), d), vy = __fmul_rn(__fdiv_rn(ry, nrm), d), vz = __fmul_rn(__fdiv_rn(rz, nrm), d);
            if (ctw) {
                // mesh_transform with the 4x4 camera-to-world matrix (mesh_tools.cc: Matrix4f::mult(v, 1))
                const float ox = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(ctw[0], vx)), __fmul_rn(ctw[1], vy)), __fmul_rn(ctw[2], vz)), __fmul_rn(ctw[3], 1.0f));
                const float oy = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(ctw[4], vx)), __fmul_rn(ctw[5], vy)), __fmul_rn(ctw[6], vz)), __fmul_rn(ctw[7], 1.0f));
                const float oz = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.f, __fmul_rn(ctw[8], vx)), __fmul_rn(ctw[9], vy)), __fmul_rn(ctw[10], vz)), __fmul_rn(ctw[11], 1.0f));
                vx = ox; vy = oy; vz = oz;
            }
            verts[3 * (size_t)id] = vx; verts[3 * (size_t)id + 1] = vy; verts[3 * (size_t)id + 2] = vz;
            if (colors) {
                // depthmap.cc:349-364: (r, g, b, 255) / 255, grey expanded; texels cstride bytes apart, rows cpitch texels
                const unsigned char* c = M->color.p + ((size_t)py * M->color.pitch + px) * M->color.stride;
                const float r = (float)c[0], g = M->color.ch >= 3 ? (float)c[1] : r, b = M->color.ch >= 3 ? (float)c[2] : r;
                colors[4 * (size_t)id] = __fdiv_rn(r, 255.0f); colors[4 * (size_t)id + 1] = __fdiv_rn(g, 255.0f);
                colors[4 * (size_t)id + 2] = __fdiv_rn(b, 255.0f); colors[4 * (size_t)id + 3] = 1.0f;
            }
            ++id;
        }
    }
}
__global__ void k_tri_faces(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned char* __restrict__ chunk_codes,
                            const unsigned long long* __restrict__ offsets)
{
    unsigned i;
    const TriMap& M = map_of(maps, block_map, i);
    if (i >= M.n || !M.faces) return;
    const unsigned* vids = M.vids;
    unsigned* faces = M.faces;
    const size_t w = M.w;
    const unsigned code = chunk_codes[(size_t)M.px0 + i];
    size_t f = (size_t)((offsets[(size_t)M.px0 + i] - offsets[M.px0]) & 0xFFFFFFFFull);
    for (int j = 0; j < 2; ++j) {
        const int t = (code >> (4 * j)) & 0xF;
        if (!t) continue;
        for (int q = 0; q < 3; ++q) {
            const int c = c_tris[t - 1][q];
            faces[3 * f + q] = vids[i + (c & 1) + w * (c >> 1)];
        }
        ++f;
    }
}

// ---- per-vertex attributes of the triangulated depth map: what apps/scene2pset adds per view (scene2pset.cc:316-358) ----
// All of them are functions of a vertex' adjacent faces, which on a depth-map mesh are the <= 8 triangles of the four 2x2
// blocks around its pixel; visiting those blocks in raster order (and a block's triangles in emission order) enumerates the
// faces in ascending face id - the order in which the reference accumulates (mesh.cc:45-119, mesh_info.cc:28-33).
struct AdjFace { unsigned a, b, c, first, second; };
constexpr unsigned RING_NONE = 0xFFFFFFFFu;          // confidence ring of a vertex no border ring has reached (yet)

__device__ __forceinline__ int adjacent_faces(const unsigned char* __restrict__ codes, const unsigned* __restrict__ vids, int w, int h,
                                              int px, int py, unsigned v, AdjFace* out)
{
    const int bx[4] = {px - 1, px, px - 1, px}, by[4] = {py - 1, py - 1, py, py}, corner[4] = {3, 2, 1, 0};
    int n = 0;
    for (int k = 0; k < 4; ++k) {
        if (bx[k] < 0 || by[k] < 0 || bx[k] >= w - 1 || by[k] >= h - 1) continue;
        const size_t bi = (size_t)by[k] * w + bx[k];
        const unsigned code = codes[bi];
        for (int j = 0; j < 2; ++j) {
            const int t = (code >> (4 * j)) & 0xF;
            if (!t) continue;
            const int* tv = c_tris[t - 1];
            int pos = -1;
            for (int q = 0; q < 3; ++q) if (tv[q] == corner[k]) pos = q;
            if (pos < 0) continue;
            unsigned id[3];
            for (int q = 0; q < 3; ++q) id[q] = vids[bi + (tv[q] & 1) + (size_t)w * (tv[q] >> 1)];
            AdjFace f;
            f.a = id[0]; f.b = id[1]; f.c = id[2];
            f.first = id[(pos + 1) % 3]; f.second = id[(pos + 2) % 3];
            out[n++] = f;
        }
    }
    (void)v;
    return n;
}

__device__ __forceinline__ float clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// MeshInfo::update_vertex (mesh_info.cc:55-163): chains the adjacent faces; returns the class (0 simple, 1 complex, 2 border,
// 3 unreferenced - MeshInfo::VertexClass) and the adjacent vertices in the reference's order.
__device__ __forceinline__ int classify_vertex(const AdjFace* faces, int n, unsigned* verts, int* n_verts)
{
    *n_verts = 0;
    if (n == 0) return 3;
    bool used[8] = {false, false, false, false, false, false, false, false};
    unsigned sf[17], ss[17];                 // sorted chain as a deque in the middle of an array
    int lo = 8, hi = 8;
    sf[8] = faces[0].first; ss[8] = faces[0].second; used[0] = true;
    int left = n - 1;
    while (left > 0) {
        const unsigned front_id = sf[lo], back_id = ss[hi];
        bool found = false;
        for (int i = 0; i < n; ++i) {
            if (used[i]) continue;
            if (front_id == faces[i].second) { --lo; sf[lo] = faces[i].first; ss[lo] = faces[i].second; used[i] = true; found = true; break; }
            if (back_id == faces[i].first) { ++hi; sf[hi] = faces[i].first; ss[hi] = faces[i].second; used[i] = true; found = true; break; }
        }
        if (!found) break;
        --left;
    }
    if (left > 0) {
        // complex: unique, ascending list of all adjacent vertices (std::set)
        unsigned tmp[16];
        int m = 0;
        for (int i = 0; i < n; ++i) { tmp[m++] = faces[i].first; tmp[m++] = faces[i].second; }
        for (int i = 1; i < m; ++i) { const unsigned key = tmp[i]; int j = i - 1; while (j >= 0 && tmp[j] > key) { tmp[j + 1] = tmp[j]; --j; } tmp[j + 1] = key; }
        int k = 0;
        for (int i = 0; i < m; ++i) if (i == 0 || tmp[i] != tmp[i - 1]) verts[k++] = tmp[i];
        *n_verts = k;
        return 1;
    }
    const bool simple = sf[lo] == ss[hi];
    int k = 0;
    for (int i = lo; i <= hi; ++i) verts[k++] = sf[i];
    if (!simple) verts[k++] = ss[hi];
    *n_verts = k;
    return simple ? 0 : 2;
}

// ring: the chunk's confidence rings, NULL when no confidences are computed
__global__ void k_vertex_attributes(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned char* __restrict__ chunk_codes,
                                    float scale_factor, unsigned* __restrict__ chunk_ring)
{
    const TriMap* M; unsigned pi; int x, y;
    if (!tri_pixel(maps, block_map, M, pi, x, y) || !M->filled) return;
    const unsigned char* codes = chunk_codes + M->px0;
    const unsigned* vids = M->vids;
    const int w = (int)M->w, h = (int)M->h;
    const float* verts = M->verts;
    float *normals = M->normals, *scales = M->scales;
    unsigned* ring = chunk_ring ? chunk_ring + M->px0 : nullptr;
    const unsigned v = vids[pi];
    if (ring) ring[pi] = RING_NONE;
    if (v == 0xFFFFFFFFu) return;
    AdjFace faces[8];
    const int n = adjacent_faces(codes, vids, w, h, x, y, v, faces);
    if (normals) {
        // TriangleMesh::recalc_normals, angle-weighted pseudo normals (mesh.cc:45-151)
        float nx = 0.f, ny = 0.f, nz = 0.f;
        for (int i = 0; i < n; ++i) {
            const float* A = verts + 3 * (size_t)faces[i].a; const float* B = verts + 3 * (size_t)faces[i].b; const float* C = verts + 3 * (size_t)faces[i].c;
            const float abx = B[0] - A[0], aby = B[1] - A[1], abz = B[2] - A[2];
            const float bcx = C[0] - B[0], bcy = C[1] - B[1], bcz = C[2] - B[2];
            const float cax = A[0] - C[0], cay = A[1] - C[1], caz = A[2] - C[2];
            // fn = ab x (-ca)
            float fx = aby * (-caz) - abz * (-cay), fy = abz * (-cax) - abx * (-caz), fz = abx * (-cay) - aby * (-cax);
            const float fnl = sqrtf(fx * fx + fy * fy + fz * fz);
            if (fnl == 0.0f) continue;
            fx /= fnl; fy /= fnl; fz /= fnl;
            const float abl = sqrtf(abx * abx + aby * aby + abz * abz), bcl = sqrtf(bcx * bcx + bcy * bcy + bcz * bcz), cal = sqrtf(cax * cax + cay * cay + caz * caz);
            float ratio;
            if (faces[i].a == v) ratio = (abx / abl) * (-cax / cal) + (aby / abl) * (-cay / cal) + (abz / abl) * (-caz / cal);
            else if (faces[i].b == v) ratio = (-abx / abl) * (bcx / bcl) + (-aby / abl) * (bcy / bcl) + (-abz / abl) * (bcz / bcl);
            else ratio = (cax / cal) * (-bcx / bcl) + (cay / cal) * (-bcy / bcl) + (caz / cal) * (-bcz / bcl);
            const float angle = acosf(clampf(ratio, -1.0f, 1.0f));
            nx += fx * angle; ny += fy * angle; nz += fz * angle;
        }
        const float vnl = sqrtf(nx * nx + ny * ny + nz * nz);
        if (vnl > 0.0f) { nx /= vnl; ny /= vnl; nz /= vnl; }
        normals[3 * (size_t)v] = nx; normals[3 * (size_t)v + 1] = ny; normals[3 * (size_t)v + 2] = nz;
    }
    if (scales || ring) {
        unsigned adj[16];
        int na = 0;
        const int cls = classify_vertex(faces, n, adj, &na);
        if (ring && cls == 2) ring[pi] = 0;                       // MeshInfo::VERTEX_CLASS_BORDER starts the confidence rings
        if (scales) {
            // scene2pset.cc:347-357: mean distance to the adjacent vertices, times the scale factor
            const float* P0 = verts + 3 * (size_t)v;
            float sum = 0.f;
            for (int k = 0; k < na; ++k) {
                const float* Q = verts + 3 * (size_t)adj[k];
                const float dx = P0[0] - Q[0], dy = P0[1] - Q[1], dz = P0[2] - Q[2];
                sum += sqrtf(dx * dx + dy * dy + dz * dz);
            }
            sum /= (float)na;
            scales[v] = sum * scale_factor;
        }
    }
}

// depthmap_mesh_confidences (depthmap.cc:497-548): ring d = vertices at d face-edge hops from a border vertex get d / iterations.
// One launch per ring over every map of a chunk.  A ring distance is below the number of vertices (< 2^32), so RING_NONE
// never collides with one.  A round that reaches a vertex of any map stores its d in *last_hit; once a round reaches
// none, no later round can, and the host stops.
__global__ void k_conf_ring(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned char* __restrict__ chunk_codes,
                            const unsigned* __restrict__ chunk_in, unsigned* __restrict__ chunk_out, unsigned d, unsigned* __restrict__ last_hit)
{
    const TriMap* M; unsigned pi; int x, y;
    if (!tri_pixel(maps, block_map, M, pi, x, y) || !M->filled) return;
    const unsigned char* codes = chunk_codes + M->px0;
    const unsigned* vids = M->vids;
    const unsigned* ring_in = chunk_in + M->px0;
    const int w = (int)M->w, h = (int)M->h;
    unsigned r = ring_in[pi];
    const unsigned v = vids[pi];
    if (v != 0xFFFFFFFFu && r == RING_NONE) {
        AdjFace faces[8];
        const int n = adjacent_faces(codes, vids, w, h, x, y, v, faces);
        // the adjacent vertices are pixels of the 3x3 neighbourhood: look their rings up through their vertex ids
        bool hit = false;
        for (int dy = -1; dy <= 1 && !hit; ++dy)
            for (int dx = -1; dx <= 1 && !hit; ++dx) {
                const int qx = x + dx, qy = y + dy;
                if ((dx == 0 && dy == 0) || qx < 0 || qy < 0 || qx >= w || qy >= h) continue;
                const size_t qi = (size_t)qy * w + qx;
                if (ring_in[qi] != d - 1u) continue;
                const unsigned u = vids[qi];
                for (int i = 0; i < n; ++i) if (faces[i].first == u || faces[i].second == u) { hit = true; break; }
            }
        if (hit) { r = d; *last_hit = d; }
    }
    chunk_out[(size_t)M->px0 + pi] = r;
}
__global__ void k_conf_write(const TriMap* __restrict__ maps, const unsigned* __restrict__ block_map, const unsigned* __restrict__ chunk_ring,
                             int iterations)
{
    unsigned i;
    const TriMap& M = map_of(maps, block_map, i);
    if (i >= M.n || !M.confs) return;
    const unsigned v = M.vids[i];
    if (v == 0xFFFFFFFFu) return;
    const unsigned r = chunk_ring[(size_t)M.px0 + i];
    // current * (1 / iterations): the reference build hoists the division of depthmap.cc:527 out of its loop
    M.confs[v] = r < (unsigned)iterations ? __fmul_rn((float)r, __frcp_rn((float)iterations)) : 1.0f;
}

// ---- one view's pointset on the device, in a workspace that outlives the call ----
// Buffers grow to the largest view they have served and are reused after that, so a handle that adds many views holds
// one view's worth of device memory (b200mvs_pset_*); the stateless entry point makes a workspace per call.
struct Buf { void* p = nullptr; size_t n = 0; };
struct Work {
    enum Id { dm, codes, counts, offsets, vids, tab, color, tmp, verts, colors, faces, normals, scales, confs, ring0, ring1, last_hit,
              // scene-level filters of the handle: fill lanes, box flags + their scan, compacted attributes, pixel of each vertex
              fill, flags, pos, scan_tmp, o_verts, o_normals, o_colors, o_scales, o_confs, pix, N_BUFS };
    Buf buf[N_BUFS];
    size_t held = 0, peak = 0;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // 0-3: timing; 4: the caller's stream
    b200mvs_pset_dev::Allocator A;      // no alloc function: cudaMalloc
    Work() = default;
    Work(const Work&) = delete;
    Work& operator=(const Work&) = delete;
    ~Work() { release(); }
    Buf& operator[](Id i) { return buf[i]; }
    cudaError_t need(Buf& b, size_t bytes)
    {
        if (b.n >= bytes) return cudaSuccess;
        drop(b);
        const cudaError_t e = A.alloc ? A.alloc(A.user, &b.p, bytes) : cudaMalloc(&b.p, bytes);
        if (e != cudaSuccess) { b.p = nullptr; return e; }
        b.n = bytes; held += bytes;
        if (held > peak) peak = held;
        return cudaSuccess;
    }
    void drop(Buf& b)
    {
        if (b.p) { if (A.alloc) A.free(A.user, b.p, b.n); else cudaFree(b.p); held -= b.n; }
        b.p = nullptr; b.n = 0;
    }
    cudaError_t events()
    {
        for (cudaEvent_t& e : ev) if (!e) { const cudaError_t r = cudaEventCreate(&e); if (r != cudaSuccess) return r; }
        return cudaSuccess;
    }
    void release()
    {
        for (Buf& b : buf) drop(b);
        for (cudaEvent_t& e : ev) if (e) { cudaEventDestroy(e); e = nullptr; }
    }
};
template <class T> T* P(const Buf& b) { return static_cast<T*>(b.p); }

// A buffer from W's allocator for the length of the scope that declares it
struct TempBuf : Buf {
    Work& W;
    explicit TempBuf(Work& w) : W(w) {}
    TempBuf(const TempBuf&) = delete;
    TempBuf& operator=(const TempBuf&) = delete;
    ~TempBuf() { W.drop(*this); }
};

// ---- the maps of one triangulation, as the kernels see them ----
// The table in Work::tab: the maps, each map's (vertices << 32) | faces, the block -> map table.
struct TriBatch {
    struct Chunk { size_t first_block, blocks; unsigned first_map, n_maps; uint64_t pixels; bool filled; };
    std::vector<TriMap> maps;
    std::vector<unsigned> block_map;          // the map of every block, the chunks' blocks one after another
    std::vector<Chunk> chunks;
    uint64_t max_pixels = 0;
    bool faces = false, attributes = false, confs = false;     // some filled map wants them
    // m.n, m.px0 and m.block0 are set here
    void add(TriMap m)
    {
        const uint64_t n = (uint64_t)m.w * m.h;
        if (chunks.empty() || chunks.back().pixels + n > DM_CHUNK_PIXELS)
            chunks.push_back(Chunk{block_map.size(), 0, (unsigned)maps.size(), 0, 0, false});
        Chunk& c = chunks.back();
        m.n = (unsigned)n; m.px0 = (unsigned)c.pixels; m.block0 = (unsigned)c.blocks;
        const size_t nb = (size_t)((n + DM_BLOCK - 1) / DM_BLOCK);
        block_map.insert(block_map.end(), nb, (unsigned)(maps.size() - c.first_map));
        c.blocks += nb; c.pixels += n; c.n_maps += 1;
        max_pixels = std::max(max_pixels, c.pixels);
        if (m.filled) {
            c.filled = true;
            faces |= m.faces != nullptr;
            attributes |= m.normals || m.scales || m.confs;
            confs |= m.confs != nullptr;
        }
        maps.push_back(m);
    }
};
size_t tri_table_bytes(size_t n_maps, size_t blocks) { return n_maps * (sizeof(TriMap) + 8) + blocks * 4; }
const TriMap* tri_maps(Work& W) { return P<TriMap>(W[Work::tab]); }
unsigned long long* tri_totals(Work& W, const TriBatch& B) { return reinterpret_cast<unsigned long long*>(P<TriMap>(W[Work::tab]) + B.maps.size()); }
const unsigned* tri_block_map(Work& W, const TriBatch& B) { return reinterpret_cast<const unsigned*>(tri_totals(W, B) + B.maps.size()); }

// B's table into Work::tab on s
int tri_upload(Work& W, const TriBatch& B, cudaStream_t s)
{
    CK(W.need(W[Work::tab], tri_table_bytes(B.maps.size(), B.block_map.size())));
    CK(cudaMemcpyAsync(W[Work::tab].p, B.maps.data(), B.maps.size() * sizeof(TriMap), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(const_cast<unsigned*>(tri_block_map(W, B)), B.block_map.data(), B.block_map.size() * 4, cudaMemcpyHostToDevice, s));
    return 0;
}

// Chunk c's block codes, their counts and the exclusive scan of the counts, in Work::codes, counts and offsets
int tri_scan(Work& W, const TriBatch& B, const TriBatch::Chunk& c, float dd_factor, cudaStream_t s)
{
    const TriMap* maps = tri_maps(W) + c.first_map;
    const unsigned* bm = tri_block_map(W, B) + c.first_block;
    unsigned char* codes = P<unsigned char>(W[Work::codes]);
    unsigned long long *counts = P<unsigned long long>(W[Work::counts]), *offsets = P<unsigned long long>(W[Work::offsets]);
    const float dd_diag = (float)((double)dd_factor * 1.41421356237309504880);       // MATH_SQRT2, rounded like depthmap.cc:198
    const unsigned nb = (unsigned)c.blocks;
    k_tri_codes<<<nb, DM_BLOCK, 0, s>>>(maps, bm, dd_factor, dd_diag, codes);
    CK(cudaMemsetAsync(counts + c.pixels, 0, 8, s));
    k_tri_counts<<<nb, DM_BLOCK, 0, s>>>(maps, bm, codes, counts);
    size_t tmp_bytes = W[Work::tmp].n;
    CK(cub::DeviceScan::ExclusiveSum(W[Work::tmp].p, tmp_bytes, counts, offsets, (int)(c.pixels + 1), s));
    return 0;
}

// The count pass: every map's (vertices << 32) | faces into `totals`, read back with the one synchronisation of s
int tri_count(Work& W, const TriBatch& B, float dd_factor, cudaStream_t s, std::vector<uint64_t>& totals)
{
    for (const TriBatch::Chunk& c : B.chunks) {
        if (const int rc = tri_scan(W, B, c, dd_factor, s)) return rc;
        k_tri_totals<<<(c.n_maps + 255) / 256, 256, 0, s>>>(tri_maps(W) + c.first_map, c.n_maps, P<unsigned long long>(W[Work::offsets]),
                                                            tri_totals(W, B) + c.first_map);
    }
    CK(cudaGetLastError());
    totals.assign(B.maps.size(), 0);
    CK(cudaMemcpyAsync(totals.data(), tri_totals(W, B), totals.size() * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return 0;
}

// The fill pass after tri_count: the outputs of every filled map.  A batch of one chunk keeps the count pass's scan,
// a longer one scans each chunk again.  The confidence rings of a chunk's maps advance together.
int tri_fill(Work& W, const TriBatch& B, float dd_factor, int conf_iterations, float scale_factor, cudaStream_t s)
{
    const unsigned char* codes = P<unsigned char>(W[Work::codes]);
    const unsigned long long* offsets = P<unsigned long long>(W[Work::offsets]);
    for (const TriBatch::Chunk& c : B.chunks) {
        if (!c.filled) continue;
        if (B.chunks.size() > 1)
            if (const int rc = tri_scan(W, B, c, dd_factor, s)) return rc;
        const TriMap* maps = tri_maps(W) + c.first_map;
        const unsigned* bm = tri_block_map(W, B) + c.first_block;
        const unsigned nb = (unsigned)c.blocks;
        k_tri_clear<<<nb, DM_BLOCK, 0, s>>>(maps, bm);
        k_tri_vertices<<<nb, DM_BLOCK, 0, s>>>(maps, bm, codes, offsets);
        if (B.faces) k_tri_faces<<<nb, DM_BLOCK, 0, s>>>(maps, bm, codes, offsets);
        if (B.attributes) k_vertex_attributes<<<nb, DM_BLOCK, 0, s>>>(maps, bm, codes, scale_factor, B.confs ? P<unsigned>(W[Work::ring0]) : nullptr);
        if (B.confs) {
            // rings 1 .. conf_iterations - 1; every RING_CHECK rounds the host asks whether the last round still reached a
            // vertex, so a large conf_iterations costs as many launches as the meshes have rings, not conf_iterations
            constexpr int RING_CHECK = 16;
            unsigned *cur = P<unsigned>(W[Work::ring0]), *nxt = P<unsigned>(W[Work::ring1]), *last_hit = P<unsigned>(W[Work::last_hit]);
            CK(cudaMemsetAsync(last_hit, 0, 4, s));
            for (int d = 1; d < conf_iterations; ++d) {
                k_conf_ring<<<nb, DM_BLOCK, 0, s>>>(maps, bm, codes, cur, nxt, (unsigned)d, last_hit);
                std::swap(cur, nxt);
                if (d % RING_CHECK == 0) {
                    unsigned last = 0;
                    CK(cudaMemcpyAsync(&last, last_hit, 4, cudaMemcpyDeviceToHost, s));
                    CK(cudaStreamSynchronize(s));
                    if (last != (unsigned)d) break;
                }
            }
            k_conf_write<<<nb, DM_BLOCK, 0, s>>>(maps, bm, cur, conf_iterations);
        }
    }
    CK(cudaGetLastError());
    return 0;
}

struct ViewJob {
    const float* dm = nullptr;          // device depth map
    int w = 0, h = 0;
    InvProj P;
    float dd_factor = 5.0f;
    const float* ctw = nullptr;         // host 4x4 camera-to-world or NULL
    Color color;                        // device colour image or none
    bool want_colors = false;           // a colour image is given and colours are wanted
    bool want_faces = true, want_normals = false, want_scales = false;
    int conf_iterations = 0;
    float scale_factor = 0.f;
    uint64_t cap_v = ~0ull, cap_f = ~0ull;
    const b200mvs_pset_options* opt = nullptr;    // a point-set handle's view: the handle's options (its filters)
};

// The workspace of one view: which buffers of Work it needs and their sizes in bytes, for a map of J.w x J.h pixels of
// which `points` are vertices.  Only the pixel map of -C depends on the points, which are known after the kernels' scan.
// Each buffer comes with the step that reserves it: the fill fraction of -f before the kernels, run_view's buffers before
// its clock starts (cudaMalloc synchronises), the filters of a handle's view after the kernels.  workspace_bytes sums the
// same list with a vertex per pixel, so the bytes a reconstruction keeps free for a handle and the bytes the handle
// takes cannot drift apart.
enum Step { FILL, KERNELS, FILTERS };
template <class F> void for_each_view_buffer(const ViewJob& J, uint64_t points, F&& f)
{
    const b200mvs_pset_options* o = J.opt;
    const size_t n = (size_t)J.w * J.h;
    if (o && o->min_valid_fraction > 0.0f) f(FILL, Work::fill, 8 * 8 + 4);                 // eight lanes and the fraction
    size_t scan = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)(n + 1));
    f(KERNELS, Work::codes, n); f(KERNELS, Work::counts, (n + 1) * 8); f(KERNELS, Work::offsets, (n + 1) * 8);
    f(KERNELS, Work::vids, n * 4); f(KERNELS, Work::tmp, scan);
    f(KERNELS, Work::tab, tri_table_bytes(1, (n + DM_BLOCK - 1) / DM_BLOCK));
    // worst-case sized outputs: a vertex per pixel, two faces per block
    const size_t max_f = 2 * (size_t)(J.w - 1) * (J.h - 1);
    const bool conf = J.conf_iterations > 0;
    f(KERNELS, Work::verts, n * 12);
    if (J.want_colors) f(KERNELS, Work::colors, n * 16);
    if (J.want_faces) f(KERNELS, Work::faces, (max_f ? max_f : 1) * 12);
    if (J.want_normals) f(KERNELS, Work::normals, n * 12);
    if (J.want_scales) f(KERNELS, Work::scales, n * 4);
    if (conf) { f(KERNELS, Work::confs, n * 4); f(KERNELS, Work::ring0, n * 4); f(KERNELS, Work::ring1, n * 4); f(KERNELS, Work::last_hit, 4); }
    if (o && o->correspondence) f(FILTERS, Work::pix, std::max<uint64_t>(points, 1) * 8);
    if (o && o->use_aabb) {
        // box flags, their scan, the kept attributes
        size_t flag_scan = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, flag_scan, (unsigned*)nullptr, (unsigned*)nullptr, (int)(n + 1));
        f(FILTERS, Work::flags, (n + 1) * 4); f(FILTERS, Work::pos, (n + 1) * 4); f(FILTERS, Work::scan_tmp, flag_scan);
        f(FILTERS, Work::o_verts, n * 12);
        if (J.want_normals) f(FILTERS, Work::o_normals, n * 12);
        if (J.want_colors) f(FILTERS, Work::o_colors, n * 16);
        if (J.want_scales) f(FILTERS, Work::o_scales, n * 4);
        if (conf) f(FILTERS, Work::o_confs, n * 4);
    }
}
cudaError_t reserve_view(Work& W, Step step, const ViewJob& J, uint64_t points)
{
    cudaError_t e = cudaSuccess;
    for_each_view_buffer(J, points, [&](Step s, Work::Id b, size_t bytes) { if (s == step && e == cudaSuccess) e = W.need(W[b], bytes); });
    return e;
}

// A host depth map and colour image (NULL: none) into the workspace; returns the colour as run_view reads it
int upload(Work& W, const float* depth, const uint8_t* color, int cch, int w, int h, Color* col)
{
    const size_t n = (size_t)w * h;
    CK(W.need(W[Work::dm], n * 4));
    CK(cudaMemcpy(W[Work::dm].p, depth, n * 4, cudaMemcpyHostToDevice));
    *col = Color{};
    if (color) {
        CK(W.need(W[Work::color], n * cch));
        CK(cudaMemcpy(W[Work::color].p, color, n * cch, cudaMemcpyHostToDevice));
        *col = Color{P<uint8_t>(W[Work::color]), cch, cch, w};
    }
    return 0;
}

// The kernels of b200mvs_depthmap_pointset on one device map, a batch of one, between events ev[0] and ev[1] (not
// synchronised).  Results stay in W: vids, verts, colors, faces, normals, confs, scales.
int run_view(Work& W, const ViewJob& J, uint64_t* nv_out, uint64_t* nf_out)
{
    CK(reserve_view(W, KERNELS, J, (size_t)J.w * J.h));
    CK(W.events());
    TriMap m = {};
    m.dm = J.dm; m.w = (unsigned)J.w; m.h = (unsigned)J.h; m.filled = 1; m.P = J.P;
    m.has_ctw = J.ctw != nullptr;
    if (J.ctw) std::memcpy(m.ctw, J.ctw, sizeof(m.ctw));
    m.color = J.color;
    m.vids = P<unsigned>(W[Work::vids]); m.verts = P<float>(W[Work::verts]);
    m.colors = J.want_colors ? P<float>(W[Work::colors]) : nullptr;
    m.faces = J.want_faces ? P<unsigned>(W[Work::faces]) : nullptr;
    m.normals = J.want_normals ? P<float>(W[Work::normals]) : nullptr;
    m.scales = J.want_scales ? P<float>(W[Work::scales]) : nullptr;
    m.confs = J.conf_iterations > 0 ? P<float>(W[Work::confs]) : nullptr;
    TriBatch B;
    B.add(m);
    const cudaStream_t s = cudaStreamLegacy;
    if (const int rc = tri_upload(W, B, s)) return rc;
    CK(cudaEventRecord(W.ev[0], s));
    std::vector<uint64_t> totals;
    if (const int rc = tri_count(W, B, J.dd_factor, s, totals)) return rc;
    const uint64_t nv = totals[0] >> 32, nf = totals[0] & 0xFFFFFFFFull;
    *nv_out = nv; *nf_out = nf;
    if (nv > J.cap_v || nf > J.cap_f) return fail(B200MVS_ERR_OVERFLOW, "depthmap_triangulate: output capacity too small");
    if (const int rc = tri_fill(W, B, J.dd_factor, J.conf_iterations, J.scale_factor, s)) return rc;
    CK(cudaEventRecord(W.ev[1], s));
    return 0;
}

// ---- scene-level filters of scene2pset ----

// Fill fraction (scene2pset.cc:284-291).  The reference build vectorises `num_recon += 1.0f` over eight float lanes
// (element j feeds lane j % 8 up to the last multiple of 8), each lane saturating at 2^24, then reduces the lanes as
// ((a0+a4) + (a2+a6)) + ((a1+a5) + (a3+a7)).  A remainder of 4 or more goes through one 4-lane step c_k = b_k + (a_k +
// a_k+4), reduced as (c0+c2) + (c1+c3), and the last 0-3 elements add 1.0f one by one.  k_fill_lanes counts the lanes
// exactly; k_fill_fraction replays the float sums in that order.
__global__ void k_fill_lanes(const float* __restrict__ dm, size_t n8, unsigned long long* __restrict__ lanes)
{
    __shared__ unsigned long long s[8];
    if (threadIdx.x < 8) s[threadIdx.x] = 0ull;
    __syncthreads();
    // the grid stride is a multiple of 8, so each thread stays on the lane of its first element
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    unsigned long long c = 0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride) c += dm[i] > 0.0f;
    if (c) atomicAdd(&s[threadIdx.x & 7], c);
    __syncthreads();
    if (threadIdx.x < 8 && s[threadIdx.x]) atomicAdd(&lanes[threadIdx.x], s[threadIdx.x]);
}
__global__ void k_fill_fraction(const float* __restrict__ dm, size_t n, const unsigned long long* __restrict__ lanes, float* __restrict__ out)
{
    const size_t n8 = n & ~(size_t)7;
    float a[8];
    for (int k = 0; k < 8; ++k) a[k] = (float)(lanes[k] < (1ull << 24) ? lanes[k] : (1ull << 24));
    float v[4];
    for (int k = 0; k < 4; ++k) v[k] = __fadd_rn(a[k], a[k + 4]);
    size_t j = n8;
    float sum;
    if (n - n8 >= 4) {
        float c[4];
        for (int k = 0; k < 4; ++k) c[k] = __fadd_rn(dm[n8 + k] > 0.0f ? 1.0f : 0.0f, v[k]);
        sum = __fadd_rn(__fadd_rn(c[0], c[2]), __fadd_rn(c[1], c[3]));
        j += 4;
    } else {
        sum = __fadd_rn(__fadd_rn(v[0], v[2]), __fadd_rn(v[1], v[3]));
    }
    for (; j < n; ++j) if (dm[j] > 0.0f) sum = __fadd_rn(sum, 1.0f);
    *out = __fdiv_rn(sum, (float)(long long)n);      // num_total = static_cast<float>(value amount)
}

// normal *= confidence (scene2pset.cc:120-128, -p)
__global__ void k_poisson(float* __restrict__ normals, const float* __restrict__ confs, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float c = confs[i];
    for (int k = 0; k < 3; ++k) normals[3 * i + k] = __fmul_rn(normals[3 * i + k], c);
}
// math::geom::point_box_overlap (octree_tools.h:356-364): outside when p < min or p > max on an axis (NaN is inside)
__global__ void k_aabb_flags(const float* __restrict__ verts, size_t n, float3 lo, float3 hi, unsigned* __restrict__ flags)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = verts[3 * i], y = verts[3 * i + 1], z = verts[3 * i + 2];
    const bool out = x < lo.x || x > hi.x || y < lo.y || y > hi.y || z < lo.z || z > hi.z;
    flags[i] = out ? 0u : 1u;
}
// stream compaction of every attribute array by the exclusive scan of the box flags
__global__ void k_compact(const unsigned* __restrict__ flags, const unsigned* __restrict__ pos, size_t n,
                          const float* __restrict__ v, const float* __restrict__ nr, const float* __restrict__ co,
                          const float* __restrict__ sc, const float* __restrict__ cf,
                          float* __restrict__ ov, float* __restrict__ onr, float* __restrict__ oco, float* __restrict__ osc, float* __restrict__ ocf)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !flags[i]) return;
    const size_t j = pos[i];
    for (int k = 0; k < 3; ++k) ov[3 * j + k] = v[3 * i + k];
    if (nr) for (int k = 0; k < 3; ++k) onr[3 * j + k] = nr[3 * i + k];
    if (co) for (int k = 0; k < 4; ++k) oco[4 * j + k] = co[4 * i + k];
    if (sc) osc[j] = sc[i];
    if (cf) ocf[j] = cf[i];
}
// the inverse of the vertex-id image: pixel (x, y) of every vertex (scene2pset.cc:64-83)
__global__ void k_vertex_pixels(const unsigned* __restrict__ vids, int w, size_t n, unsigned* __restrict__ xy)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned v = vids[i];
    if (v == 0xFFFFFFFFu) return;
    xy[2 * (size_t)v] = (unsigned)(i % (size_t)w);
    xy[2 * (size_t)v + 1] = (unsigned)(i / (size_t)w);
}

// Mask projection (scene2pset.cc:434-457) in the reference build's own arithmetic:
//   c_r = fma(z, W[r][2], fma(x, W[r][0], y * W[r][1])) + W[r][3]          (Matrix4f::mult(v, 1), contracted)
//   p0 = fma(c2, K2, fma(K0, c0, c1 * K1)), p1 = fma(c2, K5, fma(K3, c0, c1 * K4)), p2 = fma(c2, K8, fma(c0, K6, c1 * K7))
//   x = p0 / p2, y = p1 / p2 (true divisions); outside when x < 0 || y < 0 || x >= w || y >= h.
// Row y of a mask starts at mask + y * pitch, in the block the host masks are uploaded to or in the caller's device memory.
struct MaskCam { float W[12]; float K[9]; int w, h; const unsigned char* mask; long long pitch; };
__global__ void k_mask_clip(const float* __restrict__ verts, size_t n, const MaskCam* __restrict__ cams, int n_masks,
                            unsigned char* __restrict__ del)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = verts[3 * i], y = verts[3 * i + 1], z = verts[3 * i + 2];
    unsigned char d = 0;
    for (int m = 0; m < n_masks && !d; ++m) {
        const MaskCam& C = cams[m];
        float c[3];
        for (int r = 0; r < 3; ++r)
            c[r] = __fadd_rn(__fmaf_rn(z, C.W[4 * r + 2], __fmaf_rn(x, C.W[4 * r], __fmul_rn(y, C.W[4 * r + 1]))), C.W[4 * r + 3]);
        const float p0 = __fmaf_rn(c[2], C.K[2], __fmaf_rn(C.K[0], c[0], __fmul_rn(c[1], C.K[1])));
        const float p1 = __fmaf_rn(c[2], C.K[5], __fmaf_rn(C.K[3], c[0], __fmul_rn(c[1], C.K[4])));
        const float p2 = __fmaf_rn(c[2], C.K[8], __fmaf_rn(c[0], C.K[6], __fmul_rn(c[1], C.K[7])));
        const float px = __fdiv_rn(p0, p2), py = __fdiv_rn(p1, p2);
        if (px < 0.0f || py < 0.0f || px >= (float)C.w || py >= (float)C.h) continue;
        if (isnan(px) || isnan(py)) continue;       // the reference would index its mask at INT_MIN
        if (C.mask[(int)py * C.pitch + (int)px] == 0) d = 1;
    }
    del[i] = d;
}
// One list of a device-resident set after the mask clip, stable: entry i moves to i - (points deleted before i)
__global__ void k_clip_compact(const unsigned char* __restrict__ del, const unsigned long long* __restrict__ deleted_before, uint64_t n,
                               int per, const float* __restrict__ src, float* __restrict__ dst)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || del[i]) return;
    const uint64_t j = i - deleted_before[i];
    for (int k = 0; k < per; ++k) dst[j * per + k] = src[i * per + k];
}

// CameraInfo::fill_cam_to_world (camera.cc:82-94) with the reference build's arithmetic: the translation column is
// -fma(r6, t2, fma(r0, t0, r3 * t1)) etc.
void cam_to_world(const b200mvs_pset_camera& c, float* m)
{
    const float* r = c.rot;
    const float* t = c.trans;
    const float M[16] = {r[0], r[3], r[6], -std::fmaf(r[6], t[2], std::fmaf(r[0], t[0], r[3] * t[1])),
                         r[1], r[4], r[7], -std::fmaf(r[7], t[2], std::fmaf(r[1], t[0], r[4] * t[1])),
                         r[2], r[5], r[8], -std::fmaf(r[8], t[2], std::fmaf(r[2], t[0], r[5] * t[1])),
                         0.f, 0.f, 0.f, 1.f};
    std::memcpy(m, M, sizeof(M));
}

} // namespace

struct b200mvs_pset {
    int device = 0;
    b200mvs_pset_options opt;
    Work W;                                                      // W.held / W.peak also count the lists of a device set
    b200mvs_pset_dev::Lists set;
    std::vector<b200mvs_pset_corr_view> corr;
    uint64_t n_views = 0;
    bool clipped = false;
    double ms_pointset = 0, ms_filter = 0, ms_mask = 0;
};

namespace {

using b200mvs_pset_dev::Block;
using b200mvs_pset_dev::Lists;

// Memory for the lists of the set and their scratch copies.  A device set's is the caller's memory, like the buffers of
// b200mvs_reconstruct_device: plain cudaMalloc, never a context's accounted allocator, counted in the handle's device
// bytes.  A host set's is pageable host memory; pinning it would count against the process' locked memory.
cudaError_t store_alloc(b200mvs_pset* ps, void** p, size_t bytes)
{
    if (!ps->set.on_device) return (*p = std::malloc(bytes)) ? cudaSuccess : cudaErrorMemoryAllocation;
    if (const cudaError_t e = cudaMalloc(p, bytes)) return e;
    ps->W.held += bytes;
    ps->W.peak = std::max(ps->W.peak, ps->W.held);
    return cudaSuccess;
}
void store_free(b200mvs_pset* ps, void* p, size_t bytes)
{
    if (!p) return;
    if (!ps->set.on_device) { std::free(p); return; }
    cudaFree(p);
    ps->W.held -= bytes;
}
// A copy within the set's memory, or out of it into the caller's host memory.  A host set's are host to host, which
// cudaMemcpy does well below the speed of memcpy.
// Scratch memory of the set's store for the length of the scope that declares it
struct StoreTemp {
    b200mvs_pset* ps;
    void* p = nullptr;
    size_t bytes;
    StoreTemp(b200mvs_pset* ps, size_t bytes) : ps(ps), bytes(bytes) {}
    StoreTemp(const StoreTemp&) = delete;
    StoreTemp& operator=(const StoreTemp&) = delete;
    ~StoreTemp() { store_free(ps, p, bytes); }
    cudaError_t alloc() { return store_alloc(ps, &p, bytes); }
};
cudaError_t store_copy(const b200mvs_pset* ps, void* dst, const void* src, size_t bytes)
{
    if (ps->set.on_device) return cudaMemcpy(dst, src, bytes, cudaMemcpyDefault);
    std::memcpy(dst, src, bytes);
    return cudaSuccess;
}

// Room for `entries` entries in list k: the capacity at least doubles and the entries so far are copied over
cudaError_t reserve(b200mvs_pset* ps, int k, uint64_t entries)
{
    Lists& S = ps->set;
    if (entries <= S.cap[k]) return cudaSuccess;
    const size_t item = 4 * (size_t)Lists::PER[k];
    const uint64_t cap = std::max<uint64_t>({entries, 2 * S.cap[k], (uint64_t)1 << 14});
    void* p = nullptr;
    cudaError_t e = store_alloc(ps, &p, cap * item);
    if (e != cudaSuccess) return e;
    const uint64_t used = S.n[k] + S.staged[k];
    if (used) e = store_copy(ps, p, S.p[k], used * item);
    if (e != cudaSuccess) { store_free(ps, p, cap * item); return e; }
    store_free(ps, S.p[k], S.cap[k] * item);
    S.p[k] = p; S.cap[k] = cap;
    return cudaSuccess;
}

// The per-view kernels of a handle's view (scene2pset.cc:316-358): no faces, the vertices in world coordinates (`ctw`),
// colours when the view has a colour image
ViewJob pset_job(const b200mvs_pset_options& o, int w, int h, const float* ctw, bool colors)
{
    ViewJob J;
    J.w = w; J.h = h; J.dd_factor = o.dd_factor; J.ctw = ctw; J.want_colors = colors;
    J.want_faces = false; J.want_normals = o.with_normals != 0; J.want_scales = o.with_scale != 0; J.scale_factor = o.scale_factor;
    J.conf_iterations = o.with_conf ? o.conf_iterations : 0;
    J.opt = &o;
    return J;
}

// The per-view work of scene2pset (scene2pset.cc:284-399) on a depth map in device memory: the fill fraction of -f, the
// per-view kernels, the bounding box, -p and the pixel map of -C.  The surviving points are staged behind the entries of
// the handle's set; `res` receives the view's record except first_index, ms_view / ms_filt the device times.
int add_device_view(b200mvs_pset* ps, const float* dm, int w, int h, const Color& color, const b200mvs_pset_camera& cam,
                    b200mvs_pset_view& res, float& ms_view, float& ms_filt)
{
    const b200mvs_pset_options& o = ps->opt;
    Work& W = ps->W;
    const size_t n = (size_t)w * h;
    float ctw[16];
    cam_to_world(cam, ctw);
    ViewJob J = pset_job(o, w, h, ctw, color.p != nullptr);
    J.dm = dm; J.color = color;
    fill_calibration(cam.flen, cam.paspect, cam.ppoint[0], cam.ppoint[1], (float)w, (float)h, nullptr, J.P.m);
    CK(W.events());
    ms_view = ms_filt = 0.f;
    if (o.min_valid_fraction > 0.0f) {
        CK(reserve_view(W, FILL, J, n));
        CK(cudaMemsetAsync(W[Work::fill].p, 0, 8 * 8));
        CK(cudaEventRecord(W.ev[2]));
        const size_t n8 = n & ~(size_t)7;
        if (n8) k_fill_lanes<<<(unsigned)std::min<size_t>((n8 + 255) / 256, 1024), 256>>>(dm, n8, P<unsigned long long>(W[Work::fill]));
        k_fill_fraction<<<1, 1>>>(dm, n, P<unsigned long long>(W[Work::fill]), reinterpret_cast<float*>(P<unsigned long long>(W[Work::fill]) + 8));
        CK(cudaEventRecord(W.ev[3]));
        CK(cudaGetLastError());
        CK(cudaMemcpy(&res.fraction, P<unsigned long long>(W[Work::fill]) + 8, 4, cudaMemcpyDeviceToHost));
        cudaEventElapsedTime(&ms_filt, W.ev[2], W.ev[3]);
        if (res.fraction < o.min_valid_fraction) return 0;                                             // scene2pset.cc:292-298
    }
    uint64_t nv = 0, nf = 0;
    const int rc = run_view(W, J, &nv, &nf);
    if (rc) return rc;
    CK(reserve_view(W, FILTERS, J, nv));
    const unsigned nb = (unsigned)((std::max<uint64_t>(nv, 1) + 255) / 256);
    const bool conf = J.conf_iterations > 0;
    float *v = P<float>(W[Work::verts]), *nr = J.want_normals ? P<float>(W[Work::normals]) : nullptr, *co = J.want_colors ? P<float>(W[Work::colors]) : nullptr;
    float *sc = J.want_scales ? P<float>(W[Work::scales]) : nullptr, *cf = conf ? P<float>(W[Work::confs]) : nullptr;
    uint64_t kept = nv;
    CK(cudaEventRecord(W.ev[2]));
    if (o.poisson_normals && nv) k_poisson<<<nb, 256>>>(nr, cf, nv);
    if (o.correspondence) k_vertex_pixels<<<(unsigned)((n + 255) / 256), 256>>>(P<unsigned>(W[Work::vids]), w, n, P<unsigned>(W[Work::pix]));
    if (o.use_aabb && nv) {
        CK(cudaMemsetAsync(P<unsigned>(W[Work::flags]) + nv, 0, 4));
        k_aabb_flags<<<nb, 256>>>(v, nv, make_float3(o.aabb_min[0], o.aabb_min[1], o.aabb_min[2]),
                                  make_float3(o.aabb_max[0], o.aabb_max[1], o.aabb_max[2]), P<unsigned>(W[Work::flags]));
        size_t scan_bytes = W[Work::scan_tmp].n;
        CK(cub::DeviceScan::ExclusiveSum(W[Work::scan_tmp].p, scan_bytes, P<unsigned>(W[Work::flags]), P<unsigned>(W[Work::pos]), (int)(nv + 1)));
        k_compact<<<nb, 256>>>(P<unsigned>(W[Work::flags]), P<unsigned>(W[Work::pos]), nv, v, nr, co, sc, cf, P<float>(W[Work::o_verts]),
                               nr ? P<float>(W[Work::o_normals]) : nullptr, co ? P<float>(W[Work::o_colors]) : nullptr, sc ? P<float>(W[Work::o_scales]) : nullptr,
                               cf ? P<float>(W[Work::o_confs]) : nullptr);
        unsigned k = 0;
        CK(cudaMemcpy(&k, P<unsigned>(W[Work::pos]) + nv, 4, cudaMemcpyDeviceToHost));
        kept = k;
        v = P<float>(W[Work::o_verts]); nr = nr ? P<float>(W[Work::o_normals]) : nullptr; co = co ? P<float>(W[Work::o_colors]) : nullptr;
        sc = sc ? P<float>(W[Work::o_scales]) : nullptr; cf = cf ? P<float>(W[Work::o_confs]) : nullptr;
    }
    CK(cudaEventRecord(W.ev[3]));
    CK(cudaGetLastError());
    CK(cudaEventSynchronize(W.ev[3]));
    float ms_kept = 0.f;
    cudaEventElapsedTime(&ms_view, W.ev[0], W.ev[1]);
    cudaEventElapsedTime(&ms_kept, W.ev[2], W.ev[3]);
    ms_filt += ms_kept;
    // append to the point set (scene2pset.cc:360-399), colours only from a view that has them: list k staged behind its
    // committed and staged entries
    Lists& S = ps->set;
    auto append = [&](int k, const void* src) -> cudaError_t {
        const uint64_t at = S.n[k] + S.staged[k];
        const size_t item = 4 * (size_t)Lists::PER[k];
        if (const cudaError_t e = reserve(ps, k, at + kept)) return e;
        S.staged[k] += kept;
        return kept ? cudaMemcpyAsync(static_cast<char*>(S.p[k]) + at * item, src, kept * item, cudaMemcpyDefault, cudaStreamLegacy) : cudaSuccess;
    };
    CK(append(Lists::VERTS, v));
    if (nr) CK(append(Lists::NORMALS, nr));
    if (co) CK(append(Lists::COLORS, co));
    if (sc) CK(append(Lists::VALUES, sc));
    if (cf) CK(append(Lists::CONFS, cf));
    if (o.correspondence) CK(append(Lists::PIX, W[Work::pix].p));
    // the workspace is the next view's, and the maps of a reconstruction are the next group's: the copies end here
    CK(cudaStreamSynchronize(cudaStreamLegacy));
    res.added = 1;
    res.n_points = kept;
    return 0;
}

// The correspondence record of an added view whose pixels start at pixel pair `first` (scene2pset.cc:50-56)
void add_corr(b200mvs_pset* ps, int view_id, int w, int h, size_t first)
{
    if (ps->opt.correspondence) ps->corr.push_back(b200mvs_pset_corr_view{(uint32_t)view_id, (uint32_t)w, (uint32_t)h, (uint64_t)first});
}

// The arguments of b200mvs_pset_add_view and b200mvs_pset_add_view_device (`fn`) other than where the buffers live
int check_add_view(const char* fn, const b200mvs_pset* ps, const float* depth, int w, int h, const uint8_t* color, int color_channels,
                   const b200mvs_pset_camera* cam)
{
    if (!ps || !cam) return fail(B200MVS_ERR_INVALID_ARG, "%s: null handle or camera", fn);
    if (!depth) return fail(B200MVS_ERR_INVALID_ARG, "Null depthmap given");
    if (cam->flen == 0.0f) return fail(B200MVS_ERR_INVALID_ARG, "Invalid camera given");                 // depthmap.cc:383-384
    if (w < 2 || h < 2 || (size_t)w * h >= 0xFFFFFFFFull) return fail(B200MVS_ERR_INVALID_ARG, "%s: depth map size", fn);
    if (color && (color_channels < 1 || color_channels > 4)) return fail(B200MVS_ERR_INVALID_ARG, "Color image dimension mismatch");
    if (ps->clipped) return fail(B200MVS_ERR_INVALID_ARG, "%s: the masks have been applied already", fn);
    return 0;
}

// One view of b200mvs_pset_add_view / _device from a depth map and colour image in device memory: appended to the handle
int add_view(b200mvs_pset* ps, int view_id, const float* dm, int w, int h, const Color& col, const b200mvs_pset_camera& cam,
             b200mvs_pset_view* out)
{
    Lists& S = ps->set;
    b200mvs_pset_view res = {0, 0.f, 0, S.n[Lists::VERTS]};
    const uint64_t pix_at = S.n[Lists::PIX];
    float ms_view = 0.f, ms_filt = 0.f;
    const int rc = add_device_view(ps, dm, w, h, col, cam, res, ms_view, ms_filt);
    ps->ms_pointset += ms_view;
    ps->ms_filter += ms_filt;
    for (int k = 0; k < Lists::N_LISTS; ++k) {
        if (!rc) S.n[k] += S.staged[k];
        S.staged[k] = 0;
    }
    if (rc) return rc;
    if (res.added) { add_corr(ps, view_id, w, h, pix_at); ps->n_views += 1; }
    if (out) *out = res;
    return 0;
}

// The views were staged in the order their groups ran: a list whose segments are not in block order is put in order
// through a scratch copy of its staged entries
int order_staged(b200mvs_pset* ps, const std::vector<Block>& blocks)
{
    Lists& S = ps->set;
    for (int k = 0; k < Lists::N_LISTS; ++k) {
        uint64_t at = S.n[k];
        bool in_order = true;
        for (const Block& b : blocks) {
            if (!b.count[k]) continue;
            in_order = in_order && b.at[k] == at;
            at += b.count[k];
        }
        if (in_order) continue;
        const size_t item = 4 * (size_t)Lists::PER[k], bytes = S.staged[k] * item;
        char* base = static_cast<char*>(S.p[k]);
        StoreTemp tmp(ps, bytes);
        CK(tmp.alloc());
        uint64_t o = 0;
        for (const Block& b : blocks) {
            if (b.count[k]) CK(store_copy(ps, static_cast<char*>(tmp.p) + o * item, base + b.at[k] * item, b.count[k] * item));
            o += b.count[k];
        }
        CK(store_copy(ps, base + S.n[k] * item, tmp.p, o * item));
        CK(cudaStreamSynchronize(cudaStreamLegacy));
    }
    return 0;
}

// ---- the maps of one confidence_clean / cleanup call, as the kernels see them ----
// Cleanup takes the maps in chunks (DM_CHUNK_PIXELS), its union-find workspace (8 B per label) sized to the largest chunk.
// Confidence_clean needs no labels: its batch is one launch.
struct DmBatch {
    struct Chunk { size_t first_block, blocks; uint64_t labels; };
    std::vector<DmMap> maps;
    std::vector<unsigned> block_map;          // the map of every block, the chunks' blocks one after another
    std::vector<Chunk> chunks;
    uint64_t max_labels = 0;
    bool chunked;
    explicit DmBatch(bool chunked_) : chunked(chunked_) {}
    // w * h <= 0xFFFFFFF0
    void add(const float* dm, float* out, const float* cm, unsigned w, unsigned h, unsigned long long thres)
    {
        const uint64_t n = (uint64_t)w * h;
        if (chunks.empty() || (chunked && chunks.back().labels + n > DM_CHUNK_PIXELS)) chunks.push_back(Chunk{block_map.size(), 0, 0});
        Chunk& c = chunks.back();
        maps.push_back(DmMap{dm, out, cm, thres, w, h, (unsigned)n, chunked ? (unsigned)c.labels : 0u, (unsigned)c.blocks});
        const size_t nb = (size_t)((n + DM_BLOCK - 1) / DM_BLOCK);
        block_map.insert(block_map.end(), nb, (unsigned)(maps.size() - 1));
        c.blocks += nb;
        c.labels += n;
        max_labels = std::max(max_labels, c.labels);
    }
};

// Runs the batch on stream s: its tables in `tab`, cleanup's union-find workspace (uf != NULL) in `uf`.  Returns when the
// work is enqueued.
int dm_run(Work& W, const DmBatch& B, Buf& tab, Buf* uf, cudaStream_t s)
{
    const size_t map_bytes = B.maps.size() * sizeof(DmMap), table_bytes = B.block_map.size() * sizeof(unsigned);
    for (const DmBatch::Chunk& c : B.chunks)
        if (c.blocks > 0x7FFFFFFFull) return fail(B200MVS_ERR_INVALID_ARG, "depth maps: more pixels than one launch covers");
    CK(W.need(tab, map_bytes + table_bytes));
    const DmMap* maps = P<DmMap>(tab);
    unsigned* block_map = reinterpret_cast<unsigned*>(static_cast<char*>(tab.p) + map_bytes);
    CK(cudaMemcpyAsync(tab.p, B.maps.data(), map_bytes, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(block_map, B.block_map.data(), table_bytes, cudaMemcpyHostToDevice, s));
    if (!uf) {
        k_conf_clean<<<(unsigned)B.chunks[0].blocks, DM_BLOCK, 0, s>>>(maps, block_map);
        CK(cudaGetLastError());
        return 0;
    }
    CK(W.need(*uf, B.max_labels * 8));
    unsigned *parent = P<unsigned>(*uf), *count = parent + B.max_labels;
    for (const DmBatch::Chunk& c : B.chunks) {
        const unsigned nb = (unsigned)c.blocks;
        const unsigned* bm = block_map + c.first_block;
        k_cc_init<<<(unsigned)((c.labels + 255) / 256), 256, 0, s>>>(parent, count, c.labels);
        k_cc_link<<<nb, DM_BLOCK, 0, s>>>(maps, bm, parent);
        k_cc_count<<<nb, DM_BLOCK, 0, s>>>(maps, bm, parent, count);
        k_cc_erase<<<nb, DM_BLOCK, 0, s>>>(maps, bm, parent, count);
    }
    CK(cudaGetLastError());
    return 0;
}

// A byte range of the caller's buffers that a *_device call writes or reads: its map and its name for a message
struct Range { uintptr_t a, b; int map; std::string name; };
// 0 when no written range overlaps another written range or a read range, else B200MVS_ERR_INVALID_ARG naming both.
// in_place: a written range may start where a read range of its own map does (cleanup's out_dev[j] == depth_dev[j]).
// Empty ranges overlap nothing.
int check_overlaps(const char* fn, std::vector<Range> wr, const std::vector<Range>& rd, bool in_place)
{
    // sort the written ranges, which must be disjoint, then find for each read range the written range that starts last
    // before it ends, the only one that can overlap it
    wr.erase(std::remove_if(wr.begin(), wr.end(), [](const Range& r) { return r.a == r.b; }), wr.end());
    std::sort(wr.begin(), wr.end(), [](const Range& x, const Range& y) { return x.a != y.a ? x.a < y.a : x.map < y.map; });
    const auto overlap = [&](const Range& w, const Range& r) {
        return fail(B200MVS_ERR_INVALID_ARG, "%s: %s overlaps %s", fn, w.name.c_str(), r.name.c_str());
    };
    for (size_t k = 1; k < wr.size(); ++k)
        if (wr[k].a < wr[k - 1].b) return wr[k].map < wr[k - 1].map ? overlap(wr[k], wr[k - 1]) : overlap(wr[k - 1], wr[k]);
    for (const Range& r : rd) {
        if (r.a == r.b) continue;
        const auto it = std::partition_point(wr.begin(), wr.end(), [&](const Range& w) { return w.a < r.b; });
        if (it == wr.begin()) continue;
        const Range& w = *(it - 1);
        if (w.b <= r.a || (in_place && w.map == r.map && w.a == r.a)) continue;
        return overlap(w, r);
    }
    return 0;
}

// The arguments of b200mvs_depthmap_confidence_clean_device (depth is written, conf read) and of _cleanup_device (`cleanup`:
// depth is read, out written), checked in full before anything is launched or written, and the batch they describe.  An
// empty batch is not looked at further.
int dm_device_batch(const char* fn, bool cleanup, int device, int n_maps, const float* const* depth, const float* const* conf,
                    const int32_t* widths, const int32_t* heights, const int64_t* thres, float* const* out, DmBatch& B)
{
    if (n_maps < 0) return fail(B200MVS_ERR_INVALID_ARG, "%s: n_maps is %d, must not be negative", fn, n_maps);
    if (n_maps == 0) return 0;
    const char* dname = "depth_dev";
    const char* other = cleanup ? "out_dev" : "conf_dev";
    if (!depth) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s is NULL", fn, dname);
    if (cleanup ? !out : !conf) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s is NULL", fn, other);
    if (!widths) return fail(B200MVS_ERR_INVALID_ARG, "%s: widths is NULL", fn);
    if (!heights) return fail(B200MVS_ERR_INVALID_ARG, "%s: heights is NULL", fn);
    if (cleanup && !thres) return fail(B200MVS_ERR_INVALID_ARG, "%s: thres is NULL", fn);
    for (int j = 0; j < n_maps; ++j) {
        const void* second = cleanup ? static_cast<const void*>(out[j]) : static_cast<const void*>(conf[j]);
        if (!depth[j]) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s[%d] is NULL", fn, dname, j);
        if (!second) return fail(B200MVS_ERR_INVALID_ARG, "%s: %s[%d] is NULL", fn, other, j);
        if (widths[j] < 1) return fail(B200MVS_ERR_INVALID_ARG, "%s: widths[%d] is %d, must be at least 1", fn, j, widths[j]);
        if (heights[j] < 1) return fail(B200MVS_ERR_INVALID_ARG, "%s: heights[%d] is %d, must be at least 1", fn, j, heights[j]);
        const uint64_t n = (uint64_t)widths[j] * heights[j];
        if (n > 0xFFFFFFF0ull)
            return fail(B200MVS_ERR_INVALID_ARG, "%s: map %d has %llu pixels (widths[%d] x heights[%d]), more than 4294967280", fn, j,
                        (unsigned long long)n, j, j);
    }
    std::vector<Range> wr, rd;
    for (int j = 0; j < n_maps; ++j) {
        const uintptr_t bytes = (uintptr_t)widths[j] * heights[j] * 4;
        const uintptr_t d = reinterpret_cast<uintptr_t>(depth[j]);
        const uintptr_t o = cleanup ? reinterpret_cast<uintptr_t>(out[j]) : reinterpret_cast<uintptr_t>(conf[j]);
        const std::string idx = "[" + std::to_string(j) + "]";
        (cleanup ? rd : wr).push_back(Range{d, d + bytes, j, dname + idx});
        (cleanup ? wr : rd).push_back(Range{o, o + bytes, j, other + idx});
    }
    if (const int rc = check_overlaps(fn, std::move(wr), rd, cleanup)) return rc;       // out_dev[j] == depth_dev[j]: in place
    CK(cudaSetDevice(device));
    for (int j = 0; j < n_maps; ++j) {
        const std::string idx = "[" + std::to_string(j) + "]";
        if (const int rc = check_device_buffer(fn, dname + idx, depth[j], device, 4)) return rc;
        if (const int rc = check_device_buffer(fn, other + idx, cleanup ? static_cast<const void*>(out[j]) : conf[j], device, 4)) return rc;
    }
    for (int j = 0; j < n_maps; ++j)
        B.add(depth[j], cleanup ? out[j] : const_cast<float*>(depth[j]), cleanup ? nullptr : conf[j], (unsigned)widths[j],
              (unsigned)heights[j], cleanup ? (unsigned long long)thres[j] : 0ull);
    return 0;
}

// Runs a checked batch on the caller's stream (NULL: the legacy default stream), after the work already there, and returns
// when the maps are written.  The workspace is freed on return.
int dm_device_run(const DmBatch& B, bool cleanup, void* cuda_stream)
{
    const cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    Work W;
    TempBuf tab(W), uf(W);
    if (const int rc = dm_run(W, B, tab, cleanup ? &uf : nullptr, s)) return rc;
    CK(cudaStreamSynchronize(s));
    return 0;
}

// ---- b200mvs_depthmap_pointset_device ----
// The outputs of a map, in b200mvs_dm_mesh order: what each element takes, how many the call may write, the names
struct MeshOut { void* p; uint64_t count; unsigned bytes; const char* name; const char* cap; };
void mesh_outputs(const b200mvs_dm_mesh& m, MeshOut out[7])
{
    const uint64_t n = (uint64_t)m.width * m.height, cv = m.cap_vertices;
    out[0] = {m.vertex_ids, n, 4, "vertex_ids", "width x height"};
    out[1] = {m.vertices, cv, 12, "vertices", "cap_vertices"};
    out[2] = {m.colors, cv, 16, "colors", "cap_vertices"};
    out[3] = {m.faces, m.cap_faces, 12, "faces", "cap_faces"};
    out[4] = {m.normals, cv, 12, "normals", "cap_vertices"};
    out[5] = {m.confidences, cv, 4, "confidences", "cap_vertices"};
    out[6] = {m.scales, cv, 4, "scales", "cap_vertices"};
}
bool count_only(const b200mvs_dm_mesh& m)
{
    return !m.vertex_ids && !m.vertices && !m.colors && !m.faces && !m.normals && !m.confidences && !m.scales;
}

// The largest map of b200mvs_depthmap_pointset_device.  A map larger than DM_CHUNK_PIXELS is a chunk of its own, whose
// scan must stay exact: up to two faces per pixel in the low 32 bits of (vertices << 32) | faces, and a pixel count plus
// one that cub takes as an int.
constexpr uint64_t MESH_MAX_PIXELS = 0x7FFFFFFEull;

// The arguments of b200mvs_depthmap_pointset_device, checked in full before anything is launched or written
int mesh_check(const char* fn, int device, int n_maps, const b200mvs_dm_mesh* maps, int conf_iterations)
{
    if (!maps) return fail(B200MVS_ERR_INVALID_ARG, "%s: maps is NULL", fn);
    if (conf_iterations < 0)                                                                             // depthmap.cc:503-504
        return fail(B200MVS_ERR_INVALID_ARG, "%s: conf_iterations is %d: Invalid amount of iterations", fn, conf_iterations);
    std::vector<Range> wr, rd;
    for (int j = 0; j < n_maps; ++j) {
        const b200mvs_dm_mesh& m = maps[j];
        if (!m.depth_dev) return fail(B200MVS_ERR_INVALID_ARG, "%s: maps[%d].depth_dev is NULL", fn, j);
        if (m.width < 2) return fail(B200MVS_ERR_INVALID_ARG, "%s: maps[%d].width is %d, must be at least 2", fn, j, m.width);
        if (m.height < 2) return fail(B200MVS_ERR_INVALID_ARG, "%s: maps[%d].height is %d, must be at least 2", fn, j, m.height);
        const uint64_t n = (uint64_t)m.width * m.height;
        if (n > MESH_MAX_PIXELS)
            return fail(B200MVS_ERR_INVALID_ARG, "%s: maps[%d] has %llu pixels (width x height), more than %llu", fn, j,
                        (unsigned long long)n, (unsigned long long)MESH_MAX_PIXELS);
        if (m.color_dev && (m.color_channels < 1 || m.color_channels > 4))
            return fail(B200MVS_ERR_INVALID_ARG, "%s: maps[%d].color_channels is %d, must be 1 to 4", fn, j, m.color_channels);
        const std::string map = "maps[" + std::to_string(j) + "].";
        const uintptr_t d = reinterpret_cast<uintptr_t>(m.depth_dev), c = reinterpret_cast<uintptr_t>(m.color_dev);
        rd.push_back(Range{d, d + n * 4, j, map + "depth_dev"});
        if (m.color_dev) rd.push_back(Range{c, c + n * (uint64_t)m.color_channels, j, map + "color_dev"});
        if (count_only(m)) continue;
        MeshOut out[7];
        mesh_outputs(m, out);
        for (const MeshOut& o : out) {
            if (!o.p) continue;
            const uintptr_t a = reinterpret_cast<uintptr_t>(o.p);
            if (o.count > (UINTPTR_MAX - a) / o.bytes)
                return fail(B200MVS_ERR_INVALID_ARG, "%s: %s%s: %llu x %u bytes from %p wrap the address space (%s)", fn, map.c_str(), o.name,
                            (unsigned long long)o.count, o.bytes, o.p, o.cap);
            wr.push_back(Range{a, a + o.count * o.bytes, j, map + o.name});
        }
    }
    if (const int rc = check_overlaps(fn, std::move(wr), rd, false)) return rc;
    CK(cudaSetDevice(device));
    for (int j = 0; j < n_maps; ++j) {
        const b200mvs_dm_mesh& m = maps[j];
        const std::string map = "maps[" + std::to_string(j) + "].";
        if (const int rc = check_device_buffer(fn, map + "depth_dev", m.depth_dev, device, 4)) return rc;
        if (m.color_dev) if (const int rc = check_device_buffer(fn, map + "color_dev", m.color_dev, device, 1)) return rc;
        MeshOut out[7];
        mesh_outputs(m, out);
        for (const MeshOut& o : out)
            if (o.p) if (const int rc = check_device_buffer(fn, map + o.name, o.p, device, 4)) return rc;
    }
    return 0;
}

// A checked call: the count pass over every map, the counts written back, then the outputs of every map that has any
// when none overflows.  The work runs on s; the workspace is freed on return.
int mesh_run(const char* fn, int n_maps, b200mvs_dm_mesh* maps, float dd_factor, int conf_iterations, float scale_factor, cudaStream_t s)
{
    TriBatch B;
    bool need_vids = false, need_verts = false;
    for (int j = 0; j < n_maps; ++j) {
        const b200mvs_dm_mesh& in = maps[j];
        TriMap m = {};
        m.dm = in.depth_dev; m.w = (unsigned)in.width; m.h = (unsigned)in.height; m.filled = !count_only(in);
        std::memcpy(m.P.m, in.invproj, sizeof(m.P.m));
        m.has_ctw = in.cam_to_world != nullptr;
        if (in.cam_to_world) std::memcpy(m.ctw, in.cam_to_world, sizeof(m.ctw));
        m.color = Color{in.color_dev, in.color_channels, in.color_channels, in.width};
        if (m.filled) {
            m.vids = in.vertex_ids; m.verts = in.vertices; m.colors = in.color_dev ? in.colors : nullptr; m.faces = in.faces;
            m.normals = in.normals; m.scales = in.scales; m.confs = conf_iterations > 0 ? in.confidences : nullptr;
            need_vids |= !m.vids;
            need_verts |= !m.verts;
        }
        B.add(m);
    }
    // the workspace of the largest chunk: codes, counts and their scan, and where the caller has no buffer for them, the
    // vertex ids and the vertices, which the kernels write for every filled map
    Work W;
    const size_t px = B.max_pixels;
    size_t scan = 0;
    CK(cub::DeviceScan::ExclusiveSum(nullptr, scan, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)(px + 1)));
    CK(W.need(W[Work::codes], px));
    CK(W.need(W[Work::counts], (px + 1) * 8));
    CK(W.need(W[Work::offsets], (px + 1) * 8));
    CK(W.need(W[Work::tmp], scan));
    if (need_vids) CK(W.need(W[Work::vids], px * 4));
    if (need_verts) CK(W.need(W[Work::verts], px * 12));
    if (B.confs) { CK(W.need(W[Work::ring0], px * 4)); CK(W.need(W[Work::ring1], px * 4)); CK(W.need(W[Work::last_hit], 4)); }
    for (TriMap& m : B.maps) {
        if (!m.filled) continue;
        if (!m.vids) m.vids = P<unsigned>(W[Work::vids]) + m.px0;
        if (!m.verts) m.verts = P<float>(W[Work::verts]) + 3 * (size_t)m.px0;
    }
    if (const int rc = tri_upload(W, B, s)) return rc;
    std::vector<uint64_t> totals;
    if (const int rc = tri_count(W, B, dd_factor, s, totals)) return rc;
    int over = -1;
    for (int j = 0; j < n_maps; ++j) {
        b200mvs_dm_mesh& m = maps[j];
        m.n_vertices = totals[j] >> 32;
        m.n_faces = totals[j] & 0xFFFFFFFFull;
        if (over < 0 && B.maps[j].filled && (m.n_vertices > m.cap_vertices || m.n_faces > m.cap_faces)) over = j;
    }
    if (over >= 0) {
        const b200mvs_dm_mesh& m = maps[over];
        return fail(B200MVS_ERR_OVERFLOW, "%s: maps[%d] has %llu vertices and %llu faces, cap_vertices is %llu and cap_faces %llu", fn, over,
                    (unsigned long long)m.n_vertices, (unsigned long long)m.n_faces, (unsigned long long)m.cap_vertices,
                    (unsigned long long)m.cap_faces);
    }
    if (const int rc = tri_fill(W, B, dd_factor, conf_iterations, scale_factor, s)) return rc;
    CK(cudaStreamSynchronize(s));
    return 0;
}

} // namespace

extern "C" {

const char* b200mvs_depthmap_last_error(void) { return last_error.c_str(); }

int b200mvs_depthmap_confidence_clean(int device, float* depth, const float* conf, int w, int h)
{
    if (!depth || !conf) return fail(B200MVS_ERR_INVALID_ARG, "Null depth or confidence map");     // depthmap.cc:120-121
    if (w < 1 || h < 1) return fail(B200MVS_ERR_INVALID_ARG, "Image dimensions do not match");
    const size_t n = (size_t)w * h;
    Work W;
    TempBuf d_dm(W), d_cm(W), tab(W);
    CK(cudaSetDevice(device));
    CK(W.need(d_dm, n * 4));
    CK(W.need(d_cm, n * 4));
    CK(cudaMemcpy(d_dm.p, depth, n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_cm.p, conf, n * 4, cudaMemcpyHostToDevice));
    // a batch of the staged map in pieces of at most 2^30 pixels: the filter is per pixel, and this entry point has no size limit
    DmBatch B(false);
    for (size_t o = 0; o < n; o += (size_t)1 << 30)
        B.add(P<float>(d_dm) + o, P<float>(d_dm) + o, P<float>(d_cm) + o, (unsigned)std::min(n - o, (size_t)1 << 30), 1u, 0ull);
    if (const int rc = dm_run(W, B, tab, nullptr, cudaStreamLegacy)) return rc;
    CK(cudaMemcpy(depth, d_dm.p, n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int b200mvs_depthmap_cleanup(int device, const float* depth, int w, int h, int64_t thres, float* out)
{
    if (!depth || !out || w < 1 || h < 1 || (size_t)w * h > 0xFFFFFFF0ull) return fail(B200MVS_ERR_INVALID_ARG, "depthmap_cleanup");
    const size_t n = (size_t)w * h;
    Work W;
    TempBuf d_dm(W), d_out(W), tab(W), uf(W);
    CK(cudaSetDevice(device));
    CK(W.need(d_dm, n * 4));
    CK(W.need(d_out, n * 4));
    CK(cudaMemcpy(d_dm.p, depth, n * 4, cudaMemcpyHostToDevice));
    // the reference compares collected.size() (size_t) < thres (size_t conversion of a negative int64 is huge: nothing survives)
    DmBatch B(true);
    B.add(P<float>(d_dm), P<float>(d_out), nullptr, (unsigned)w, (unsigned)h, (unsigned long long)thres);
    if (const int rc = dm_run(W, B, tab, &uf, cudaStreamLegacy)) return rc;
    CK(cudaMemcpy(out, d_out.p, n * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int b200mvs_depthmap_confidence_clean_device(int device, int n_maps, float* const* depth_dev, const float* const* conf_dev,
                                             const int32_t* widths, const int32_t* heights, void* cuda_stream)
{
    DmBatch B(false);
    if (const int rc = dm_device_batch("b200mvs_depthmap_confidence_clean_device", false, device, n_maps, depth_dev, conf_dev, widths,
                                       heights, nullptr, nullptr, B))
        return rc;
    return B.maps.empty() ? 0 : dm_device_run(B, false, cuda_stream);
}

int b200mvs_depthmap_cleanup_device(int device, int n_maps, const float* const* depth_dev, const int32_t* widths, const int32_t* heights,
                                    const int64_t* thres, float* const* out_dev, void* cuda_stream)
{
    DmBatch B(true);
    if (const int rc = dm_device_batch("b200mvs_depthmap_cleanup_device", true, device, n_maps, depth_dev, nullptr, widths, heights, thres,
                                       out_dev, B))
        return rc;
    return B.maps.empty() ? 0 : dm_device_run(B, true, cuda_stream);
}

int b200mvs_depthmap_triangulate(int device, const float* depth, int w, int h, const float invproj[9], float dd_factor,
                                 const float* cam_to_world, const uint8_t* color, int color_channels,
                                 uint32_t* vertex_ids, float* vertices, float* colors, uint32_t* faces,
                                 uint64_t cap_vertices, uint64_t cap_faces, uint64_t* n_vertices, uint64_t* n_faces,
                                 double* device_ms)
{
    return b200mvs_depthmap_pointset(device, depth, w, h, invproj, dd_factor, cam_to_world, color, color_channels, vertex_ids, vertices,
                                     colors, faces, nullptr, nullptr, 0, nullptr, 0.f, cap_vertices, cap_faces, n_vertices, n_faces, device_ms);
}

int b200mvs_depthmap_pointset(int device, const float* depth, int w, int h, const float invproj[9], float dd_factor,
                              const float* cam_to_world, const uint8_t* color, int color_channels,
                              uint32_t* vertex_ids, float* vertices, float* colors, uint32_t* faces,
                              float* normals, float* confidences, int conf_iterations, float* scales, float scale_factor,
                              uint64_t cap_vertices, uint64_t cap_faces, uint64_t* n_vertices, uint64_t* n_faces,
                              double* device_ms)
{
    if (!depth) return fail(B200MVS_ERR_INVALID_ARG, "Null depthmap given");                              // depthmap.cc:214-215
    if (!invproj || !n_vertices || !n_faces || w < 2 || h < 2) return fail(B200MVS_ERR_INVALID_ARG, "depthmap_triangulate");
    if (color && (color_channels < 1 || color_channels > 4)) return fail(B200MVS_ERR_INVALID_ARG, "Color image dimension mismatch");
    Work W;
    CK(cudaSetDevice(device));
    if (conf_iterations < 0) return fail(B200MVS_ERR_INVALID_ARG, "Invalid amount of iterations");     // depthmap.cc:503-504
    ViewJob J;
    *n_vertices = 0; *n_faces = 0;
    int rc = upload(W, depth, color, color_channels, w, h, &J.color);
    if (rc) return rc;
    J.dm = P<float>(W[Work::dm]); J.w = w; J.h = h; std::memcpy(J.P.m, invproj, sizeof(J.P.m)); J.dd_factor = dd_factor;
    J.ctw = cam_to_world; J.want_colors = colors && J.color.p;
    J.want_normals = normals != nullptr; J.want_scales = scales != nullptr; J.scale_factor = scale_factor;
    J.conf_iterations = confidences ? conf_iterations : 0;
    J.cap_v = cap_vertices; J.cap_f = cap_faces;
    uint64_t nv = 0, nf = 0;
    rc = run_view(W, J, &nv, &nf);
    *n_vertices = nv; *n_faces = nf;
    if (rc) return rc;
    CK(cudaEventSynchronize(W.ev[1]));
    if (device_ms) { float ms = 0.f; cudaEventElapsedTime(&ms, W.ev[0], W.ev[1]); *device_ms = ms; }
    const size_t n = (size_t)w * h;
    if (vertex_ids) CK(cudaMemcpy(vertex_ids, W[Work::vids].p, n * 4, cudaMemcpyDeviceToHost));
    if (vertices && nv) CK(cudaMemcpy(vertices, W[Work::verts].p, nv * 12, cudaMemcpyDeviceToHost));
    if (colors && W[Work::colors].p && nv) CK(cudaMemcpy(colors, W[Work::colors].p, nv * 16, cudaMemcpyDeviceToHost));
    if (faces && nf) CK(cudaMemcpy(faces, W[Work::faces].p, nf * 12, cudaMemcpyDeviceToHost));
    if (normals && nv) CK(cudaMemcpy(normals, W[Work::normals].p, nv * 12, cudaMemcpyDeviceToHost));
    if (scales && nv) CK(cudaMemcpy(scales, W[Work::scales].p, nv * 4, cudaMemcpyDeviceToHost));
    if (J.conf_iterations > 0 && nv) CK(cudaMemcpy(confidences, W[Work::confs].p, nv * 4, cudaMemcpyDeviceToHost));
    return 0;
}

int b200mvs_depthmap_pointset_device(int device, int n_maps, b200mvs_dm_mesh* maps, float dd_factor, int conf_iterations,
                                     float scale_factor, void* cuda_stream)
{
    static const char* fn = "b200mvs_depthmap_pointset_device";
    if (n_maps < 0) return fail(B200MVS_ERR_INVALID_ARG, "%s: n_maps is %d, must not be negative", fn, n_maps);
    if (n_maps == 0) return 0;
    if (const int rc = mesh_check(fn, device, n_maps, maps, conf_iterations)) return rc;
    return mesh_run(fn, n_maps, maps, dd_factor, conf_iterations, scale_factor, static_cast<cudaStream_t>(cuda_stream));
}

} // extern "C"

namespace {

// b200mvs_pset_create and b200mvs_pset_create_on_device (`fn`): the options checked, then a handle on `device`
int create(const char* fn, int device, bool on_device, const b200mvs_pset_options* o, b200mvs_pset** out)
{
    if (!o || !out) return fail(B200MVS_ERR_INVALID_ARG, "%s: null argument", fn);
    *out = nullptr;
    if (o->poisson_normals && !(o->with_normals && o->with_conf))
        return fail(B200MVS_ERR_INVALID_ARG, "%s: poisson_normals needs with_normals and with_conf", fn);
    // with_conf asks for a confidence per point: zero rings would give none (and -p, which reads them, would have nothing
    // to scale by; the reference's poisson_scale_normals throws on that, scene2pset.cc:124-125)
    if (o->with_conf && o->conf_iterations < 1) return fail(B200MVS_ERR_INVALID_ARG, "Invalid amount of iterations");
    if (o->correspondence && o->use_aabb)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: correspondence needs every vertex of a view (no bounding box)", fn);
    CK(cudaSetDevice(device));
    b200mvs_pset* ps = new b200mvs_pset;
    ps->device = device;
    ps->opt = *o;
    ps->set.on_device = on_device;
    *out = ps;
    return 0;
}

} // namespace

extern "C" {

int b200mvs_pset_create(int device, const b200mvs_pset_options* o, b200mvs_pset** out)
{
    return create("b200mvs_pset_create", device, false, o, out);
}

int b200mvs_pset_create_on_device(int device, const b200mvs_pset_options* o, b200mvs_pset** out)
{
    return create("b200mvs_pset_create_on_device", device, true, o, out);
}

void b200mvs_pset_destroy(b200mvs_pset* ps)
{
    if (!ps) return;
    cudaSetDevice(ps->device);
    for (int k = 0; k < Lists::N_LISTS; ++k) store_free(ps, ps->set.p[k], ps->set.cap[k] * 4 * Lists::PER[k]);
    delete ps;
}

int b200mvs_pset_add_view(b200mvs_pset* ps, int view_id, const float* depth, int w, int h, const uint8_t* color, int color_channels,
                          const b200mvs_pset_camera* cam, b200mvs_pset_view* out)
{
    int rc = check_add_view("b200mvs_pset_add_view", ps, depth, w, h, color, color_channels, cam);
    if (rc) return rc;
    CK(cudaSetDevice(ps->device));
    Color col;
    if ((rc = upload(ps->W, depth, color, color_channels, w, h, &col))) return rc;
    return add_view(ps, view_id, P<float>(ps->W[Work::dm]), w, h, col, *cam, out);
}

int b200mvs_pset_add_view_device(b200mvs_pset* ps, int view_id, const float* depth_dev, int w, int h, const uint8_t* color_dev,
                                 int color_channels, const b200mvs_pset_camera* cam, void* cuda_stream, b200mvs_pset_view* out)
{
    static const char* fn = "b200mvs_pset_add_view_device";
    int rc = check_add_view(fn, ps, depth_dev, w, h, color_dev, color_channels, cam);
    if (rc) return rc;
    CK(cudaSetDevice(ps->device));
    if ((rc = check_device_buffer(fn, "depth_dev", depth_dev, ps->device, 4)) || (color_dev && (rc = check_device_buffer(fn, "color_dev", color_dev, ps->device, 1))))
        return rc;
    // the handle's work runs on the legacy default stream, after what the caller enqueued on its stream
    CK(ps->W.events());
    if ((rc = wait_for_stream(ps->W.ev[4], cuda_stream, cudaStreamLegacy))) return rc;
    return add_view(ps, view_id, depth_dev, w, h, Color{color_dev, color_channels, color_channels, w}, *cam, out);
}

} // extern "C"

namespace {

// b200mvs_pset_clip_masks (`fn`: host masks, uploaded into one block) and b200mvs_pset_clip_masks_device (in_place: device
// masks with row pitches, read where they are after the work of cuda_stream)
int clip_masks(const char* fn, bool in_place, b200mvs_pset* ps, int n_masks, const uint8_t* const* masks, const int32_t* widths,
               const int32_t* heights, const int64_t* pitches, const b200mvs_pset_camera* cams, void* cuda_stream, uint64_t* num_filtered)
{
    if (!ps || n_masks < 0 || (n_masks && (!masks || !widths || !heights || !cams || (in_place && !pitches))))
        return fail(B200MVS_ERR_INVALID_ARG, "%s: null argument", fn);
    if (ps->opt.correspondence)
        return fail(B200MVS_ERR_INVALID_ARG, "%s: correspondence needs every vertex (no mask clipping)", fn);
    for (int m = 0; m < n_masks; ++m) {
        if (!masks[m] || widths[m] < 1 || heights[m] < 1 || cams[m].flen == 0.0f)
            return fail(B200MVS_ERR_INVALID_ARG, "%s: bad mask, size or camera", fn);
        if (in_place && pitches[m] < widths[m])
            return fail(B200MVS_ERR_INVALID_ARG, "%s: row_pitches[%d] is %lld, less than widths[%d] (%d)", fn, m, (long long)pitches[m], m,
                        widths[m]);
    }
    if (ps->clipped) return fail(B200MVS_ERR_INVALID_ARG, "%s: the masks have been applied already", fn);
    Work& W = ps->W;
    Lists& S = ps->set;
    TempBuf d_masks(W), d_cams(W), d_verts(W), d_del(W), before(W), scan_tmp(W), out(W);
    CK(cudaSetDevice(ps->device));
    if (in_place) {
        for (int m = 0; m < n_masks; ++m)
            if (const int rc = check_device_buffer(fn, "masks_dev[" + std::to_string(m) + "]", masks[m], ps->device, 1)) return rc;
        // the handle's work runs on the legacy default stream, after what the caller enqueued on its stream
        CK(W.events());
        if (const int rc = wait_for_stream(W.ev[4], cuda_stream, cudaStreamLegacy)) return rc;
    }
    ps->clipped = true;
    const uint64_t np = S.n[Lists::VERTS];
    std::vector<MaskCam> mc((size_t)n_masks);
    std::vector<size_t> offset((size_t)n_masks);
    size_t bytes = 0;
    for (int m = 0; m < n_masks; ++m) {
        MaskCam& C = mc[m];
        const b200mvs_pset_camera& c = cams[m];
        // CameraInfo::fill_world_to_cam (camera.cc:61-67) and fill_calibration for the mask's size
        const float Wm[12] = {c.rot[0], c.rot[1], c.rot[2], c.trans[0], c.rot[3], c.rot[4], c.rot[5], c.trans[1],
                              c.rot[6], c.rot[7], c.rot[8], c.trans[2]};
        std::memcpy(C.W, Wm, sizeof(Wm));
        fill_calibration(c.flen, c.paspect, c.ppoint[0], c.ppoint[1], (float)widths[m], (float)heights[m], C.K, nullptr);
        C.w = widths[m]; C.h = heights[m];
        C.mask = in_place ? masks[m] : nullptr;           // a host mask's place in d_masks is known once it is allocated
        C.pitch = in_place ? pitches[m] : widths[m];
        offset[m] = bytes;
        if (!in_place) bytes += (size_t)widths[m] * heights[m];
    }
    uint64_t filtered = 0;
    if (n_masks && np) {
        // mve::TriangleMesh::delete_vertices (mesh.cc:178-194): a per-point list is cleaned (math::algo::vector_clean,
        // algo.h:165-185) only when it has one entry per point (has_vertex_colors etc., mesh.h:256-274); a shorter colour
        // list - some view had no colour image - is left as it is
        bool clean[Lists::N_LISTS];
        int widest = 0;
        for (int k = 0; k < Lists::N_LISTS; ++k) if ((clean[k] = S.n[k] == np)) widest = std::max(widest, Lists::PER[k]);
        // The deletion flags come from the vertex list in chunks: a device set's chunk is read in place, a host set's goes
        // up first and its flags come back.  A device set keeps every flag for a 64-bit scan of them (cub takes int item
        // counts, so the scan runs in spans, each starting from the count before it); a host set needs device memory
        // for one chunk only.
        constexpr uint64_t CHUNK = (uint64_t)1 << 22, SPAN = (uint64_t)1 << 30;
        const bool dev = S.on_device;
        size_t scan_bytes = 0;
        CK(W.need(d_masks, bytes));
        CK(W.need(d_cams, mc.size() * sizeof(MaskCam)));
        CK(W.need(d_del, dev ? np : CHUNK));
        if (dev) {
            CK(cub::DeviceScan::ExclusiveScan(nullptr, scan_bytes, (const unsigned char*)nullptr, (unsigned long long*)nullptr,
                                               cuda::std::plus<unsigned long long>{}, 0ull, (int)std::min(np, SPAN)));
            CK(W.need(before, np * 8));
            CK(W.need(scan_tmp, scan_bytes));
            CK(W.need(out, np * widest * 4));
        } else {
            CK(W.need(d_verts, CHUNK * 12));
        }
        std::vector<unsigned char> del(dev ? 0 : np);
        // ms_mask (b200mvs_pset_info): a host set's time includes every transfer, a device set's only the work in place
        CK(W.events());
        if (!dev) CK(cudaEventRecord(W.ev[2]));
        for (int m = 0; m < n_masks && !in_place; ++m) {
            mc[m].mask = P<unsigned char>(d_masks) + offset[m];
            CK(cudaMemcpy(P<unsigned char>(d_masks) + offset[m], masks[m], (size_t)widths[m] * heights[m], cudaMemcpyHostToDevice));
        }
        CK(cudaMemcpy(d_cams.p, mc.data(), mc.size() * sizeof(MaskCam), cudaMemcpyHostToDevice));
        if (dev) CK(cudaEventRecord(W.ev[2]));
        for (uint64_t at = 0; at < np; at += CHUNK) {
            const uint64_t k = std::min(CHUNK, np - at);
            const float* v = static_cast<const float*>(S.p[Lists::VERTS]) + 3 * at;
            unsigned char* d = P<unsigned char>(d_del) + (dev ? at : 0);
            if (!dev) { CK(cudaMemcpy(d_verts.p, v, k * 12, cudaMemcpyHostToDevice)); v = P<float>(d_verts); }
            k_mask_clip<<<(unsigned)((k + 255) / 256), 256>>>(v, k, P<MaskCam>(d_cams), n_masks, d);
            CK(cudaGetLastError());
            if (!dev) CK(cudaMemcpy(del.data() + at, d, k, cudaMemcpyDeviceToHost));
        }
        if (dev) {
            // one stable compaction of every cleaned list: entry i moves to i - (points deleted before i)
            const unsigned char* d_flags = P<unsigned char>(d_del);
            unsigned long long* d_before = P<unsigned long long>(before);
            for (uint64_t a = 0; a < np; a += SPAN) {
                const uint64_t k = std::min(SPAN, np - a);
                CK(cub::DeviceScan::ExclusiveScan(scan_tmp.p, scan_bytes, d_flags + a, d_before + a, cuda::std::plus<unsigned long long>{},
                                                   (unsigned long long)filtered, (int)k));
                unsigned long long last = 0;
                unsigned char last_del = 0;
                CK(cudaMemcpy(&last, d_before + a + k - 1, 8, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy(&last_del, d_flags + a + k - 1, 1, cudaMemcpyDeviceToHost));
                filtered = last + last_del;
            }
            for (int k = 0; k < Lists::N_LISTS; ++k) {
                if (!clean[k]) continue;
                const int per = Lists::PER[k];
                k_clip_compact<<<(unsigned)((np + 255) / 256), 256>>>(d_flags, d_before, np, per, static_cast<const float*>(S.p[k]), P<float>(out));
                CK(cudaGetLastError());
                if (np > filtered) CK(cudaMemcpyAsync(S.p[k], out.p, (np - filtered) * per * 4, cudaMemcpyDeviceToDevice, cudaStreamLegacy));
            }
        }
        CK(cudaEventRecord(W.ev[3]));
        CK(cudaEventSynchronize(W.ev[3]));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, W.ev[2], W.ev[3]);
        ps->ms_mask += ms;
        if (!dev) {
            // the same compaction on the host, from the flags
            for (uint64_t i = 0; i < np; ++i) filtered += del[i];
            for (int k = 0; k < Lists::N_LISTS; ++k) {
                if (!clean[k]) continue;
                const size_t item = 4 * (size_t)Lists::PER[k];
                char* a = static_cast<char*>(S.p[k]);
                uint64_t wr = 0;
                for (uint64_t i = 0; i < np; ++i) {
                    if (del[i]) continue;
                    if (wr != i) std::memmove(a + wr * item, a + i * item, item);
                    ++wr;
                }
            }
        }
        for (int k = 0; k < Lists::N_LISTS; ++k) if (clean[k]) S.n[k] = np - filtered;
    }
    if (num_filtered) *num_filtered = filtered;
    return 0;
}

} // namespace

extern "C" {

int b200mvs_pset_clip_masks(b200mvs_pset* ps, int n_masks, const uint8_t* const* masks, const int32_t* widths, const int32_t* heights,
                            const b200mvs_pset_camera* cams, uint64_t* num_filtered)
{
    return clip_masks("b200mvs_pset_clip_masks", false, ps, n_masks, masks, widths, heights, nullptr, cams, nullptr, num_filtered);
}

int b200mvs_pset_clip_masks_device(b200mvs_pset* ps, int n_masks, const uint8_t* const* masks_dev, const int32_t* widths,
                                   const int32_t* heights, const int64_t* row_pitches, const b200mvs_pset_camera* cams,
                                   void* cuda_stream, uint64_t* num_filtered)
{
    return clip_masks("b200mvs_pset_clip_masks_device", true, ps, n_masks, masks_dev, widths, heights, row_pitches, cams, cuda_stream,
                      num_filtered);
}

int b200mvs_pset_get_info(b200mvs_pset* ps, b200mvs_pset_info* out)
{
    if (!ps || !out) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_get_info: null argument");
    out->n_points = ps->set.n[Lists::VERTS];
    out->n_colors = ps->set.n[Lists::COLORS];
    out->n_views = ps->n_views;
    out->device_bytes = ps->W.held;
    out->peak_device_bytes = ps->W.peak;
    out->ms_pointset = ps->ms_pointset;
    out->ms_filter = ps->ms_filter;
    out->ms_mask = ps->ms_mask;
    return 0;
}

int b200mvs_pset_read(b200mvs_pset* ps, float* vertices, float* normals, float* colors, float* values, float* confidences)
{
    if (!ps) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_read: null handle");
    CK(cudaSetDevice(ps->device));
    const Lists& S = ps->set;
    void* dst[] = {vertices, normals, colors, values, confidences};
    for (int k = 0; k < 5; ++k)
        if (dst[k] && S.n[k]) CK(store_copy(ps, dst[k], S.p[k], S.n[k] * Lists::PER[k] * 4));
    return 0;
}

int b200mvs_pset_read_correspondence(b200mvs_pset* ps, uint32_t* pixels_xy, b200mvs_pset_corr_view* views)
{
    if (!ps) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_read_correspondence: null handle");
    if (!ps->opt.correspondence) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_read_correspondence: handle made without correspondence");
    const Lists& S = ps->set;
    if (pixels_xy && S.n[Lists::PIX]) {
        CK(cudaSetDevice(ps->device));
        CK(store_copy(ps, pixels_xy, S.p[Lists::PIX], S.n[Lists::PIX] * 8));
    }
    if (views && !ps->corr.empty()) std::memcpy(views, ps->corr.data(), ps->corr.size() * sizeof(b200mvs_pset_corr_view));
    return 0;
}

int b200mvs_pset_read_device(b200mvs_pset* ps, float* vertices, float* normals, float* colors, float* values, float* confidences,
                             uint32_t* pixels_xy, void* cuda_stream)
{
    static const char* fn = "b200mvs_pset_read_device";
    if (!ps) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_read_device: null handle");
    if (pixels_xy && !ps->opt.correspondence)
        return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_read_device: pixels_xy given for a handle made without correspondence");
    CK(cudaSetDevice(ps->device));
    const Lists& S = ps->set;
    void* dst[Lists::N_LISTS] = {vertices, normals, colors, values, confidences, pixels_xy};
    static const char* names[Lists::N_LISTS] = {"vertices", "normals", "colors", "values", "confidences", "pixels_xy"};
    for (int k = 0; k < Lists::N_LISTS; ++k)
        if (dst[k]) if (const int rc = check_device_buffer(fn, names[k], dst[k], ps->device, 4)) return rc;
    // the copies run on the legacy default stream, after what the caller enqueued on its stream
    CK(ps->W.events());
    if (const int rc = wait_for_stream(ps->W.ev[4], cuda_stream, cudaStreamLegacy)) return rc;
    for (int k = 0; k < Lists::N_LISTS; ++k)
        if (dst[k] && S.n[k]) CK(cudaMemcpyAsync(dst[k], S.p[k], S.n[k] * Lists::PER[k] * 4, cudaMemcpyDefault, cudaStreamLegacy));
    CK(cudaStreamSynchronize(cudaStreamLegacy));
    return 0;
}

} // extern "C"

namespace b200mvs_pset_dev {

int check(const b200mvs_pset* ps, int device)
{
    if (!ps) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_add_reconstruction: null handle");
    if (ps->device != device)
        return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_add_reconstruction: the handle is on device %d, the context on device %d", ps->device, device);
    if (ps->clipped) return fail(B200MVS_ERR_INVALID_ARG, "b200mvs_pset_add_reconstruction: the masks have been applied already");
    return 0;
}

uint64_t workspace_bytes(const b200mvs_pset* ps, int w, int h)
{
    // the map and the colour image stay where the reconstruction left them
    const float ctw[16] = {};
    uint64_t b = 0;
    for_each_view_buffer(pset_job(ps->opt, w, h, ctw, true), (uint64_t)w * h, [&](Step, Work::Id, size_t bytes) { b += bytes; });
    return b;
}

void use_allocator(b200mvs_pset* ps, const Allocator* a)
{
    cudaSetDevice(ps->device);
    ps->W.release();
    ps->W.A = a ? *a : Allocator{};
}

int extract(b200mvs_pset* ps, int view_id, const float* d_depth, int w, int h, const void* d_rgbx, int pitch,
            const b200mvs_pset_camera& cam, Block& out)
{
    if (cam.flen == 0.0f) return fail(B200MVS_ERR_INVALID_ARG, "Invalid camera given");                  // depthmap.cc:383-384
    CK(cudaSetDevice(ps->device));
    out = Block{};
    out.view_id = (uint32_t)view_id; out.width = (uint32_t)w; out.height = (uint32_t)h;
    // the level's texels are RGBX: three channels, four bytes apart
    const Color col{static_cast<const uint8_t*>(d_rgbx), 3, 4, pitch};
    float ms_view = 0.f, ms_filt = 0.f;
    const Lists& S = ps->set;
    for (int k = 0; k < Lists::N_LISTS; ++k) out.at[k] = S.n[k] + S.staged[k];
    const int rc = add_device_view(ps, d_depth, w, h, col, cam, out.rec, ms_view, ms_filt);
    for (int k = 0; k < Lists::N_LISTS; ++k) out.count[k] = S.n[k] + S.staged[k] - out.at[k];
    out.ms_pointset = ms_view; out.ms_filter = ms_filt;
    return rc;
}

int commit(b200mvs_pset* ps, const std::vector<Block>& blocks, b200mvs_pset_view* records)
{
    if (const int rc = order_staged(ps, blocks)) { discard(ps); return rc; }
    Lists& S = ps->set;
    for (size_t j = 0; j < blocks.size(); ++j) {
        const Block& b = blocks[j];
        b200mvs_pset_view rec = b.rec;
        rec.first_index = S.n[Lists::VERTS];
        ps->ms_pointset += b.ms_pointset;
        ps->ms_filter += b.ms_filter;
        if (rec.added) {
            add_corr(ps, (int)b.view_id, (int)b.width, (int)b.height, S.n[Lists::PIX]);
            for (int k = 0; k < Lists::N_LISTS; ++k) { S.n[k] += b.count[k]; S.staged[k] -= b.count[k]; }
            ps->n_views += 1;
        }
        if (records) records[j] = rec;
    }
    return 0;
}

void discard(b200mvs_pset* ps)
{
    for (uint64_t& s : ps->set.staged) s = 0;
}

} // namespace b200mvs_pset_dev
