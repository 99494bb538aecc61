// Depth-map consumers that run right after dmrecon (SURVEY.md 8f rank 2 and 3), on the device:
//   * mve::image::depthmap_confidence_clean and depthmap_cleanup (libs/mve/depthmap.cc:25-131)
//   * mve::geom::depthmap_triangulate with pixel_3dpos / pixel_footprint (libs/mve/depthmap.cc:136-375), the per-view work of
//     apps/scene2pset (scene2pset.cc:264-328): vertex ids, vertices, colours and faces in EXACTLY the reference's order.
// All of these are streaming kernels over one depth map; the results are bit-exact for the integer parts (masks, component
// sizes, vertex ids, faces) and for the float parts that are pure per-pixel functions evaluated in the reference's operation
// order with IEEE operations (__fmul_rn / __fadd_rn; __fmaf_rn only where the reference build itself contracts and the
// result decides a face: pixel_footprint).
#include "../../include/b200mvs.h"

#include <cub/device/device_scan.cuh>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

namespace {

thread_local std::string g_dm_error;

int dm_fail(int code, const char* what, cudaError_t e)
{
    char buf[256];
    std::snprintf(buf, sizeof(buf), "%s: %s", what, e == cudaSuccess ? "invalid argument" : cudaGetErrorString(e));
    g_dm_error = buf;
    return code;
}
#define DCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { cleanup(); return dm_fail(B200MVS_ERR_CUDA, #call, e_); } } while (0)

// ---- depthmap_confidence_clean (depthmap.cc:118-131) ----
__global__ void k_conf_clean(float* __restrict__ dm, const float* __restrict__ cm, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && cm[i] <= 0.0f) dm[i] = 0.0f;
}

// ---- depthmap_cleanup (depthmap.cc:25-113): 4-connected components of dm != 0, components smaller than thres are erased ----
// Union-find on the pixel grid: every pixel links to its right and lower neighbour (atomicMin on roots), the roots are then
// flattened, counted, and small components zeroed.  Component sizes are exact, so the result equals the reference's region
// growing bit for bit.
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
__global__ void k_cc_init(const float* __restrict__ dm, unsigned* __restrict__ parent, unsigned* __restrict__ count, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    parent[i] = (unsigned)i;
    count[i] = 0u;
}
__global__ void k_cc_link(const float* __restrict__ dm, unsigned* __restrict__ parent, int w, int h)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t i = (size_t)y * w + x;
    if (dm[i] == 0.0f) return;
    if (x + 1 < w && dm[i + 1] != 0.0f) uf_union(parent, (unsigned)i, (unsigned)(i + 1));
    if (y + 1 < h && dm[i + w] != 0.0f) uf_union(parent, (unsigned)i, (unsigned)(i + w));
}
__global__ void k_cc_count(const float* __restrict__ dm, unsigned* __restrict__ parent, unsigned* __restrict__ count, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || dm[i] == 0.0f) return;
    const unsigned r = uf_find(parent, (unsigned)i);
    parent[i] = r;
    atomicAdd(&count[r], 1u);
}
__global__ void k_cc_erase(const float* __restrict__ dm, const unsigned* __restrict__ parent, const unsigned* __restrict__ count,
                           unsigned long long thres, float* __restrict__ out, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float d = dm[i];
    out[i] = (d != 0.0f && (unsigned long long)count[parent[i]] < thres) ? 0.0f : d;
}

// ---- depthmap_triangulate ----
// pixel_3dpos / pixel_footprint (depthmap.cc:136-156): ray = invproj * (x + .5, y + .5, 1), math::Matrix::mult accumulates
// from zero, left to right.
struct InvProj { float m[9]; };
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

__global__ void k_tri_codes(const float* __restrict__ dm, int w, int h, InvProj P, float dd_factor, float dd_diag,
                            unsigned char* __restrict__ codes)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    codes[(size_t)y * w + x] = (unsigned char)block_code(dm, w, h, x, y, P, dd_factor, dd_diag);
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
__global__ void k_tri_counts(const unsigned char* __restrict__ codes, int w, int h, unsigned long long* __restrict__ counts)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t i = (size_t)y * w + x;
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
    counts[i] = ((unsigned long long)nv << 32) | nf;
}
__global__ void k_tri_vertices(const float* __restrict__ dm, const unsigned char* __restrict__ codes, int w, int h, InvProj P,
                               const unsigned long long* __restrict__ offsets, const float* __restrict__ ctw,
                               const unsigned char* __restrict__ color, int cch,
                               unsigned* __restrict__ vids, float* __restrict__ verts, float* __restrict__ colors)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t i = (size_t)y * w + x;
    const unsigned code = codes[i];
    unsigned id = (unsigned)(offsets[i] >> 32), seen = 0u;
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
            const float nrm = vec_norm(rx, ry, rz), d = dm[pi];
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
                // depthmap.cc:349-364: (r, g, b, 255) / 255, grey expanded
                const float r = (float)color[pi * cch], g = cch >= 3 ? (float)color[pi * cch + 1] : r, b = cch >= 3 ? (float)color[pi * cch + 2] : r;
                colors[4 * (size_t)id] = __fdiv_rn(r, 255.0f); colors[4 * (size_t)id + 1] = __fdiv_rn(g, 255.0f);
                colors[4 * (size_t)id + 2] = __fdiv_rn(b, 255.0f); colors[4 * (size_t)id + 3] = 1.0f;
            }
            ++id;
        }
    }
}
__global__ void k_tri_faces(const unsigned char* __restrict__ codes, int w, int h, const unsigned long long* __restrict__ offsets,
                            const unsigned* __restrict__ vids, unsigned* __restrict__ faces)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t i = (size_t)y * w + x;
    const unsigned code = codes[i];
    size_t f = (size_t)(offsets[i] & 0xFFFFFFFFull);
    for (int j = 0; j < 2; ++j) {
        const int t = (code >> (4 * j)) & 0xF;
        if (!t) continue;
        for (int q = 0; q < 3; ++q) {
            const int c = c_tris[t - 1][q];
            faces[3 * f + q] = vids[i + (c & 1) + (size_t)w * (c >> 1)];
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

__global__ void k_vertex_attributes(const unsigned char* __restrict__ codes, const unsigned* __restrict__ vids, int w, int h,
                                    const float* __restrict__ verts, float scale_factor,
                                    float* __restrict__ normals, float* __restrict__ scales, unsigned* __restrict__ ring)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t pi = (size_t)y * w + x;
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
// One launch per ring.  A ring distance is below the number of vertices (< 2^32), so RING_NONE never collides with one.  A
// round that reaches a vertex stores its d in *last_hit; once a round reaches none, no later round can, and the host stops.
__global__ void k_conf_ring(const unsigned char* __restrict__ codes, const unsigned* __restrict__ vids, int w, int h,
                            const unsigned* __restrict__ ring_in, unsigned* __restrict__ ring_out, unsigned d,
                            unsigned* __restrict__ last_hit)
{
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t pi = (size_t)y * w + x;
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
    ring_out[pi] = r;
}
__global__ void k_conf_write(const unsigned* __restrict__ vids, const unsigned* __restrict__ ring, size_t n, int iterations, float* __restrict__ confs)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned v = vids[i];
    if (v == 0xFFFFFFFFu) return;
    const unsigned r = ring[i];
    // current * (1 / iterations): the reference build hoists the division of depthmap.cc:527 out of its loop
    confs[v] = r < (unsigned)iterations ? __fmul_rn((float)r, __frcp_rn((float)iterations)) : 1.0f;
}

__global__ void k_fill_u32(unsigned* p, unsigned v, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

} // namespace

extern "C" {

const char* b200mvs_depthmap_last_error(void) { return g_dm_error.c_str(); }

int b200mvs_depthmap_confidence_clean(int device, float* depth, const float* conf, int w, int h)
{
    float *d_dm = nullptr, *d_cm = nullptr;
    auto cleanup = [&]() { if (d_dm) cudaFree(d_dm); if (d_cm) cudaFree(d_cm); };
    if (!depth || !conf) return dm_fail(B200MVS_ERR_INVALID_ARG, "Null depth or confidence map", cudaSuccess);     // depthmap.cc:120-121
    if (w < 1 || h < 1) return dm_fail(B200MVS_ERR_INVALID_ARG, "Image dimensions do not match", cudaSuccess);
    const size_t n = (size_t)w * h;
    DCK(cudaSetDevice(device));
    DCK(cudaMalloc(&d_dm, n * 4));
    DCK(cudaMalloc(&d_cm, n * 4));
    DCK(cudaMemcpy(d_dm, depth, n * 4, cudaMemcpyHostToDevice));
    DCK(cudaMemcpy(d_cm, conf, n * 4, cudaMemcpyHostToDevice));
    k_conf_clean<<<(unsigned)((n + 255) / 256), 256>>>(d_dm, d_cm, n);
    DCK(cudaGetLastError());
    DCK(cudaMemcpy(depth, d_dm, n * 4, cudaMemcpyDeviceToHost));
    cleanup();
    return 0;
}

int b200mvs_depthmap_cleanup(int device, const float* depth, int w, int h, int64_t thres, float* out)
{
    float *d_dm = nullptr, *d_out = nullptr;
    unsigned *d_parent = nullptr, *d_count = nullptr;
    auto cleanup = [&]() { if (d_dm) cudaFree(d_dm); if (d_out) cudaFree(d_out); if (d_parent) cudaFree(d_parent); if (d_count) cudaFree(d_count); };
    if (!depth || !out || w < 1 || h < 1 || (size_t)w * h > 0xFFFFFFF0ull) return dm_fail(B200MVS_ERR_INVALID_ARG, "depthmap_cleanup", cudaSuccess);
    const size_t n = (size_t)w * h;
    DCK(cudaSetDevice(device));
    DCK(cudaMalloc(&d_dm, n * 4));
    DCK(cudaMalloc(&d_out, n * 4));
    DCK(cudaMalloc(&d_parent, n * 4));
    DCK(cudaMalloc(&d_count, n * 4));
    DCK(cudaMemcpy(d_dm, depth, n * 4, cudaMemcpyHostToDevice));
    const unsigned nb = (unsigned)((n + 255) / 256);
    const dim3 blk(32, 8), grd((w + 31) / 32, (h + 7) / 8);
    k_cc_init<<<nb, 256>>>(d_dm, d_parent, d_count, n);
    k_cc_link<<<grd, blk>>>(d_dm, d_parent, w, h);
    k_cc_count<<<nb, 256>>>(d_dm, d_parent, d_count, n);
    // the reference compares collected.size() (size_t) < thres (size_t conversion of a negative int64 is huge: nothing survives)
    k_cc_erase<<<nb, 256>>>(d_dm, d_parent, d_count, (unsigned long long)thres, d_out, n);
    DCK(cudaGetLastError());
    DCK(cudaMemcpy(out, d_out, n * 4, cudaMemcpyDeviceToHost));
    cleanup();
    return 0;
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
    float *d_dm = nullptr, *d_verts = nullptr, *d_colors = nullptr, *d_ctw = nullptr, *d_normals = nullptr, *d_confs = nullptr, *d_scales = nullptr;
    unsigned char *d_codes = nullptr, *d_color = nullptr;
    unsigned *d_ring0 = nullptr, *d_ring1 = nullptr, *d_last_hit = nullptr;
    unsigned long long *d_counts = nullptr, *d_offsets = nullptr;
    unsigned *d_vids = nullptr, *d_faces = nullptr;
    void* d_tmp = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    auto cleanup = [&]() {
        for (void* p : {(void*)d_dm, (void*)d_verts, (void*)d_colors, (void*)d_ctw, (void*)d_codes, (void*)d_color, (void*)d_counts,
                        (void*)d_offsets, (void*)d_vids, (void*)d_faces, d_tmp, (void*)d_normals, (void*)d_confs, (void*)d_scales,
                        (void*)d_ring0, (void*)d_ring1, (void*)d_last_hit}) if (p) cudaFree(p);
        if (e0) cudaEventDestroy(e0);
        if (e1) cudaEventDestroy(e1);
    };
    if (!depth) return dm_fail(B200MVS_ERR_INVALID_ARG, "Null depthmap given", cudaSuccess);                              // depthmap.cc:214-215
    if (!invproj || !n_vertices || !n_faces || w < 2 || h < 2) return dm_fail(B200MVS_ERR_INVALID_ARG, "depthmap_triangulate", cudaSuccess);
    if (color && (color_channels < 1 || color_channels > 4)) return dm_fail(B200MVS_ERR_INVALID_ARG, "Color image dimension mismatch", cudaSuccess);
    const size_t n = (size_t)w * h;
    InvProj P;
    std::memcpy(P.m, invproj, sizeof(P.m));
    DCK(cudaSetDevice(device));
    DCK(cudaMalloc(&d_dm, n * 4));
    DCK(cudaMalloc(&d_codes, n));
    DCK(cudaMalloc(&d_counts, (n + 1) * 8));
    DCK(cudaMalloc(&d_offsets, (n + 1) * 8));
    DCK(cudaMalloc(&d_vids, n * 4));
    DCK(cudaMemcpy(d_dm, depth, n * 4, cudaMemcpyHostToDevice));
    if (cam_to_world) { DCK(cudaMalloc(&d_ctw, 64)); DCK(cudaMemcpy(d_ctw, cam_to_world, 64, cudaMemcpyHostToDevice)); }
    if (color) { DCK(cudaMalloc(&d_color, n * color_channels)); DCK(cudaMemcpy(d_color, color, n * color_channels, cudaMemcpyHostToDevice)); }
    size_t tmp_bytes = 0;
    DCK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_counts, d_offsets, (int)(n + 1)));
    DCK(cudaMalloc(&d_tmp, tmp_bytes));
    DCK(cudaEventCreate(&e0));
    DCK(cudaEventCreate(&e1));
    // worst-case sized outputs, allocated before the clock starts (cudaMalloc synchronises): a vertex per pixel, two faces per block
    const size_t max_v = n, max_f = 2 * (size_t)(w - 1) * (h - 1);
    DCK(cudaMalloc(&d_verts, max_v * 12));
    if (color && colors) DCK(cudaMalloc(&d_colors, max_v * 16));
    DCK(cudaMalloc(&d_faces, (max_f ? max_f : 1) * 12));
    if (conf_iterations < 0) { cleanup(); return dm_fail(B200MVS_ERR_INVALID_ARG, "Invalid amount of iterations", cudaSuccess); }     // depthmap.cc:503-504
    const bool want_conf = confidences && conf_iterations > 0;
    if (normals) DCK(cudaMalloc(&d_normals, max_v * 12));
    if (scales) DCK(cudaMalloc(&d_scales, max_v * 4));
    if (want_conf) {
        DCK(cudaMalloc(&d_confs, max_v * 4)); DCK(cudaMalloc(&d_ring0, n * 4)); DCK(cudaMalloc(&d_ring1, n * 4));
        DCK(cudaMalloc(&d_last_hit, 4));
    }
    const dim3 blk(32, 8), grd((w + 31) / 32, (h + 7) / 8);
    DCK(cudaEventRecord(e0));
    const float dd_diag = (float)((double)dd_factor * 1.41421356237309504880);       // MATH_SQRT2, rounded like depthmap.cc:198
    k_tri_codes<<<grd, blk>>>(d_dm, w, h, P, dd_factor, dd_diag, d_codes);
    DCK(cudaMemsetAsync(d_counts + n, 0, 8));
    k_tri_counts<<<grd, blk>>>(d_codes, w, h, d_counts);
    DCK(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_counts, d_offsets, (int)(n + 1)));
    unsigned long long total = 0;
    DCK(cudaMemcpy(&total, d_offsets + n, 8, cudaMemcpyDeviceToHost));
    const uint64_t nv = total >> 32, nf = total & 0xFFFFFFFFull;
    *n_vertices = nv; *n_faces = nf;
    if (nv > cap_vertices || nf > cap_faces) { cleanup(); return dm_fail(B200MVS_ERR_OVERFLOW, "depthmap_triangulate: output capacity too small", cudaSuccess); }
    k_fill_u32<<<(unsigned)((n + 255) / 256), 256>>>(d_vids, 0xFFFFFFFFu, n);
    k_tri_vertices<<<grd, blk>>>(d_dm, d_codes, w, h, P, d_offsets, d_ctw, d_color, color_channels, d_vids, d_verts, d_colors);
    k_tri_faces<<<grd, blk>>>(d_codes, w, h, d_offsets, d_vids, d_faces);
    if (normals || scales || want_conf)
        k_vertex_attributes<<<grd, blk>>>(d_codes, d_vids, w, h, d_verts, scale_factor, d_normals, d_scales, d_ring0);
    if (want_conf) {
        // rings 1 .. conf_iterations - 1; every RING_CHECK rounds the host asks whether the last round still reached a
        // vertex, so a large conf_iterations costs as many launches as the mesh has rings, not conf_iterations
        constexpr int RING_CHECK = 16;
        unsigned *cur = d_ring0, *nxt = d_ring1;
        DCK(cudaMemsetAsync(d_last_hit, 0, 4));
        for (int d = 1; d < conf_iterations; ++d) {
            k_conf_ring<<<grd, blk>>>(d_codes, d_vids, w, h, cur, nxt, (unsigned)d, d_last_hit);
            unsigned* t = cur; cur = nxt; nxt = t;
            if (d % RING_CHECK == 0) {
                unsigned last = 0;
                DCK(cudaMemcpy(&last, d_last_hit, 4, cudaMemcpyDeviceToHost));
                if (last != (unsigned)d) break;
            }
        }
        k_conf_write<<<(unsigned)((n + 255) / 256), 256>>>(d_vids, cur, n, conf_iterations, d_confs);
    }
    DCK(cudaEventRecord(e1));
    DCK(cudaGetLastError());
    DCK(cudaEventSynchronize(e1));
    if (device_ms) { float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1); *device_ms = ms; }
    if (vertex_ids) DCK(cudaMemcpy(vertex_ids, d_vids, n * 4, cudaMemcpyDeviceToHost));
    if (vertices && nv) DCK(cudaMemcpy(vertices, d_verts, nv * 12, cudaMemcpyDeviceToHost));
    if (colors && d_colors && nv) DCK(cudaMemcpy(colors, d_colors, nv * 16, cudaMemcpyDeviceToHost));
    if (faces && nf) DCK(cudaMemcpy(faces, d_faces, nf * 12, cudaMemcpyDeviceToHost));
    if (normals && nv) DCK(cudaMemcpy(normals, d_normals, nv * 12, cudaMemcpyDeviceToHost));
    if (scales && nv) DCK(cudaMemcpy(scales, d_scales, nv * 4, cudaMemcpyDeviceToHost));
    if (want_conf && nv) DCK(cudaMemcpy(confidences, d_confs, nv * 4, cudaMemcpyDeviceToHost));
    cleanup();
    return 0;
}

} // extern "C"
