"""A plain NumPy restatement of the depth-map operations of the reference (libs/mve/depthmap.cc, mesh.cc, mesh_info.cc and the
per-view work of apps/scene2pset/scene2pset.cc:316-358), independent of the CUDA kernels in mve_b200/csrc/depthmap.cu.

Every decision (masks, component sizes, triangle choice, depth discontinuities, vertex numbering, faces, vertex classes,
confidence rings) is evaluated exactly: in float32 where the reference uses float, with the arithmetic the reference build
(-O3 -funsafe-math-optimizations -march=x86-64-v3) actually emits.  Vertex positions come in two forms: `vertices` repeats
the reference build's float32 operations, `vertices64` is the same quantity in float64.  Normals and scale values are
float64.  tests/test_depthmap_reference.py pins this module against the reference binary's own results."""
import numpy as np
import scipy.ndimage
import scipy.sparse
import scipy.sparse.csgraph

F32 = np.float32
NO_VERTEX = np.uint32(0xFFFFFFFF)
MATH_SQRT2 = 1.41421356237309504880168872420969808      # math/defines.h:49, a double literal
TRIS = np.array([[0, 2, 1], [0, 3, 1], [0, 2, 3], [1, 2, 3]])  # depthmap.cc:251-253, corner j = pixel (j % 2, j / 2)
FOUR = np.array([[0, 1, 0], [1, 1, 1], [0, 1, 0]])


# ---- depthmap.cc:25-111 / 116-128 ----
def cleanup(dm, thres):
    """depthmap_cleanup: 4-connected components of `dm != 0.0f` (so -0.0 is empty; NaN, +-inf and negative depths are
    filled) with fewer than `thres` pixels are set to 0.0f.  `thres` is compared as size_t (depthmap.cc:27, :82), so a
    negative value erases every component."""
    dm = np.asarray(dm, F32)
    filled = dm != 0.0
    labels, _ = scipy.ndimage.label(filled, structure=FOUR)
    size = np.bincount(labels.ravel())
    t = int(thres) % (1 << 64)
    small = filled if t > dm.size else filled & (size[labels] < t)
    out = dm.copy()
    out[small] = 0.0
    return out


def confidence_clean(dm, cm):
    """depthmap_confidence_clean: depth = 0.0f where `conf <= 0.0f` (NaN keeps the depth, -0.0 clears it)."""
    out = np.array(dm, F32)
    out[np.asarray(cm, F32) <= 0.0] = 0.0
    return out


# ---- float32 arithmetic of the reference build ----
def fma32(a, b, c):
    """Single-precision fused multiply-add, correctly rounded: a*b is exact in float64 and the sum's float64 rounding error
    (TwoSum) breaks the rare float64 results that sit exactly half-way between two float32 values."""
    a, b, c = (np.asarray(v, F32).astype(np.float64) for v in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        half = (s.view(np.uint64) & np.uint64((1 << 29) - 1)) == np.uint64(1 << 28)
        fix = half & (err != 0) & np.isfinite(s)
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


def pixel_rays(invproj, xs, ys):
    """invproj * (x + .5, y + .5, 1) and its squared norm as the reference build computes them for pixel_footprint and
    pixel_3dpos (depthmap.cc:139-156): g++ contracts the products into
        rx = fma(m0, vx, fma(m1, vy, m2)), ry = fma(m3, vx, fma(m4, vy, m5)), rz = fma(m7, vy, fma(m6, vx, m8)),
        |r|^2 = fma(rz, rz, rx*rx + ry*ry)."""
    m = np.asarray(invproj, F32).reshape(9)
    vx = np.asarray(xs).astype(F32) + F32(0.5)
    vy = np.asarray(ys).astype(F32) + F32(0.5)
    rx = fma32(m[0], vx, fma32(m[1], vy, m[2]))
    ry = fma32(m[3], vx, fma32(m[4], vy, m[5]))
    rz = fma32(m[7], vy, fma32(m[6], vx, m[8]))
    sq = fma32(rz, rz, rx * rx + ry * ry)
    return rx, ry, rz, sq


def footprints(dm, invproj):
    """pixel_footprint of every pixel: invproj[0] * depth / |ray| (a true division in the reference build)."""
    dm = np.asarray(dm, F32)
    h, w = dm.shape
    ys, xs = np.mgrid[0:h, 0:w]
    _, _, _, sq = pixel_rays(invproj, xs, ys)
    with np.errstate(invalid="ignore", over="ignore"):
        return (F32(np.asarray(invproj, F32).reshape(9)[0]) * dm) / np.sqrt(sq)


def diagonal_factor(dd_factor):
    """`dd_factor *= MATH_SQRT2` on a float (depthmap.cc:198): the product is formed in double and rounded to float."""
    return F32(float(F32(dd_factor)) * MATH_SQRT2)


def is_depthdisc(depths, widths, dd_factor, i1, i2):
    """dm_is_depthdisc (depthmap.cc:187-205) over arrays of blocks: depths / widths are [4, ...] float32."""
    swap = depths[i2] < depths[i1]
    d_min = np.where(swap, depths[i2], depths[i1])
    d_max = np.where(swap, depths[i1], depths[i2])
    w_min = np.where(swap, widths[i2], widths[i1])
    dd = diagonal_factor(dd_factor) if i1 + i2 == 3 else F32(dd_factor)
    with np.errstate(invalid="ignore", over="ignore"):
        return (d_max - d_min) > (w_min * dd)


def block_triangles(dm, invproj, dd_factor):
    """The triangles each 2x2 block issues (depthmap.cc:226-300): int [H-1, W-1, 2], 1..4 = TRIS row + 1, 0 = none."""
    dm = np.asarray(dm, F32)
    depths = np.stack([dm[:-1, :-1], dm[:-1, 1:], dm[1:, :-1], dm[1:, 1:]])
    valid = depths > 0.0
    mask = sum(valid[j].astype(np.int64) << j for j in range(4))
    with np.errstate(invalid="ignore"):
        smaller_03 = np.abs(depths[0] - depths[3]) < np.abs(depths[1] - depths[2])     # a NaN difference takes the else branch
    tri = np.zeros(mask.shape + (2,), np.int64)
    for m, t in ((7, 1), (11, 2), (13, 3), (14, 4)):
        tri[..., 0][mask == m] = t
    full = mask == 15
    tri[..., 0][full] = np.where(smaller_03, 2, 1)[full]
    tri[..., 1][full] = np.where(smaller_03, 3, 4)[full]
    if F32(dd_factor) > 0.0:
        fp = footprints(dm, invproj)
        widths = np.stack([fp[:-1, :-1], fp[:-1, 1:], fp[1:, :-1], fp[1:, 1:]])
        for t in range(1, 5):
            a, b, c = TRIS[t - 1]
            disc = (is_depthdisc(depths, widths, dd_factor, a, b) | is_depthdisc(depths, widths, dd_factor, b, c)
                    | is_depthdisc(depths, widths, dd_factor, c, a))
            tri[(tri == t) & disc[..., None]] = 0
    return tri


def triangulate(dm, invproj, dd_factor=5.0, color=None, cam_to_world=None):
    """depthmap_triangulate (depthmap.cc:209-372) plus mesh_transform with a 4x4 camera-to-world matrix (mesh_tools.cc:64-78).
    Returns dict(vertex_ids [H, W] uint32, faces [F, 3] uint32, vertices [V, 3] float32 (the reference build's operations),
    vertices64 [V, 3] float64, colors [V, 4] float32 or None, tri [H-1, W-1, 2])."""
    dm = np.asarray(dm, F32)
    h, w = dm.shape
    m = np.asarray(invproj, F32).reshape(9)
    tri = block_triangles(dm, invproj, dd_factor)
    # faces in emission order: blocks in raster order, tri[0] before tri[1], corners as listed in TRIS
    blk, slot = np.nonzero(tri.reshape(-1, 2))
    t = tri.reshape(-1, 2)[blk, slot]
    base = (blk // (w - 1)) * w + blk % (w - 1)
    off = (TRIS % 2) + w * (TRIS // 2)
    face_pix = base[:, None] + off[t - 1]
    # a vertex is numbered when a face references its pixel for the first time (dm_make_triangle, depthmap.cc:160-183)
    pix, first = np.unique(face_pix.ravel(), return_index=True)
    pix = pix[np.argsort(first, kind="stable")]
    vids = np.full(h * w, NO_VERTEX, np.uint32)
    vids[pix] = np.arange(len(pix), dtype=np.uint32)
    faces = vids[face_pix].astype(np.uint32)
    xs, ys = pix % w, pix // w
    d = dm.reshape(-1)[pix]
    # pixel_3dpos: ray.normalized() * depth, which the reference build evaluates as (depth * ray) * (1 / |ray|)
    rx, ry, rz, sq = pixel_rays(m, xs, ys)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        inv = F32(1.0) / np.sqrt(sq)
        verts = np.stack([(d * rx) * inv, (d * ry) * inv, (d * rz) * inv], -1).astype(F32)
    m64 = m.astype(np.float64).reshape(3, 3)
    ray64 = np.stack([xs + 0.5, ys + 0.5, np.ones(len(pix))], -1) @ m64.T
    with np.errstate(invalid="ignore", over="ignore"):
        verts64 = ray64 / np.linalg.norm(ray64, axis=1, keepdims=True) * d.astype(np.float64)[:, None]
    if cam_to_world is not None:
        ctw = np.asarray(cam_to_world, F32).reshape(4, 4)
        with np.errstate(invalid="ignore", over="ignore"):
            verts = np.stack([((verts[:, 0] * ctw[r, 0] + verts[:, 1] * ctw[r, 1]) + verts[:, 2] * ctw[r, 2]) + ctw[r, 3]
                              for r in range(3)], -1).astype(F32)
            verts64 = verts64 @ ctw[:3, :3].astype(np.float64).T + ctw[:3, 3].astype(np.float64)
    colors = None
    if color is not None:
        ci = np.asarray(color, np.uint8).reshape(h * w, -1)
        c = ci[pix].astype(F32)
        rgb = c[:, :3] if ci.shape[1] >= 3 else np.repeat(c[:, :1], 3, 1)      # grey expansion (depthmap.cc:354-363)
        colors = np.concatenate([rgb, np.full((len(pix), 1), 255.0, F32)], 1) / F32(255.0)
    return dict(vertex_ids=vids.reshape(h, w), faces=faces, vertices=verts, vertices64=verts64, colors=colors, tri=tri)


# ---- the per-view attributes of scene2pset ----
def vertex_normals(verts, faces):
    """Angle-weighted pseudo normals of TriangleMesh::recalc_normals (mesh.cc:45-151), in float64 from float32 vertices."""
    v = np.asarray(verts, F32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    ab, bc, ca = b - a, c - b, a - c
    with np.errstate(invalid="ignore", divide="ignore"):
        fn = np.cross(ab, -ca)
        fnl = np.linalg.norm(fn, axis=1)
        keep = fnl != 0.0
        fn = fn / fnl[:, None]
        abl, bcl, cal = (np.linalg.norm(e, axis=1)[:, None] for e in (ab, bc, ca))
        angles = [np.arccos(np.clip(np.sum(p * q, 1), -1.0, 1.0)) for p, q in
                  ((ab / abl, -ca / cal), (-ab / abl, bc / bcl), (ca / cal, -bc / bcl))]
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[keep, k], fn[keep] * angles[k][keep, None])
    ln = np.linalg.norm(n, axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(ln[:, None] > 0, n / ln[:, None], n)


def mesh_info(n_verts, faces):
    """MeshInfo (mesh_info.cc:18-156): vertex class (0 simple, 1 complex, 2 border, 3 unreferenced) and the adjacent vertices
    as an edge list (v, u), both directions, each edge once.

    update_vertex chains the faces around v through their opposite edges (first -> second).  The depth-map mesh is
    consistently oriented and its faces do not overlap in the image, so at a vertex each neighbour starts at most one
    opposite edge and ends at most one: the opposite edges form disjoint paths, or one closed cycle.  The chain started at
    the first face collects exactly its own path or cycle, so a vertex is complex when it has more than one path, simple when
    its edges close (links == faces) and border otherwise.  A vertex's adjacent vertices (chain order or std::set) are then
    all the vertices it shares a face with."""
    f = np.asarray(faces, np.int64)
    v = f.reshape(-1)
    first = f[:, [1, 2, 0]].reshape(-1)
    second = f[:, [2, 0, 1]].reshape(-1)
    key_first = np.sort(v * n_verts + first)
    assert (key_first[1:] != key_first[:-1]).all(), "two faces at a vertex share an opposite edge"
    key_second = v * n_verts + second
    at = np.minimum(np.searchsorted(key_first, key_second), len(key_first) - 1)
    linked = key_first[at] == key_second
    n_faces = np.bincount(v, minlength=n_verts)
    n_links = np.bincount(v[linked], minlength=n_verts)
    cls = np.full(n_verts, 3, np.int64)
    cls[(n_faces > 0) & (n_links == n_faces)] = 0
    cls[(n_faces > 0) & (n_faces - n_links == 1)] = 2
    cls[(n_faces > 0) & (n_faces - n_links > 1)] = 1
    edges = np.sort(np.concatenate([key_first, key_second]))
    edges = edges[np.concatenate([[True], edges[1:] != edges[:-1]])]
    return cls, np.stack([edges // n_verts, edges % n_verts], -1)


def border_rings(n_verts, faces, info=None):
    """Edge hops from the nearest border vertex (inf where no border vertex is connected): the rings that
    depthmap_mesh_confidences grows one per iteration (depthmap.cc:523-544)."""
    cls, edges = mesh_info(n_verts, faces) if info is None else info
    border = np.flatnonzero(cls == 2)
    if len(border) == 0:
        return np.full(n_verts, np.inf)
    g = scipy.sparse.csr_matrix((np.ones(len(edges)), (edges[:, 0], edges[:, 1])), shape=(n_verts, n_verts))
    return scipy.sparse.csgraph.dijkstra(g, directed=True, indices=border, unweighted=True, min_only=True)


def confidences(n_verts, faces, iterations, rings=None):
    """depthmap_mesh_confidences (depthmap.cc:496-545): a vertex `current` rings away from a border vertex gets
    current / iterations, a vertex no ring below `iterations` reaches keeps 1.0 - for any iterations >= 1.  The reference
    build hoists the division out of the loop (-freciprocal-math): current * (1.0f / iterations), e.g. 3/7 -> 0.42857146."""
    rings = border_rings(n_verts, faces) if rings is None else rings
    conf = np.ones(n_verts, F32)
    near = rings < iterations
    conf[near] = rings[near].astype(F32) * (F32(1.0) / F32(iterations))
    return conf


def scales(verts, faces, scale_factor, info=None):
    """scene2pset.cc:345-357: mean distance to the adjacent vertices of MeshInfo, times scale_factor, in float64."""
    v = np.asarray(verts, F32).astype(np.float64)
    _, edges = mesh_info(len(v), faces) if info is None else info
    dist = np.linalg.norm(v[edges[:, 0]] - v[edges[:, 1]], axis=1)
    total = np.bincount(edges[:, 0], weights=dist, minlength=len(v))
    count = np.bincount(edges[:, 0], minlength=len(v))
    with np.errstate(invalid="ignore", divide="ignore"):
        return total / count * float(F32(scale_factor))


def pointset(dm, invproj, dd_factor=5.0, color=None, cam_to_world=None, conf_iterations=4, scale_factor=2.5):
    """The per-view work of scene2pset: triangulate(...) plus normals [V, 3], vertex classes, border rings, confidences [V]
    float32 (None when conf_iterations is 0) and scales [V], all float64 except the confidences."""
    r = triangulate(dm, invproj, dd_factor, color, cam_to_world)
    nv = len(r["vertices"])
    info = mesh_info(nv, r["faces"])
    r["normals"] = vertex_normals(r["vertices"], r["faces"])
    r["classes"] = info[0]
    r["rings"] = border_rings(nv, r["faces"], info)
    r["confidences"] = confidences(nv, r["faces"], conf_iterations, r["rings"]) if conf_iterations > 0 else None
    r["scales"] = scales(r["vertices"], r["faces"], scale_factor, info)
    return r
