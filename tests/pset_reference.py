"""NumPy restatement of the scene-level filters of apps/scene2pset (scene2pset.cc:284-464), with every decision in the
float32 arithmetic the reference build (-O3 -march=x86-64-v3 -funsafe-math-optimizations) emits, read from the
disassembly of its scene2pset.o and camera.o.  Also the helpers the point-set tests share: an MVE scene directory with
depth maps, colour images and masks, the PLY reader and the runs of the reference app and the drop-in CLI.

tests/test_scene_pointset_reference.py pins this module to the reference binary (oracle/_ref/scene2pset);
tests/test_gpu_scene_pointset.py holds the device to it."""
import os
import re
import subprocess

import numpy as np

from tests import dm_reference as R
from tests.util import ROOT, golden_ref, golden_scene

F32 = np.float32
REF_APP = os.path.join(ROOT, "oracle", "_ref", "scene2pset")
CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "scene2pset_b200")


# ---- the reference build's arithmetic ----
def fill_fraction(dm):
    """scene2pset.cc:284-291.  `num_recon += 1.0f` is vectorised over eight float lanes: element j < 8*(n // 8) feeds lane
    j % 8, each lane saturating at 2^24; the lanes reduce as ((a0+a4) + (a2+a6)) + ((a1+a5) + (a3+a7)).  A remainder of 4
    or more goes through one 4-lane step c_k = b_k + (a_k + a_k+4) reduced as (c0+c2) + (c1+c3); the last 0-3 elements add
    1.0f one at a time.  fraction = sum / float(n), a true division."""
    d = np.asarray(dm, F32).reshape(-1)
    n = d.size
    n8 = n & ~7
    filled = d > 0.0
    lanes = np.bincount(np.arange(n8) % 8, weights=filled[:n8], minlength=8).astype(np.int64)
    a = np.minimum(lanes, 1 << 24).astype(F32)
    v = a[:4] + a[4:]
    j = n8
    if n - n8 >= 4:
        c = filled[n8:n8 + 4].astype(F32) + v
        s = (c[0] + c[2]) + (c[1] + c[3])
        j += 4
    else:
        s = (v[0] + v[2]) + (v[1] + v[3])
    for k in range(j, n):
        if filled[k]:
            s = F32(s + F32(1.0))
    return F32(s / F32(n))


def aabb_keep(verts, lo, hi):
    """math::geom::point_box_overlap (octree_tools.h:356-364): both faces inclusive, NaN inside."""
    v = np.asarray(verts, F32)
    lo, hi = np.asarray(lo, F32), np.asarray(hi, F32)
    with np.errstate(invalid="ignore"):
        return ~((v < lo) | (v > hi)).any(-1)


def calibration(cam, width, height):
    """CameraInfo::fill_calibration (camera.cc:125-144) as the reference build computes it (no contraction there)."""
    w, h = F32(width), F32(height)
    flen, pa = F32(cam["flen"]), F32(cam["paspect"])
    pp = np.asarray(cam["ppoint"], F32)
    if (w / h) * pa < F32(1.0):
        ay = flen * h
        ax = ay / pa
    else:
        ax = flen * w
        ay = ax * pa
    return np.array([ax, 0, w * pp[0], 0, ay, h * pp[1], 0, 0, 1], F32)


def world_to_cam(cam):
    """CameraInfo::fill_world_to_cam (camera.cc:61-67), rows 0-2."""
    r, t = np.asarray(cam["rot"], F32).reshape(3, 3), np.asarray(cam["trans"], F32)
    return np.concatenate([r, t[:, None]], 1).reshape(12)


def project(verts, cam, width, height):
    """scene2pset.cc:445-447 with the reference build's contractions:
        c_r = fma(z, W[r][2], fma(x, W[r][0], y * W[r][1])) + W[r][3]
        p0 = fma(c2, K2, fma(K0, c0, c1 * K1)), p1 = fma(c2, K5, fma(K3, c0, c1 * K4)), p2 = fma(c2, K8, fma(c0, K6, c1 * K7))
        x = p0 / p2, y = p1 / p2."""
    v = np.asarray(verts, F32)
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    W = world_to_cam(cam)
    K = calibration(cam, width, height)
    fma = R.fma32
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        c = [fma(z, W[4 * r + 2], fma(x, W[4 * r], y * W[4 * r + 1])) + W[4 * r + 3] for r in range(3)]
        p0 = fma(c[2], K[2], fma(K[0], c[0], c[1] * K[1]))
        p1 = fma(c[2], K[5], fma(K[3], c[0], c[1] * K[4]))
        p2 = fma(c[2], K[8], fma(c[0], K[6], c[1] * K[7]))
        return p0 / p2, p1 / p2


def mask_deleted(verts, masks):
    """scene2pset.cc:407-458: masks = [(mask [H, W] uint8, camera)].  A point is deleted when any mask it projects inside
    of (x >= 0, y >= 0, x < W, y < H) is 0 at (int(x), int(y)).  NaN projections count as outside."""
    v = np.asarray(verts, F32)
    dele = np.zeros(len(v), bool)
    for m, cam in masks:
        h, w = m.shape
        px, py = project(v, cam, w, h)
        with np.errstate(invalid="ignore"):
            inside = (px >= 0) & (py >= 0) & (px < F32(w)) & (py < F32(h))
        ix = np.where(inside, px, 0).astype(np.int64)
        iy = np.where(inside, py, 0).astype(np.int64)
        dele |= inside & (m[iy, ix] == 0)
    return dele


def edge_distance(verts, masks):
    """Per point, the smallest distance in pixels (over the masks it projects into) from its projection to a pixel edge;
    used to explain decisions that differ between two nearly equal vertices."""
    v = np.asarray(verts, F32)
    best = np.full(len(v), np.inf)
    for m, cam in masks:
        h, w = m.shape
        px, py = (a.astype(np.float64) for a in project(v, cam, w, h))
        with np.errstate(invalid="ignore"):
            inside = (px >= -1) & (py >= -1) & (px < w + 1) & (py < h + 1)
            d = np.minimum(np.abs(px - np.round(px)), np.abs(py - np.round(py)))
        best = np.where(inside, np.minimum(best, d), best)
    return best


def correspondence_csv(vertex_ids_per_view):
    """scene2pset.cc:64-118 from the vertex-id images [(view_id, vertex_ids [H, W])]: (data, metadata) CSV texts."""
    data, meta, first = ["x, y\n"], ["View_ID, Width, Height, First_Vertex_Index\n"], 0
    for vid, ids in vertex_ids_per_view:
        h, w = ids.shape
        meta.append("%d, %d, %d, %d\n" % (vid, w, h, first))
        flat = ids.reshape(-1)
        pix = np.flatnonzero(flat != R.NO_VERTEX)
        order = np.argsort(flat[pix], kind="stable")
        pix = pix[order]
        data.extend("%d, %d\n" % (p % w, p // w) for p in pix)
        first += len(pix)
    return "".join(data), "".join(meta)


# ---- scene directories ----
def camera_of(s, v):
    return dict(flen=float(s.flen[v]), paspect=float(s.paspect[v]), ppoint=np.asarray(s.ppoint[v], F32),
                rot=np.asarray(s.rot[v], F32), trans=np.asarray(s.trans[v], F32))


def hand_map(h, w, base, seed):
    """A smooth hand-made depth map around `base` with a step and holes."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    d = (base * (1.0 + 0.05 * np.sin(xx / 9.0) + 0.04 * np.cos(yy / 7.0))).astype(F32)
    d[(xx > 0.55 * w) & (yy < 0.4 * h)] *= F32(1.08)
    d[rng.random((h, w)) < 0.04] = 0.0
    d[:, :2] = 0.0
    return d


def make_mask(h, w, seed, cam=None):
    """255 with zero regions: a slanted band, a disc and random blocks, so the zero regions cut through the points."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    m = np.full((h, w), 255, np.uint8)
    m[(xx / w + 0.6 * yy / h) < 0.3 + 0.1 * rng.random()] = 0
    cx, cy, r = w * (0.4 + 0.3 * rng.random()), h * (0.4 + 0.3 * rng.random()), 0.12 * min(w, h)
    m[(xx - cx) ** 2 + (yy - cy) ** 2 < r * r] = 0
    for _ in range(6):
        bx, by = rng.integers(0, w), rng.integers(0, h)
        m[by:by + max(1, h // 20), bx:bx + max(1, w // 15)] = 0
    return m


SCENES = ("T0", "T5", "T6")


def build_scene(tmp, name, hand_views=(), mask_kinds=None, drop_color=(), extra_maps=None):
    """Writes golden scene `name` as an MVE scene directory with the reference dmrecon's depth maps (golden fixtures) under
    depth-L<scale>, hand-made maps for `hand_views`, colour images of the map's size (undistorted, or undist-L<s> as MVEI
    for scale > 0: the oracle libmve has no PNG support and reads only MVEI), and masks per view:
    mask_kinds[v] in {"same", "double", "odd", "rgb", "zero"} (absent: no mask; "zero": all background).  Returns dict(scene, maps {v: depth}, masks
    {v: mask}, views in view order)."""
    from mve_b200 import synth
    s = golden_scene(name)
    ref = golden_ref(name)
    synth.write_mve_scene(s, tmp)
    maps = {int(k.split("_")[1]): np.ascontiguousarray(ref[k], F32) for k in ref.files if k.startswith("depth_")}
    dw, dh = next(iter(maps.values())).shape[::-1]
    for i, v in enumerate(hand_views):
        base = float(np.median(next(iter(maps.values()))[next(iter(maps.values())) > 0]))
        maps[v] = hand_map(dh, dw, base, seed=100 + i)
    for v, d in (extra_maps or {}).items():
        maps[v] = np.ascontiguousarray(d, F32)
    masks = {}
    for v in range(s.n_views):
        vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
        if v in maps:
            synth.write_mvei(os.path.join(vd, "depth-L%d.mvei" % s.scale), maps[v])
            if s.scale:
                img = ref["undist_%d" % v] if ("undist_%d" % v) in ref.files else None
                if img is None or img.shape[:2] != maps[v].shape:
                    img = np.random.default_rng(v).integers(0, 255, size=maps[v].shape + (3,), dtype=np.uint8)
                synth.write_mvei(os.path.join(vd, "undist-L%d.mvei" % s.scale), np.ascontiguousarray(img[:, :, :3], np.uint8))
        if v in drop_color:
            for f in os.listdir(vd):
                if f.startswith("undist"):
                    os.remove(os.path.join(vd, f))
        kind = (mask_kinds or {}).get(v)
        if kind is None:
            continue
        h, w = s.size(v)[1], s.size(v)[0]
        if s.scale:
            h, w = maps[v].shape if v in maps else (dh, dw)
        if kind == "double":
            h, w = 2 * h, 2 * w
        elif kind == "odd":
            h, w = h * 3 // 4 + 1, w * 5 // 4 + 3
        m = np.zeros((h, w), np.uint8) if kind == "zero" else make_mask(h, w, seed=v)
        if kind == "rgb":
            m = np.repeat(m[:, :, None], 3, 2)
        synth.write_mvei(os.path.join(vd, "mask.mvei"), m)
        masks[v] = m
    return dict(scene=s, maps=maps, masks=masks)


# ---- running the apps and reading their outputs ----
def run(exe, args, scene_dir, out, threads=1, env=None):
    e = dict(os.environ, OMP_NUM_THREADS=str(threads))
    e.update(env or {})
    r = subprocess.run([exe] + list(args) + [scene_dir, out], capture_output=True, text=True, timeout=1200, env=e)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def num_filtered(stdout):
    m = re.findall(r"Filtered a total of (\d+) points", stdout)
    return int(m[-1]) if m else None


def skipped_views(stdout):
    return re.findall(r"View (\S+): Fill status ([0-9.]+)%, skipping", stdout)


def processed_views(stdout):
    return re.findall(r'Processing view "([^"]+)"', stdout)


_PLY_TYPES = {"float": "<f4", "uchar": "u1", "int": "<i4", "uint": "<u4", "double": "<f8"}


def read_ply(path):
    """Binary little-endian point PLY of mve::geom::save_ply_mesh: (header text, structured vertex array)."""
    raw = open(path, "rb").read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    head = raw[:end].decode("ascii")
    n = int(re.search(r"element vertex (\d+)", head).group(1))
    props = re.findall(r"property (\w+) (\w+)", head.split("element vertex")[1].split("element")[0])
    dt = np.dtype([(name, _PLY_TYPES[t]) for t, name in props])
    return head, np.frombuffer(raw[end:end + n * dt.itemsize], dt)


def xyz(v):
    return np.stack([v["x"], v["y"], v["z"]], -1)
