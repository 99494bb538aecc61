"""Deterministic synthetic multi-view scenes for the dmrecon hot path.

The reference ships no sample scene and no dmrecon fixture (SURVEY.md §4), so
every workload named in BASELINE.json ("synthetic N-view WxH scene") is made
here.  A scene is exactly what `mvs::DMRecon` consumes through `mve::Scene`:

* per view an `undistorted` uint8 RGB image and an `mve::CameraInfo`
  (flen, paspect, ppoint, rot (row-major world->cam), trans) -
  libs/mve/camera.h:23-170, written to `meta.ini` as libs/mve/view.cc:594-621
  reads it;
* a bundle of SfM features (position + the ids of the views that see it) in the
  "drews 1.0" text layout parsed at libs/mve/bundle_io.cc:282-393.

Images are rendered analytically (ray / surface intersection per pixel centre,
solid procedural texture evaluated at the hit point) so every view is exact and
consistent.  Rendering uses torch so that it runs on CPU here and on the GPU in
bench.py; all quantities handed to the reconstruction are float32 / uint8 numpy.
"""
from __future__ import annotations

import dataclasses
import os
import struct
from typing import Dict, List, Optional

import numpy as np
import torch

MVEI_SIGNATURE = b"\x89MVE_IMAGE\n"  # libs/mve/image_io.cc:45-46
MVEI_TYPE_UINT8 = 1                  # libs/mve/image_base.h:27-43
MVEI_TYPE_FLOAT = 9


@dataclasses.dataclass
class Scene:
    name: str
    width: int
    height: int
    images: List[np.ndarray]          # [H, W, 3] uint8 per view
    flen: np.ndarray                  # [V] float32
    paspect: np.ndarray               # [V] float32
    ppoint: np.ndarray                # [V, 2] float32
    rot: np.ndarray                   # [V, 9] float32, row-major world->cam
    trans: np.ndarray                 # [V, 3] float32
    feat_pos: np.ndarray              # [F, 3] float32
    feat_refs: List[np.ndarray]       # per feature: int32 view ids
    scale: int                        # dmrecon scale (pyramid level of the ref view)
    nr_recon_neighbors: int = 4
    meta: Dict = dataclasses.field(default_factory=dict)
    sizes: Optional[np.ndarray] = None  # [V, 2] int (width, height) per view; None: every view is width x height

    @property
    def n_views(self) -> int:
        return len(self.images)

    def size(self, v: int):
        """(width, height) of view v's image."""
        if self.sizes is None:
            return self.width, self.height
        return int(self.sizes[v, 0]), int(self.sizes[v, 1])


# ----------------------------------------------------------------------------
# configs (BASELINE.json "configs", SURVEY.md §8d)
# ----------------------------------------------------------------------------
CONFIGS: Dict[str, Dict] = {
    # C1: 4 views + default nrReconNeighbors=4 can never succeed (SURVEY §8a quirks: the
    # local selection must find EXACTLY nrReconNeighbors views) -> run with 3.
    "C1": dict(seed=1, views=4, width=640, height=480, layout="grid", grid=(2, 2), pitch=0.9,
               surface="plane", features=800, scale=2, nr_recon_neighbors=3),
    "C2": dict(seed=2, views=16, width=1920, height=1080, layout="grid", grid=(4, 4), pitch=0.8,
               surface="bumps", features=4000, scale=1),
    "C3": dict(seed=3, views=64, width=1920, height=1080, layout="grid", grid=(8, 8), pitch=0.6,
               surface="bumps", features=8000, scale=0),
    "C4": dict(seed=4, views=32, width=4096, height=3072, layout="grid", grid=(8, 4), pitch=0.6,
               surface="bumps", features=8000, scale=0),
    "C5": dict(seed=5, views=128, width=1280, height=960, layout="orbit",
               surface="sphere", features=16000, scale=0),
    # small cases for tests (oracle finishes in seconds)
    "T0": dict(seed=11, views=6, width=160, height=120, layout="grid", grid=(3, 2), pitch=0.8,
               surface="bumps", features=300, scale=0),
    "T1": dict(seed=12, views=9, width=320, height=240, layout="grid", grid=(3, 3), pitch=0.8,
               surface="bumps", features=600, scale=1),
    "T2": dict(seed=13, views=12, width=160, height=120, layout="orbit", surface="sphere",
               features=800, scale=0, orbit_views_per_ring=6),
    # odd image dimensions at every pyramid level: exercises the principal-point correction of image_pyramid.cc:39-44
    "T4": dict(seed=15, views=6, width=161, height=121, layout="grid", grid=(3, 2), pitch=0.8,
               surface="bumps", features=300, scale=1),
    # many candidates: global view selection must pick 20 of 39 (images are tiny, they do not matter for it)
    "T3": dict(seed=14, views=40, width=96, height=72, layout="grid", grid=(10, 4), pitch=0.45,
               surface="bumps", features=1500, scale=0),
    # general pinhole cameras at scale 0: portrait 101x135 (odd sizes), non-square pixels, off-centre principal points and rolls;
    # view 2 is wide (flen 0.4: its footprint is 2.5x the others', so the local selection's resolution penalty fires) and
    # views 5 and 6 are zoomed (flen 3 and 4.5: sampled at pyramid levels 1 and 2)
    "T5": dict(seed=16, views=8, width=101, height=135, layout="grid", grid=(4, 2), pitch=0.8,
               surface="bumps", features=400, scale=0,
               flen=[1.0, 1.0, 0.4, 1.0, 1.0, 3.0, 4.5, 1.0], paspect=[0.95, 1.08, 0.92, 1.04, 0.97, 0.9, 1.1, 1.02],
               ppoint=[(0.45, 0.55), (0.56, 0.43), (0.5, 0.5), (0.42, 0.58), (0.52, 0.49), (0.58, 0.46), (0.47, 0.52),
                       (0.5, 0.44)],
               roll=[0.0, 20.0, -15.0, 10.0, -8.0, -20.0, 5.0, 14.0]),
    # scale 1 with views of different sizes: the five 179x180 views at paspect 1.003 are portrait at level 0 and
    # landscape at level 1 (90x90); the five crops (118x58 and 58x118: 2 pyramid levels each) at 4.5x to 8.5x the wide
    # views' ax ask for level 2 or 3 at scale 1, past their last level, so the level is clamped
    "T6": dict(seed=17, views=10, width=179, height=180, layout="grid", grid=(5, 2), pitch=0.8,
               surface="bumps", features=600, scale=1,
               flen=[1.0, 3.4, 1.0, 4.0, 1.0, 6.5, 1.0, 3.4, 1.0, 4.0],
               paspect=[1.003, 1.0, 1.003, 1.0, 1.003, 1.0, 1.003, 1.0, 1.003, 1.0],
               ppoint=[(0.48, 0.53), (0.5, 0.5), (0.53, 0.47), (0.5, 0.5), (0.46, 0.5), (0.5, 0.5), (0.5, 0.52),
                       (0.5, 0.5), (0.51, 0.49), (0.5, 0.5)],
               sizes=[None, (118, 58), None, (58, 118), None, (118, 58), None, (58, 118), None, (118, 58)]),
}


def fill_calibration(flen, paspect, ppoint, width, height, dtype=np.float64):
    """CameraInfo::fill_calibration and fill_inverse_calibration (libs/mve/camera.cc:125-144,180-200), both branches,
    evaluated in `dtype`: (K, K^-1, portrait) of a width x height image whose principal point `ppoint` is given as
    fractions of the size."""
    f = np.dtype(dtype).type
    flen, paspect, width, height = f(flen), f(paspect), f(width), f(height)
    ppx, ppy = f(ppoint[0]), f(ppoint[1])
    portrait = bool(width / height * paspect < f(1))
    if portrait:
        ax, ay = flen * height / paspect, flen * height
    else:
        ax, ay = flen * width, flen * width * paspect
    K = np.array([[ax, 0, width * ppx], [0, ay, height * ppy], [0, 0, 1]], dtype)
    Ki = np.array([[f(1) / ax, 0, -width * ppx / ax], [0, f(1) / ay, -height * ppy / ay], [0, 0, 1]], dtype)
    return K, Ki, portrait


def _per_view(cfg, key, default, V):
    vals = cfg.get(key)
    if vals is None:
        return [default] * V
    assert len(vals) == V, key
    return [default if x is None else x for x in vals]


class _Texture:
    """Solid procedural texture: 36 random-phase 3-D sinusoids (6 octaves x 6
    directions) mixed into 3 channels; output sRGB code values in [25, 230] so a
    5x5 master patch mean stays inside (0.01, 0.99) (patch_sampler.cc:325)."""

    def __init__(self, rng: np.random.Generator, lambda_min: float):
        n_oct, n_dir = 6, 6
        omega, amp = [], []
        for o in range(n_oct):
            lam = lambda_min * (2.0 ** o)
            for _ in range(n_dir):
                ang = rng.uniform(0.0, 2.0 * np.pi)
                # mostly in-plane direction with a mild z component
                d = np.array([np.cos(ang), np.sin(ang), rng.uniform(-0.3, 0.3)])
                d /= np.linalg.norm(d)
                omega.append(2.0 * np.pi / lam * d)
                amp.append(1.15 ** o)
        self.omega = np.asarray(omega, dtype=np.float64)          # [36, 3]
        self.phase = rng.uniform(0.0, 2.0 * np.pi, size=len(omega))
        mix = rng.normal(size=(len(omega), 3)) * np.asarray(amp)[:, None]
        # normalise so that sum |mix| per channel == 1  ->  value in [-1, 1]
        self.mix = mix / np.abs(mix).sum(axis=0, keepdims=True)

    def __call__(self, pts: torch.Tensor) -> torch.Tensor:
        """pts [..., 3] float64 -> uint8 [..., 3]."""
        om = torch.as_tensor(self.omega, dtype=pts.dtype, device=pts.device)
        ph = torch.as_tensor(self.phase, dtype=pts.dtype, device=pts.device)
        mx = torch.as_tensor(self.mix, dtype=pts.dtype, device=pts.device)
        out = torch.zeros(pts.shape[:-1] + (3,), dtype=pts.dtype, device=pts.device)
        for k in range(om.shape[0]):
            s = torch.sin(pts[..., 0] * om[k, 0] + pts[..., 1] * om[k, 1] + pts[..., 2] * om[k, 2] + ph[k])
            out += s[..., None] * mx[k]
        # typical |value| << 1; stretch then clamp into [25, 230]
        val = 127.5 + out * 3.0 * 102.5
        return val.clamp(25.0, 230.0).round().to(torch.uint8)


class _Surface:
    def __init__(self, kind: str, rng: np.random.Generator):
        self.kind = kind
        if kind == "bumps":
            self.bumps = [(-0.6, 0.3, 0.3, 0.7), (0.8, -0.4, 0.3, 0.9)]  # cx, cy, height, sigma
        elif kind == "plane":
            self.bumps = []
        elif kind == "sphere":
            self.radius = 1.5
        else:
            raise ValueError(kind)

    # height field z = h(x, y), cameras sit at negative z looking towards +z
    def height(self, x, y):
        z = torch.zeros_like(x)
        for cx, cy, hh, sg in self.bumps:
            z = z - hh * torch.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2.0 * sg * sg))
        return z

    def intersect(self, cpos: torch.Tensor, dirs: torch.Tensor):
        """cpos [3], dirs [..., 3] unit -> (hit points [..., 3], valid mask)."""
        if self.kind == "sphere":
            b = (dirs * cpos).sum(-1)
            c = (cpos * cpos).sum() - self.radius ** 2
            disc = b * b - c
            valid = disc > 0
            s = -b - torch.sqrt(disc.clamp_min(0.0))
            pts = cpos + s[..., None] * dirs
            return pts, valid & (s > 0)
        s = (0.0 - cpos[2]) / dirs[..., 2]
        for _ in range(40 if self.bumps else 1):
            x = cpos[0] + s * dirs[..., 0]
            y = cpos[1] + s * dirs[..., 1]
            s = (self.height(x, y) - cpos[2]) / dirs[..., 2]
        pts = cpos + s[..., None] * dirs
        return pts, s > 0


def _look_at(cpos: np.ndarray, target: np.ndarray, down=np.array([0.0, 1.0, 0.0])) -> np.ndarray:
    f = target - cpos
    f = f / np.linalg.norm(f)
    r = np.cross(down, f)
    r = r / np.linalg.norm(r)
    d = np.cross(f, r)
    return np.stack([r, d, f])  # rows: camera x (right), y (down), z (forward)


def _cast_rays(surf: _Surface, rot, trans, calib, Wv: int, Hv: int, dev):
    """The surface points under the pixel centres of a Wv x Hv image of the camera (rot, trans) with calibration
    (ax, ay, cx, cy) at that size: (points [Hv, Wv, 3], where the ray hits the surface [Hv, Wv])."""
    ax, ay, cx, cy = calib
    ys, xs = torch.meshgrid(torch.arange(Hv, dtype=torch.float64, device=dev),
                            torch.arange(Wv, dtype=torch.float64, device=dev), indexing="ij")
    R = torch.as_tensor(np.asarray(rot).astype(np.float64).reshape(3, 3), device=dev)
    C = -(R.T @ torch.as_tensor(np.asarray(trans).astype(np.float64), device=dev))
    # pixel centre (x+.5, y+.5) -> camera ray K^-1 (x+.5, y+.5, 1) (libs/mve/depthmap.cc:149-156)
    dc = torch.stack([(xs + 0.5 - cx) / ax, (ys + 0.5 - cy) / ay, torch.ones_like(xs)], -1)
    dw = dc @ R  # R^T d, row-vector form
    dw = dw / dw.norm(dim=-1, keepdim=True)
    return surf.intersect(C, dw)


def silhouette(scene: Scene, v: int, width: Optional[int] = None, height: Optional[int] = None,
               device: Optional[str] = None) -> np.ndarray:
    """Object mask of view v as a segmentation would give it: a height x width uint8 image (default: the view's size),
    255 where the ray through the pixel centre hits the scene's surface and 0 elsewhere - the `valid` of make_scene's
    render, at any size.  For a height field every ray hits; for the sphere of the orbit scenes the background is 0."""
    kind = scene.meta.get("surface") or CONFIGS[scene.name]["surface"]
    Wv, Hv = scene.size(v)
    w, h = width or Wv, height or Hv
    calib = fill_calibration(scene.flen[v], scene.paspect[v], scene.ppoint[v], w, h)[0][[0, 1, 0, 1], [0, 1, 2, 2]]
    _, valid = _cast_rays(_Surface(kind, None), scene.rot[v], scene.trans[v], calib, w, h, torch.device(device or "cpu"))
    return valid.cpu().numpy().astype(np.uint8) * 255


def depth(scene: Scene, v: int, width: Optional[int] = None, height: Optional[int] = None,
          device: Optional[str] = None) -> np.ndarray:
    """Analytic depth map of view v: a height x width float32 image (default: the view's size) holding, under each pixel
    centre, the distance from the camera centre to the scene's surface along the pixel's unit ray - MVE's depth
    convention, as in depth-L<s> - and 0 where the ray misses the surface."""
    kind = scene.meta.get("surface") or CONFIGS[scene.name]["surface"]
    Wv, Hv = scene.size(v)
    w, h = width or Wv, height or Hv
    calib = fill_calibration(scene.flen[v], scene.paspect[v], scene.ppoint[v], w, h)[0][[0, 1, 0, 1], [0, 1, 2, 2]]
    dev = torch.device(device or "cpu")
    pts, valid = _cast_rays(_Surface(kind, None), scene.rot[v], scene.trans[v], calib, w, h, dev)
    R = torch.as_tensor(np.asarray(scene.rot[v]).astype(np.float64).reshape(3, 3), device=dev)
    C = -(R.T @ torch.as_tensor(np.asarray(scene.trans[v]).astype(np.float64), device=dev))
    d = torch.where(valid, (pts - C).norm(dim=-1), torch.zeros((), dtype=torch.float64, device=dev))
    return d.cpu().numpy().astype(np.float32)


def monocular(scene: Scene, v: int, width: int, height: int, seed: int = 0, noise: float = 0.02,
              outliers: float = 0.05) -> np.ndarray:
    """A synthetic monocular prior of view v, as a relative inverse-depth network gives one: the planar disparity 1/z of
    depth() at width x height under a seeded affine transform d = a / z + b (a in [0.5, 2], b in [0, 0.2]), with
    multiplicative Gaussian noise of relative size `noise` and discs of random values over about `outliers` of the
    pixels.  Where the ray misses the surface the map holds b / 2, a disparity beyond infinity, as a network's sky.
    Float32, for Scene.set_view_prior_relative(kind="disparity")."""
    rng = np.random.default_rng([seed, v])
    Wv, Hv = scene.size(v)
    K = fill_calibration(scene.flen[v], scene.paspect[v], scene.ppoint[v], Wv, Hv, np.float32)[0].astype(np.float64)
    ray = depth(scene, v, width, height).astype(np.float64)
    a = ((np.arange(width) + 0.5) * Wv / width - K[0, 2]) / K[0, 0]
    b = ((np.arange(height) + 0.5) * Hv / height - K[1, 2]) / K[1, 1]
    z = ray / np.sqrt(a[None, :] ** 2 + b[:, None] ** 2 + 1.0)
    scale, shift = rng.uniform(0.5, 2.0), rng.uniform(0.0, 0.2)
    with np.errstate(divide="ignore"):
        d = np.where(z > 0, scale / np.where(z > 0, z, 1.0) + shift, shift / 2)
    d *= 1.0 + noise * rng.standard_normal(d.shape)
    yy, xx = np.mgrid[0:height, 0:width]
    covered, lo, hi = np.zeros(d.shape, bool), float(d.min()), float(d.max())
    while covered.mean() < outliers:
        r = rng.uniform(1.0, max(2.0, 0.03 * max(width, height)))
        cx, cy = rng.uniform(0, width), rng.uniform(0, height)
        disc = (xx - cx) ** 2 + (yy - cy) ** 2 <= r * r
        d[disc] = rng.uniform(lo, hi)
        covered |= disc
    return d.astype(np.float32)


def make_scene(config, device: Optional[str] = None, only_views=None, **overrides) -> Scene:
    """Build a synthetic scene. `config` is a key of CONFIGS or a dict.
    only_views: render only these views' images (the others are None) - used when ranks render their own shard.
    Optional per-view camera keys (lists of length `views`, None entries take the default): flen (1), paspect (1),
    ppoint ((0.5, 0.5)), roll (degrees about the optical axis, 0) and sizes ((width, height))."""
    name = config if isinstance(config, str) else config.get("name", "custom")
    cfg = dict(CONFIGS[config]) if isinstance(config, str) else dict(config)
    cfg.update(overrides)
    dev = torch.device(device or "cpu")
    rng = np.random.default_rng(cfg["seed"])
    W, H, V = cfg["width"], cfg["height"], cfg["views"]
    flen = 1.0
    dist = 5.0
    surf = _Surface(cfg["surface"], rng)
    tex = _Texture(rng, lambda_min=6.0 * dist / (flen * max(W, H)))
    flens = np.asarray(_per_view(cfg, "flen", flen, V), np.float32)
    paspects = np.asarray(_per_view(cfg, "paspect", 1.0, V), np.float32)
    ppoints = np.asarray(_per_view(cfg, "ppoint", (0.5, 0.5), V), np.float32).reshape(V, 2)
    rolls = _per_view(cfg, "roll", 0.0, V)
    sizes = np.asarray(_per_view(cfg, "sizes", (W, H), V), np.int64).reshape(V, 2)

    cams_pos, cams_rot = [], []
    if cfg["layout"] == "grid":
        gx, gy = cfg["grid"]
        assert gx * gy == V
        p = cfg["pitch"]
        # `blocks` > 1 tiles the scene along x with identical gx/blocks x gy camera blocks (weak scaling: every block has
        # the geometry of the single-block scene, view ids are block-major so that rank r owns block r)
        nb = cfg.get("blocks", 1)
        bx = gx // nb
        for b in range(nb):
            for j in range(gy):
                for i in range(bx):
                    lx, ly = (i - (bx - 1) / 2) * p, (j - (gy - 1) / 2) * p        # position inside the block
                    c = np.array([lx + b * bx * p - (nb - 1) * bx * p / 2, ly,
                                  -dist * (1.0 + rng.uniform(-0.07, 0.07))])
                    # converge mildly towards the centre of the camera's own block
                    tgt = np.array([c[0] - 0.65 * lx, c[1] - 0.65 * ly, 0.0])
                    cams_pos.append(c)
                    cams_rot.append(_look_at(c, tgt))
    elif cfg["layout"] == "orbit":
        per_ring = cfg.get("orbit_views_per_ring", V // 2)
        rings = V // per_ring
        for r_i in range(rings):
            hgt = (r_i - (rings - 1) / 2) * 1.6
            for i in range(per_ring):
                a = 2.0 * np.pi * (i + 0.5 * r_i) / per_ring
                rad = dist * (1.0 + rng.uniform(-0.07, 0.07))
                c = np.array([rad * np.cos(a), hgt, rad * np.sin(a)])
                cams_pos.append(c)
                cams_rot.append(_look_at(c, np.zeros(3)))
    else:
        raise ValueError(cfg["layout"])
    for v, deg in enumerate(rolls):
        if deg:
            c, s = np.cos(np.radians(deg)), np.sin(np.radians(deg))
            cams_rot[v] = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]) @ cams_rot[v]

    rot32 = np.asarray(cams_rot, dtype=np.float64).reshape(V, 9).astype(np.float32)
    pos = np.asarray(cams_pos, dtype=np.float64)
    # t = -R C, computed from the float32 rotation so R, t are mutually consistent
    trans32 = np.stack([-(rot32[v].astype(np.float64).reshape(3, 3) @ pos[v]) for v in range(V)]).astype(np.float32)

    images = []
    # (ax, ay, cx, cy) of each view at its own size, from the float32 camera the reconstruction reads
    calib = [fill_calibration(flens[v], paspects[v], ppoints[v], sizes[v, 0], sizes[v, 1])[0][[0, 1, 0, 1], [0, 1, 2, 2]]
             for v in range(V)]
    for v in range(V):
        if only_views is not None and v not in only_views:
            images.append(None)
            continue
        pts, valid = _cast_rays(surf, rot32[v], trans32[v], calib[v], int(sizes[v, 0]), int(sizes[v, 1]), dev)
        img = tex(pts)
        img = torch.where(valid[..., None], img, torch.full_like(img, 128))
        images.append(img.cpu().numpy())

    # SfM features: random surface points + every view whose frustum contains them
    F = cfg["features"]
    if cfg["surface"] == "sphere":
        p = rng.normal(size=(F, 3))
        p = p / np.linalg.norm(p, axis=1, keepdims=True) * surf.radius
        p[:, 1] = np.clip(p[:, 1], -1.2, 1.2)
        p = p / np.linalg.norm(p, axis=1, keepdims=True) * surf.radius
        nrm = p / surf.radius
    else:
        ext = np.abs(pos[:, :2]).max(axis=0) + 0.32 * dist * np.array([1.0, H / W])
        xy = rng.uniform(-1.0, 1.0, size=(F, 2)) * ext
        z = surf.height(torch.as_tensor(xy[:, 0]), torch.as_tensor(xy[:, 1])).numpy()
        p = np.concatenate([xy, z[:, None]], 1)
        nrm = None
    feat_pos = p.astype(np.float32)
    X = feat_pos.astype(np.float64)                                   # [F, 3]
    vis = np.zeros((len(X), V), dtype=bool)
    for v in range(V):
        Rm = rot32[v].astype(np.float64).reshape(3, 3)
        cp = X @ Rm.T + trans32[v].astype(np.float64)                 # [F, 3]
        z = cp[:, 2]
        ax, ay, cx, cy = calib[v]
        Wv, Hv = int(sizes[v, 0]), int(sizes[v, 1])
        with np.errstate(divide="ignore", invalid="ignore"):
            x = ax * cp[:, 0] / z + cx - 0.5
            y = ay * cp[:, 1] / z + cy - 0.5
        ok = (z > 0) & (x >= 1.0) & (x <= Wv - 2) & (y >= 1.0) & (y <= Hv - 2)
        if nrm is not None:
            to_cam = pos[v] - X
            ok &= (np.einsum("ij,ij->i", nrm, to_cam) / np.linalg.norm(to_cam, axis=1)) >= 0.35
        vis[:, v] = ok
    feat_refs = [np.nonzero(vis[f])[0].astype(np.int32) for f in range(len(X))]
    keep = [i for i, r in enumerate(feat_refs) if len(r) >= 2]
    feat_pos = feat_pos[keep]
    feat_refs = [feat_refs[i] for i in keep]

    mixed = bool((sizes != (W, H)).any())
    return Scene(name=name, width=W, height=H, images=images, flen=flens, paspect=paspects, ppoint=ppoints,
                 rot=rot32, trans=trans32, feat_pos=feat_pos, feat_refs=feat_refs, scale=cfg["scale"],
                 nr_recon_neighbors=cfg.get("nr_recon_neighbors", 4), meta=cfg,
                 sizes=sizes.astype(np.int32) if mixed else None)


# ----------------------------------------------------------------------------
# on-disk MVE scene layout (SURVEY.md §8b "On-disk layout that must not change")
# ----------------------------------------------------------------------------
def write_mvei(path: str, arr: np.ndarray) -> None:
    """MVEI = signature + int32 w,h,c,type + raw interleaved data (image_io.cc:1295-1321)."""
    if arr.ndim == 2:
        arr = arr[:, :, None]
    h, w, c = arr.shape
    if arr.dtype == np.uint8:
        t = MVEI_TYPE_UINT8
    elif arr.dtype == np.float32:
        t = MVEI_TYPE_FLOAT
    else:
        raise TypeError(arr.dtype)
    with open(path, "wb") as f:
        f.write(MVEI_SIGNATURE)
        f.write(struct.pack("<4i", w, h, c, t))
        f.write(np.ascontiguousarray(arr).tobytes())


def read_mvei(path: str) -> np.ndarray:
    """Inverse of write_mvei (image_io.cc:1234-1290)."""
    with open(path, "rb") as f:
        sig = f.read(len(MVEI_SIGNATURE))
        if sig != MVEI_SIGNATURE:
            raise ValueError("not an MVEI file: " + path)
        w, h, c, t = struct.unpack("<4i", f.read(16))
        dt = {MVEI_TYPE_UINT8: np.uint8, MVEI_TYPE_FLOAT: np.float32}[t]
        data = np.frombuffer(f.read(), dtype=dt)
    return data.reshape(h, w, c)


def _f32(x) -> str:
    return "%.9g" % float(x)  # round-trips float32 exactly


def write_mve_scene(scene: Scene, path: str) -> None:
    """views/view_%04d.mve/{meta.ini, undistorted.mvei} + synth_0.out (scene.cc:146-176)."""
    os.makedirs(os.path.join(path, "views"), exist_ok=True)
    for v in range(scene.n_views):
        vd = os.path.join(path, "views", "view_%04d.mve" % v)
        os.makedirs(vd, exist_ok=True)
        with open(os.path.join(vd, "meta.ini"), "w") as f:
            f.write("# MVE view meta data is stored in INI-file syntax.\n")
            f.write("# This file is generated, formatting will get lost.\n\n")
            f.write("[camera]\n")
            f.write("focal_length = %s\n" % _f32(scene.flen[v]))
            f.write("pixel_aspect = %s\n" % _f32(scene.paspect[v]))
            f.write("principal_point = %s %s\n" % (_f32(scene.ppoint[v, 0]), _f32(scene.ppoint[v, 1])))
            f.write("rotation = %s\n" % " ".join(_f32(x) for x in scene.rot[v]))
            f.write("translation = %s\n" % " ".join(_f32(x) for x in scene.trans[v]))
            f.write("\n[view]\n")
            f.write("id = %d\n" % v)
            f.write("name = %04d\n" % v)
        write_mvei(os.path.join(vd, "undistorted.mvei"), scene.images[v])
    with open(os.path.join(path, "synth_0.out"), "w") as f:
        f.write("drews 1.0\n")
        f.write("%d %d\n" % (scene.n_views, len(scene.feat_pos)))
        for v in range(scene.n_views):
            f.write("%s 0 0\n" % _f32(scene.flen[v]))
            r = scene.rot[v]
            for k in range(3):
                f.write("%s %s %s\n" % (_f32(r[3 * k]), _f32(r[3 * k + 1]), _f32(r[3 * k + 2])))
            f.write("%s %s %s\n" % tuple(_f32(x) for x in scene.trans[v]))
        for i in range(len(scene.feat_pos)):
            f.write("%s %s %s\n" % tuple(_f32(x) for x in scene.feat_pos[i]))
            f.write("128 128 128\n")
            refs = scene.feat_refs[i]
            f.write("%d" % len(refs))
            for r in refs:
                f.write(" %d 0 0" % int(r))
            f.write("\n")


# ----------------------------------------------------------------------------
# self-contained scene files (used for committed test fixtures)
# ----------------------------------------------------------------------------
def save_scene_npz(scene: Scene, path: str) -> None:
    """Views of one size are stored as one stacked `images` array; views of different sizes as image_<v> each, with the
    nominal width x height beside them."""
    off = np.zeros(len(scene.feat_refs) + 1, np.int32)
    off[1:] = np.cumsum([len(r) for r in scene.feat_refs])
    ids = np.concatenate(scene.feat_refs).astype(np.int32) if scene.feat_refs else np.zeros(0, np.int32)
    if len({im.shape for im in scene.images}) == 1:
        imgs = dict(images=np.stack(scene.images))
    else:
        imgs = {"image_%d" % v: im for v, im in enumerate(scene.images)}
        imgs.update(width=scene.width, height=scene.height)
    np.savez_compressed(path, name=scene.name, flen=scene.flen, paspect=scene.paspect,
                        ppoint=scene.ppoint, rot=scene.rot, trans=scene.trans, feat_pos=scene.feat_pos,
                        feat_off=off, feat_ids=ids, scale=scene.scale, nr_recon_neighbors=scene.nr_recon_neighbors, **imgs)


def load_scene_npz(path: str) -> Scene:
    z = np.load(path, allow_pickle=False)
    off, ids = z["feat_off"], z["feat_ids"]
    refs = [ids[off[i]:off[i + 1]].astype(np.int32) for i in range(len(off) - 1)]
    if "images" in z:
        imgs = list(z["images"])
        W, H, sizes = imgs[0].shape[1], imgs[0].shape[0], None
    else:
        imgs = [z["image_%d" % v] for v in range(len(z["flen"]))]
        W, H = int(z["width"]), int(z["height"])
        sizes = np.asarray([(im.shape[1], im.shape[0]) for im in imgs], np.int32)
    return Scene(name=str(z["name"]), width=W, height=H, images=imgs,
                 flen=z["flen"], paspect=z["paspect"], ppoint=z["ppoint"], rot=z["rot"], trans=z["trans"],
                 feat_pos=z["feat_pos"], feat_refs=refs, scale=int(z["scale"]),
                 nr_recon_neighbors=int(z["nr_recon_neighbors"]), sizes=sizes)
