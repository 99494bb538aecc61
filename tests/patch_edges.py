"""The geometry of one pass of mvs::PatchOptimization restated in float64 (test infrastructure), the edge classes a patch
can fall into and the generator of the inputs that reach them.  Extends tests/camera_reference.py.

  patch_points()   PatchSampler::computePatchPoints (patch_sampler.cc:274-295): the 25 world points of a patch
  project()        SingleView::worldToScreen (single_view.h:188-197): K_l (R X + t) / z - 0.5
  view_state()     the level choice at the centre point (patch_sampler.cc:76-91, camera_reference.level_of) and the 25
                   projections at that level, for one neighbour view
  edge_classes()   which edge classes a batch of PatchOptimization inputs meets at its input state
  make_cases()     inputs built from an execution trace that sit on those edges with a margin far above the device's
                   rounding (tests/golden/make_golden.py, group patch_edges)

A sample is inside a level of width w and height h when 0 < qx < w - 1 and 0 < qy < h - 1 (patch_sampler.cc:113-120); its
signed distance to the border is min(qx, w - 1 - qx, qy, h - 1 - qy), negative outside.  The classes, per (patch, view it
samples at its input state - every global candidate for a seed, its local views otherwise):

  near_edge_in    all 25 samples inside; the smallest distance is in [MARGIN, NEAR]
  one_out_tail    exactly one sample outside, and it is sample 22, 23 or 24 (peeled after the sample loop of PatchT)
  one_out_head    the same with sample 0 or 1 (staged before the loop)
  one_out_mid     the same with any other sample
  padded_right    one of the four above at the right border of a level whose width is not a multiple of 4 (the quad
                  image's row pitch is rounded up to 4 texels, so padding sits next to the last column)
  bottom          one of the four above at the bottom border
  level_switch    the footprint ratio nfp / mfp is within RATIO_NEAR (relative) of a level switch 0.5 * 2^-k, k >= 0
  level_clamped   the requested level is past the view's last one (SingleView::clampLevel)
  master_border   x in {2, W - 3} or y in {2, H - 3} at the reference level: the master patch reads its outermost texels
  master_outside  x in {1, W - 2} or y in {1, H - 2}: the master patch does not fit, the optimisation fails

The margin rule: in the four sample classes every sample of every view the patch samples is at least MARGIN px away from
the border (inside or out), and every footprint ratio is at least RATIO_MARGIN (relative) away from a switch.  MARGIN is
about 30 times the <= 2 ulp by which the device's pixel coordinates differ from the reference's at these image sizes
(DESIGN.md section 3), so no decision at the input state depends on rounding.
"""
import numpy as np

from tests import camera_reference as CR

NS = 25
OFF = np.array([(k % 5 - 2, k // 5 - 2) for k in range(NS)], np.float64)     # (i, j) of sample k, row-major
MARGIN = 1e-3
NEAR = 0.05
RATIO_NEAR = 1e-3
RATIO_MARGIN = 1e-4
SAMPLE_CLASSES = ("near_edge_in", "one_out_tail", "one_out_head", "one_out_mid")
CLASSES = SAMPLE_CLASSES + ("padded_right", "bottom", "level_switch", "level_clamped", "master_border", "master_outside")
DELTAS = (1e-3, -1e-3, 0.01, -0.01, 0.05, -0.05)         # px: the extreme sample's signed distance to the border aimed at
RATIO_DELTAS = (5e-4, -5e-4)                 # relative: the footprint ratio's distance to the switch aimed at


def _pose(scene, v, dtype):
    R = np.asarray(scene.rot[v], np.float32).reshape(3, 3).astype(dtype)
    t = np.asarray(scene.trans[v], np.float32).astype(dtype)
    return R, t


def patch_points(scene, ref, scale, x, y, depth, dzI, dzJ, dtype=np.float64):
    """[N, 25, 3] world points: C + (depth + i dzI + j dzJ) R^T r / |r| with r = K^-1 (x + i + .5, y + j + .5, 1) at
    level `scale` of view `ref` (viewRayScaled, single_view.cc:99-106; the same as u / |u| with u = R^T r up to how far
    the float32 rotation is from orthonormal)."""
    f = np.dtype(dtype).type
    Ki = CR.view_levels(scene, ref, dtype)[scale][3]
    R, t = _pose(scene, ref, dtype)
    C = -(R.T @ t)
    col = lambda a: np.asarray(a).astype(dtype).reshape(-1, 1)      # noqa: E731
    off = OFF.astype(dtype)
    px = np.stack(np.broadcast_arrays(col(x) + off[:, 0] + f(0.5), col(y) + off[:, 1] + f(0.5), np.ones(NS, dtype)), -1)
    u = px @ Ki.T
    u = (u / np.sqrt((u * u).sum(-1, keepdims=True))) @ R      # normalised before the rotation, like pixel_3dpos
    tt = col(depth) + off[:, 0] * col(dzI) + off[:, 1] * col(dzJ)
    return C + tt[..., None] * u


def project(scene, v, level, X, dtype=np.float64):
    """[N, K, 2] screen positions of the points X [N, K, 3] in view v at the pyramid level `level` (scalar or [N])."""
    Ks = np.stack([lv[2] for lv in CR.view_levels(scene, v, dtype)])
    K = Ks[np.broadcast_to(np.asarray(level), X.shape[:1])]
    R, t = _pose(scene, v, dtype)
    p = np.einsum("nij,nkj->nki", K, X.astype(dtype) @ R.T + t)
    return p[..., :2] / p[..., 2:] - np.dtype(dtype).type(0.5)


def ratio_offset(ratio):
    """Relative distance of the footprint ratio to the nearest level switch 0.5 * 2^-k (k >= 0): ratio / switch - 1."""
    ratio = np.asarray(ratio, np.float64)
    k = np.maximum(0, np.round(-np.log2(np.maximum(ratio, 1e-30)) - 1.0))
    return ratio / (0.5 * 2.0 ** -k) - 1.0


def view_state(scene, ref, scale, v, x, y, depth, dzI, dzJ):
    """Neighbour view v of the patches: level (clamped), requested level, footprint ratio, whether the view can be
    sampled at all (nfp > 0), the 25 projections [N, 25, 2] at the level and its size."""
    X = patch_points(scene, ref, scale, x, y, depth, dzI, dzJ)
    c = X[:, NS // 2]
    mfp = CR.cam_z(scene, ref, c) * CR.view_levels(scene, ref)[scale][3][0, 0]
    lvs = CR.view_levels(scene, v)
    nfp = CR.cam_z(scene, v, c) * lvs[0][3][0, 0]
    ok = (nfp > 0) & (mfp > 0)
    level, req = CR.level_of(np.where(ok, nfp, 1.0), np.where(ok, mfp, 1.0), len(lvs))
    q = project(scene, v, level, X)
    wh = np.array([(lv[0], lv[1]) for lv in lvs])[level]
    return dict(level=level, req=req, ratio=nfp / mfp, ok=ok, q=q, w=wh[:, 0], h=wh[:, 1])


def border_distances(st):
    """[N, 25, 4] signed distances of the samples to the left, right, top and bottom border (positive inside)."""
    qx, qy = st["q"][..., 0], st["q"][..., 1]
    return np.stack([qx, (st["w"] - 1)[:, None] - qx, qy, (st["h"] - 1)[:, None] - qy], -1)


def view_classes(st):
    """Per patch, for one view state: the sample classes, padded_right / bottom, level_switch, level_clamped and
    `conditioned` (the margin rule holds for this view)."""
    db = border_distances(st)
    d = db.min(-1)                                  # [N, 25]
    nout = (d < 0).sum(1)
    kx = d.argmin(1)                                # the extreme sample
    bx = db[np.arange(len(d)), kx].argmin(-1)       # and the border it is nearest to (or outside of)
    dmin = d.min(1)
    far = (np.abs(d) >= MARGIN).all(1)
    roff = np.abs(ratio_offset(st["ratio"]))
    ok = st["ok"]
    one = ok & far & (nout == 1)
    c = dict(near_edge_in=ok & (nout == 0) & (dmin >= MARGIN) & (dmin <= NEAR),
             one_out_tail=one & (kx >= 22), one_out_head=one & (kx <= 1), one_out_mid=one & (kx > 1) & (kx < 22))
    edge = c["near_edge_in"] | one
    c["padded_right"] = edge & (bx == 1) & (st["w"] % 4 != 0)
    c["bottom"] = edge & (bx == 3)
    c["level_switch"] = ok & (roff >= RATIO_MARGIN) & (roff <= RATIO_NEAR)
    c["level_clamped"] = ok & (st["req"] > st["level"])
    c["conditioned"] = ~ok | (far & (roff >= RATIO_MARGIN))
    return c


def sampled_views(gsel, pin):
    """[N, G] which global candidates each input samples at its input state: all of them for a seed (n_local == 0), its
    local views otherwise."""
    gsel = np.asarray(gsel)
    seed = pin["n_local"] == 0
    local = ((pin["local_ids"][:, :, None] == gsel[None, None, :]) &
             (np.arange(4)[None, :, None] < pin["n_local"][:, None, None])).any(1)
    return seed[:, None] | local


def edge_classes(scene, ref, scale, gsel, pin, per_view=False):
    """One boolean mask [N] per class of CLASSES (and `conditioned`: the margin rule holds for every view the patch
    samples), evaluated on the float32 inputs `pin` (oracle_py.PATCH_IN).  per_view: [N, G] masks of the view classes
    instead, over the global candidates (the patch classes are their `any` over the views it samples)."""
    x, y = pin["x"], pin["y"]
    args = (x, y, pin["depth"].astype(np.float64), pin["dz_i"].astype(np.float64), pin["dz_j"].astype(np.float64))
    keys = SAMPLE_CLASSES + ("padded_right", "bottom", "level_switch", "level_clamped", "conditioned")
    pv = {k: np.zeros((len(pin), len(gsel)), bool) for k in keys}
    for g, v in enumerate(gsel):
        c = view_classes(view_state(scene, ref, scale, int(v), *args))
        for k in keys:
            pv[k][:, g] = c[k]
    if per_view:
        return pv
    use = sampled_views(gsel, pin)
    out = {k: (pv[k] & use).any(1) for k in keys if k != "conditioned"}
    out["conditioned"] = (pv["conditioned"] | ~use).all(1)
    W, H = CR.view_levels(scene, ref)[scale][:2]
    out["master_border"] = np.isin(x, (2, W - 3)) | np.isin(y, (2, H - 3))
    out["master_outside"] = np.isin(x, (1, W - 2)) | np.isin(y, (1, H - 2))
    return out


def _bisect(f, lo, hi, iters=45):
    """Roots of the vectorised f(t, idx) in [lo, hi] where f changes sign (NaN elsewhere); f is evaluated only on the
    entries `idx` that bracket a root."""
    out = np.full(len(lo), np.nan)
    flo = f(lo, np.arange(len(lo)))
    idx = np.nonzero(np.sign(flo) * np.sign(f(hi, np.arange(len(lo)))) < 0)[0]
    lo, hi, flo = lo[idx], hi[idx], flo[idx]
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        left = np.sign(f(mid, idx)) == np.sign(flo)
        lo, hi = np.where(left, mid, lo), np.where(left, hi, mid)
    out[idx] = 0.5 * (lo + hi)
    return out


def _targets(scene, ref, scale, v, P):
    """Depths (float64, NaN where unreachable) within +-3 % of the traced ones at which view v meets each target:
    [(kind, depths)] for the extreme sample at DELTAS from each border and the footprint ratio at RATIO_DELTAS from the
    nearest switch."""
    x, y, dzI, dzJ = P["x"], P["y"], P["dz_i"].astype(np.float64), P["dz_j"].astype(np.float64)
    t0 = P["depth"].astype(np.float64)
    st = lambda t, i: view_state(scene, ref, scale, v, x[i], y[i], t, dzI[i], dzJ[i])      # noqa: E731
    out = []
    for b in range(4):
        for delta in DELTAS:
            out.append(("border", _bisect(lambda t, i: border_distances(st(t, i))[..., b].min(1) - delta, 0.97 * t0, 1.03 * t0)))
    every = np.arange(len(t0))
    k = np.maximum(0, np.round(-np.log2(np.maximum(st(t0, every)["ratio"], 1e-30)) - 1.0))
    for delta in RATIO_DELTAS:
        out.append(("ratio", _bisect(lambda t, i: st(t, i)["ratio"] / (0.5 * 2.0 ** -k[i]) - 1.0 - delta, 0.97 * t0, 1.03 * t0)))
    return out


def _with_view(ids, v, gsel, rng):
    """Four distinct ascending local views that include v: the traced ones with v in place of a random other."""
    ids = [int(i) for i in ids if i >= 0 and i != v]
    pool = [int(g) for g in gsel if g != v and g not in ids]
    while len(ids) < 3:
        ids.append(pool.pop(int(rng.integers(len(pool)))))
    if len(ids) > 3:
        ids.pop(int(rng.integers(len(ids))))
    return sorted(ids + [v])


def make_cases(scene, ref, scale, gsel, tin, tout, rng, n_trace=None, per_label=250, per_edge=30):
    """PatchOptimization inputs (oracle_py.PATCH_IN) on the edges of CLASSES, built from an execution trace (tin / tout).
    For a seeded sample of the traced patches and every global candidate the depth is bisected in float64 until the
    extreme sample (or the footprint ratio) meets its target; the result is rounded to float32 and kept only if its class
    still holds and the margin rule holds for every view it samples.  Each kept case is given twice: as a seed and with the
    edge view among four local views.  Up to `per_label` cases per target class, plus the master-border pixels of every
    edge and corner with traced depths.  Returned in a seeded random order, so that seeds and propagated inputs, failing
    and succeeding patches sit side by side in a batch."""
    from oracle import oracle_py as O
    W, H = CR.view_levels(scene, ref)[scale][:2]
    good = np.nonzero((tin["depth"] > 0) & (tin["x"] >= 2) & (tin["y"] >= 2) & (tin["x"] <= W - 3) & (tin["y"] <= H - 3))[0]
    pick = np.sort(rng.choice(good, size=len(good) if n_trace is None else min(n_trace, len(good)), replace=False))
    P, Pout = tin[pick], tout[pick]
    labels = {k: [] for k in SAMPLE_CLASSES + ("level_switch",)}
    for g, v in enumerate(gsel):
        for kind, t in _targets(scene, ref, scale, int(v), P):
            idx = np.nonzero(np.isfinite(t))[0]
            if not len(idx):
                continue
            rec = np.array(P[idx])
            rec["depth"] = t[idx].astype(np.float32)
            rec["n_local"] = 0
            rec["local_ids"] = -1
            vc = view_classes(view_state(scene, ref, scale, int(v), rec["x"], rec["y"], rec["depth"].astype(np.float64),
                                         rec["dz_i"].astype(np.float64), rec["dz_j"].astype(np.float64)))
            for j, i in enumerate(idx):
                own = ["level_switch"] if kind == "ratio" else [k for k in SAMPLE_CLASSES if vc[k][j]]
                if own and (kind != "ratio" or vc["level_switch"][j]):
                    labels[own[0]].append((rec[j], int(v), i))
    cases = []
    for lab, items in labels.items():
        for n in rng.permutation(len(items)):
            if sum(1 for c in cases if c[0] == lab) >= per_label:
                break
            r, v, i = items[n]
            seed = np.array([r])
            local = np.array([r])
            ids = _with_view(Pout["local_ids"][i] if P["n_local"][i] == 0 else P["local_ids"][i], v, gsel, rng)
            local["n_local"], local["local_ids"] = 4, ids
            pair = np.concatenate([seed, local])
            c = edge_classes(scene, ref, scale, gsel, pair)
            if c["conditioned"].all() and c[lab].all():
                cases.append((lab, pair))
    # master-border pixels: traced depths of the patches nearest to each edge, moved onto the edge and one pixel past it
    master = []
    order = rng.permutation(len(P))
    for axis, lo_hi in ((0, (2, W - 3)), (1, (2, H - 3))):
        coord = P["x"] if axis == 0 else P["y"]
        for e, edge in enumerate(lo_hi):
            near = order[np.argsort(np.abs(coord[order] - edge), kind="stable")][:per_edge]
            for i in near:
                for pos in (edge, edge - 1 if e == 0 else edge + 1):
                    master.append((i, axis, pos))
    for cx in (2, W - 3):
        for cy in (2, H - 3):
            i = int(np.argmin(np.abs(P["x"] - cx) + np.abs(P["y"] - cy)))
            for dx in (0, -1 if cx == 2 else 1):
                for dy in (0, -1 if cy == 2 else 1):
                    master.append((i, 2, (cx + dx, cy + dy)))
    for i, axis, pos in master:
        r = np.array(P[i:i + 1])
        if axis == 2:
            r["x"], r["y"] = pos
        elif axis == 0:
            r["x"] = pos
        else:
            r["y"] = pos
        seed = r.copy()
        seed["n_local"], seed["local_ids"] = 0, -1
        local = r.copy()
        if local["n_local"][0] == 0:
            local["n_local"], local["local_ids"] = 4, sorted(int(q) for q in Pout["local_ids"][i])
        pair = np.concatenate([seed, local])
        if min(Pout["local_ids"][i]) < 0 and P["n_local"][i] == 0:
            pair = seed
        c = edge_classes(scene, ref, scale, gsel, pair)
        if c["master_outside"].all() or c["conditioned"].all():
            cases.append(("master", pair))
    out = np.concatenate([p for _, p in cases]).astype(O.PATCH_IN)
    return out[rng.permutation(len(out))]
