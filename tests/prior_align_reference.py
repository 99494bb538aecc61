"""The relative prior of b200mvs_set_view_prior_relative (include/b200mvs.h) restated in NumPy float64: the observations
of a view's features, the fit of s and t, and the apply.  Every product, quotient and sum is one NumPy operation, in the
order the header states, so the observations and the apply equal the device's bit for bit; the fit's sums may differ from
the device's in their last bits (another summation order)."""
import numpy as np

from mve_b200.synth import fill_calibration

DISPARITY, DEPTH, DEPTH_SCALE = 0, 1, 2
MIN_OBS, ROUNDS, MAD_SIGMA, CUT = 16, 3, 1.4826, 3.0


def camera(scene, v):
    """(R, t, ax, ay, cx, cy, W0, H0) of view v as the rules read them: float32 values widened to float64."""
    W0, H0 = scene.size(v)
    K = fill_calibration(scene.flen[v], scene.paspect[v], scene.ppoint[v], W0, H0, np.float32)[0]
    R = np.asarray(scene.rot[v], np.float32).reshape(3, 3).astype(np.float64)
    t = np.asarray(scene.trans[v], np.float32).reshape(3).astype(np.float64)
    return R, t, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), int(W0), int(H0)


def view_features(scene, v):
    """The positions (n x 3 float32) of the features whose refs contain view v, in ascending feature order."""
    pos = np.asarray(scene.feat_pos, np.float32).reshape(-1, 3)
    return pos[[i for i, r in enumerate(scene.feat_refs) if v in set(np.asarray(r).tolist())]]


def project(cam, X):
    """(ok, u, v, z) of points X (n x 3 float32): z > 0, u and v the photo position."""
    R, t, ax, ay, cx, cy, _, _ = cam
    X = np.asarray(X, np.float32).astype(np.float64)
    xc = [R[r, 0] * X[:, 0] + R[r, 1] * X[:, 1] + R[r, 2] * X[:, 2] + t[r] for r in range(3)]
    with np.errstate(all="ignore"):
        u = ax * xc[0] / xc[2] + cx
        v = ay * xc[1] / xc[2] + cy
    return xc[2] > 0, u, v, xc[2]


def observations(cam, X, values, kind):
    """The observations (d, y) of features X in the map `values` (h x w float32), in feature order, and the prior pixel
    (px, py) of each feature (-1 where there is none)."""
    values = np.asarray(values, np.float32)
    h, w = values.shape
    W0, H0 = cam[6], cam[7]
    ok, u, v, z = project(cam, X)
    with np.errstate(all="ignore"):
        fx, fy = u * w / W0, v * h / H0
    ok &= (fx >= 0) & (fx < w) & (fy >= 0) & (fy < h)
    px = np.where(ok, np.floor(np.where(ok, fx, 0)), -1).astype(np.int64)
    py = np.where(ok, np.floor(np.where(ok, fy, 0)), -1).astype(np.int64)
    d = np.zeros(len(z))
    d[ok] = values[py[ok], px[ok]].astype(np.float64)
    ok &= np.isfinite(d) & (d > 0)
    with np.errstate(all="ignore"):
        y = 1.0 / z if kind == DISPARITY else z
    return d[ok], y[ok], px, py


def lower_median(a):
    a = np.asarray(a, np.float64)
    return float(np.partition(a, (len(a) - 1) // 2)[(len(a) - 1) // 2])


def fit(d, y, kind):
    """The fit of the header: a dict of scale, shift, n_obs, n_inliers, median_rel_err and ok, with `reason` when it
    fails (the fields the C call leaves 0 are 0 then)."""
    d, y = np.asarray(d, np.float64), np.asarray(y, np.float64)
    n = len(d)
    out = dict(scale=0.0, shift=0.0, n_obs=n, n_inliers=0, median_rel_err=0.0, ok=False)
    if n < MIN_OBS:
        return dict(out, reason="observations")
    with np.errstate(all="ignore"):
        if kind == DEPTH_SCALE:
            s, t = lower_median(y / d), 0.0
        else:
            md, my = lower_median(d), lower_median(y)
            mad_d, mad_y = lower_median(np.abs(d - md)), lower_median(np.abs(y - my))
            if mad_d == 0:
                return dict(out, reason="MAD")
            s = mad_y / mad_d
            t = my - s * md

        def inliers(s, t):
            r = np.abs(y - (s * d + t))
            cut = CUT * (MAD_SIGMA * lower_median(r))
            return r <= cut

        for _ in range(ROUNDS):
            m = inliers(s, t)
            if m.sum() < MIN_OBS:
                return dict(out, reason="inliers")
            di, yi = d[m], y[m]
            if kind == DEPTH_SCALE:
                sdd = np.sum(di * di)
                if sdd == 0:
                    return dict(out, reason="singular")
                s, t = np.sum(di * yi) / sdd, 0.0
            else:
                dm, ym = np.sum(di) / m.sum(), np.sum(yi) / m.sum()
                sxx = np.sum((di - dm) * (di - dm))
                if sxx == 0:
                    return dict(out, reason="singular")
                s = np.sum((di - dm) * (yi - ym)) / sxx
                t = ym - s * dm
        m = inliers(s, t)
        if m.sum() < MIN_OBS:
            return dict(out, reason="inliers")
        if not (np.isfinite(s) and s > 0 and np.isfinite(t)):
            return dict(out, reason="scale")
        q = s * d[m] + t
        zf, z = (1.0 / q, 1.0 / y[m]) if kind == DISPARITY else (q, y[m])
        rel = lower_median(np.abs(zf - z) / z)
    return dict(scale=float(s), shift=float(t), n_obs=n, n_inliers=int(m.sum()), median_rel_err=rel, ok=True)


def apply(cam, values, kind, s, t):
    """The depth map (h x w float32) the fit s, t makes of `values`."""
    _, _, ax, ay, cx, cy, W0, H0 = cam
    values = np.asarray(values, np.float32)
    h, w = values.shape
    d = values.astype(np.float64)
    with np.errstate(all="ignore"):
        q = s * d + t
        z = 1.0 / q if kind == DISPARITY else q
        a = ((np.arange(w, dtype=np.float64) + 0.5) * W0 / w - cx) / ax
        b = ((np.arange(h, dtype=np.float64) + 0.5) * H0 / h - cy) / ay
        norm = np.sqrt(a[None, :] * a[None, :] + b[:, None] * b[:, None] + 1.0)
        out = (z * norm).astype(np.float32)
    good = np.isfinite(d) & (d > 0) & np.isfinite(z) & (z > 0)
    return np.where(good, out, np.float32(0))


def relative_prior(scene, v, values, kind):
    """(fit dict, depth map or None) of b200mvs_set_view_prior_relative for view v of `scene`."""
    cam = camera(scene, v)
    d, y, _, _ = observations(cam, view_features(scene, v), values, kind)
    f = fit(d, y, kind)
    return f, (apply(cam, values, kind, f["scale"], f["shift"]) if f["ok"] else None)
