"""The camera model of libs/dmrecon restated in NumPy (test infrastructure): the calibration of every pyramid level, the
pixel footprints, the mip-level choice with its clamp and the two resolution terms of the view selections.  Float64 by
default; `dtype=np.float32` evaluates the same expressions in the precision of the reference.

  levels()         image_pyramid.cc:19-53 with CameraInfo::fill_calibration / fill_inverse_calibration
                   (camera.cc:125-144,180-200, mve_b200.synth.fill_calibration)
  footprint()      SingleView::footPrint / footPrintScaled (single_view.h:154-164): camera z times 1 / ax of the level
  level_of()       patch_sampler.cc:76-91 and SingleView::clampLevel (single_view.h:113-123) with minLevel 0
  gvs_scale()      the resolution factor of GlobalViewSelection::benefitFromView (global_view_selection.cc:80-87)
  lvs_penalised()  the resolution test of LocalViewSelection::performVS (local_view_selection.cc:103-106)
"""
import numpy as np

from mve_b200.synth import fill_calibration

MIN_IMAGE_DIM = 30          # image_pyramid.cc:19


def levels(width, height, flen, paspect, ppoint, dtype=np.float64):
    """[(w, h, K, K^-1, portrait)] of every pyramid level: halved sizes rounded up, the principal point moved by
    w / (w + 1) where a dimension is odd, until the smaller dimension drops below MIN_IMAGE_DIM."""
    f = np.dtype(dtype).type
    ppx, ppy = f(ppoint[0]), f(ppoint[1])
    w, h = int(width), int(height)
    out = [(w, h) + fill_calibration(flen, paspect, (ppx, ppy), w, h, dtype)]
    while min(w, h) >= MIN_IMAGE_DIM:
        if w % 2 == 1:
            ppx = ppx * f(w) / f(w + 1)
        if h % 2 == 1:
            ppy = ppy * f(h) / f(h + 1)
        w, h = (w + 1) // 2, (h + 1) // 2
        out.append((w, h) + fill_calibration(flen, paspect, (ppx, ppy), w, h, dtype))
    return out


def view_levels(scene, v, dtype=np.float64):
    return levels(*scene.size(v), scene.flen[v], scene.paspect[v], scene.ppoint[v], dtype)


def cam_z(scene, v, X):
    """Camera-space z of world points X [..., 3] in view v."""
    R = scene.rot[v].astype(np.float64).reshape(3, 3)
    return X @ R[2] + float(scene.trans[v][2])


def footprint(scene, v, X, level=0):
    """World size of one pixel of view v's pyramid level `level` at X (footPrint: level 0; footPrintScaled: `scale`)."""
    return cam_z(scene, v, X) * view_levels(scene, v)[level][3][0, 0]


def level_of(nfp, mfp, n_levels):
    """(clamped level, requested level) of a view with footprint nfp for a master footprint mfp."""
    ratio = np.asarray(nfp / mfp, np.float64)
    req = np.zeros(ratio.shape, np.int64)
    while (ratio < 0.5).any():
        small = ratio < 0.5
        req += small
        ratio = np.where(small, ratio * 2.0, ratio)
    return np.minimum(req, n_levels - 1), req


def gvs_scale(mfp, nfp):
    """Factor of a feature's score for the footprint ratio mfp / nfp: 2 / ratio above 2, 1 in (1, 2], ratio up to 1."""
    r = np.asarray(mfp / nfp, np.float64)
    return np.where(r > 2.0, 2.0 / r, np.where(r > 1.0, 1.0, r))


def lvs_penalised(mfp, nfp):
    """The local view selection multiplies a view's score by 0.01 when its footprint is more than twice the master's."""
    return mfp / nfp < 0.5


def patch_centres(scene, ref, scale, pin):
    """World points of the centre pixels of PatchOptimization inputs (x, y, depth along the unit view ray of level
    `scale`: SingleView::viewRayScaled, patch_sampler.cc:290)."""
    Ki = view_levels(scene, ref)[scale][3]
    px = np.stack([pin["x"] + 0.5, pin["y"] + 0.5, np.ones(len(pin))], -1) @ Ki.T
    px /= np.linalg.norm(px, axis=1, keepdims=True)
    R = scene.rot[ref].astype(np.float64).reshape(3, 3)
    C = -(R.T @ scene.trans[ref].astype(np.float64))
    return C + pin["depth"][:, None].astype(np.float64) * (px @ R)


def camera_cases(scene, ref, scale, gsel, pin, pout):
    """Which camera cases a batch of PatchOptimizations meets, as one mask per case over the patches.  The sampled views
    of a patch are the local views of its input and of its result; the levels are those at the patch's centre point.
      level_ge2      a sampled view is read at pyramid level 2 or higher
      clamped        a sampled view is asked for a level past its last one, and clampLevel runs
      requested_ge3  a sampled view is asked for level 3 or higher
      penalised      a global candidate's footprint is more than twice the master's (local selection: score * 0.01)
      gvs_ratio_gt2  a global candidate's footprint is less than half the master's (global selection: 2 / ratio)"""
    X = patch_centres(scene, ref, scale, pin)
    mfp = footprint(scene, ref, X, scale)
    cases = {k: np.zeros(len(pin), bool) for k in ("level_ge2", "clamped", "requested_ge3", "penalised", "gvs_ratio_gt2")}
    for v in gsel:
        nfp = footprint(scene, v, X)
        lv, req = level_of(nfp, mfp, len(view_levels(scene, v)))
        used = (pin["local_ids"] == v).any(1) | (pout["local_ids"] == v).any(1)
        cases["level_ge2"] |= used & (lv >= 2)
        cases["clamped"] |= used & (req > lv)
        cases["requested_ge3"] |= used & (req >= 3)
        cases["penalised"] |= lvs_penalised(mfp, nfp)
        cases["gvs_ratio_gt2"] |= mfp / nfp > 2.0
    return cases
