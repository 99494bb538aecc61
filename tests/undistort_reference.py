"""NumPy restatement of mve::image::image_undistort_k2k4<uint8_t> (libs/mve/image_tools.h:1731-1769) with
Image::linear_at(float, float, T*) (image.h:438-460), in the arithmetic of the reference build (-O3 -march=x86-64-v3
-funsafe-math-optimizations), read from the disassembly of its instantiation: the contractions and reciprocals listed in
mve_b200/csrc/undistort.cuh.  Also the cases of tests/golden/undistort_ref.npz, regenerated from seeds, and how that
fixture holds their results: every byte of the images of at most FULL_PIXELS pixels, and of larger ones the SHA-256 of
every byte, the shape and a seeded sample of pixels.

NumPy has no fused multiply-add, so fma64 emulates it exactly: the product as an exact pair (Dekker), the sum with c as an
exact pair, and the two tails added with rounding to odd (Boldo and Melquiond, "Emulation of FMA and correctly rounded
sums: proved algorithms using rounding to odd", IEEE TC 2008).  A float fma is the exact double product plus c rounded to
odd, then rounded to float: 53 >= 24 + 2 bits make that double rounding innocuous."""
from __future__ import annotations

import hashlib

import numpy as np

F32 = np.float32
F64 = np.float64


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _split(a):
    t = 134217729.0 * a
    hi = t - (t - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _add_odd(a, b):
    """a + b rounded to odd (the neighbour with an odd last bit when the sum is inexact)."""
    s, e = _two_sum(a, b)
    s = np.asarray(s, F64)
    fix = (e != 0) & ((s.view(np.int64) & 1) == 0)
    return np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def fma64(a, b, c):
    a, b, c = (np.asarray(v, F64) for v in np.broadcast_arrays(a, b, c))
    uh, ul = _two_prod(a, b)
    th, tl = _two_sum(c, uh)
    return th + _add_odd(tl, ul)


def fma32(a, b, c):
    p = np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)     # exact: 48 bits
    return _add_odd(p, np.asarray(c, F32).astype(F64)).astype(F32)


def source_positions(w: int, h: int, flen: float, k2: float, k4: float):
    """(ix, iy) float32 of every output pixel, h x w, as the loop of image_undistort_k2k4 computes them."""
    flen, k2, k4 = F64(F32(flen)), F64(F32(k2)), F64(F32(k4))
    fw2, fh2 = F64(w) * 0.5, F64(h) * 0.5
    fnorm = F64(max(w, h))
    inv_fnorm = 1.0 / fnorm
    inv_f2 = 1.0 / (flen * flen)
    fx = (np.arange(w, dtype=F64) + (0.5 - fw2)) * inv_fnorm
    fy = (np.arange(h, dtype=F64) + (0.5 - fh2)) * inv_fnorm
    fx, fy = (np.ascontiguousarray(v) for v in np.broadcast_arrays(fx[None, :], fy[:, None]))
    rd = inv_f2 * fma64(fx, fx, fy * fy)
    rf = fma64(fma64(k4, rd, k2), rd, 1.0)
    ix = fma64(fnorm * fx, rf, fw2 - 0.5).astype(F32)
    iy = fma64(rf, fy * fnorm, fh2 - 0.5).astype(F32)
    return ix, iy


def undistort_k2k4(img: np.ndarray, flen: float, k2: float, k4: float) -> np.ndarray:
    """image_undistort_k2k4<uint8_t>(img, flen, k2, k4) for an h x w x c uint8 image (c = 1..4); flen, k2, k4 are taken as
    float, as sfmrecon passes CameraInfo's fields."""
    img = np.asarray(img, np.uint8)
    if img.ndim == 2:
        img = img[:, :, None]
    h, w, c = img.shape
    if F32(k2) == 0 and F32(k4) == 0:
        return img.copy()                                       # duplicate()
    ix, iy = source_positions(w, h, flen, k2, k4)
    keep = ~((ix < F32(-0.5)) | (ix.astype(F64) > w - 0.5) | (iy < F32(-0.5)) | (iy.astype(F64) > h - 0.5))
    # linear_at: min with the last index (NaN takes the bound), then max with 0
    xc = np.where(ix < F32(w - 1), ix, F32(w - 1)).astype(F32)
    yc = np.where(iy < F32(h - 1), iy, F32(h - 1)).astype(F32)
    xc = np.where(xc > F32(0), xc, F32(0)).astype(F32)
    yc = np.where(yc > F32(0), yc, F32(0)).astype(F32)
    tx, ty = np.trunc(xc), np.trunc(yc)
    x0, y0 = tx.astype(np.int64), ty.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, w - 1), np.minimum(y0 + 1, h - 1)
    w1 = xc - tx
    w0 = tx + (F32(1) - xc)
    w3 = yc - ty
    w2 = (ty + F32(1)) - yc
    out = np.zeros_like(img)
    for ch in range(c):
        v = img[:, :, ch].astype(F32)
        top = fma32(v[y0, x0], w0, v[y0, x1] * w1)
        bot = fma32(v[y1, x0], w0, v[y1, x1] * w1)
        r = fma32(top, w2, bot * w3) + F32(0.5)
        out[:, :, ch] = np.where(keep, r.astype(np.int32) & 0xFF, 0).astype(np.uint8)
    return out


# ---- the fixture's cases ----
SIZES = ((1, 1), (1, 7), (7, 1), (2, 2), (31, 7), (33, 9), (101, 135), (640, 480))    # (w, h)
FLENS = (0.6, 1.0, 2.4)
PAIRS = {"none": (0.0, 0.0), "barrel": (0.12, 0.0), "pincushion": (-0.09, 0.012), "tiny": (1e-7, 0.0),
         "strong": (0.9, -0.45)}


def make_image(w: int, h: int, c: int, seed: int) -> np.ndarray:
    """A seeded test photo: noise on small images; on large ones a smooth pattern with fine texture and noise."""
    rng = np.random.default_rng(seed)
    if w * h <= 64 * 64:
        return rng.integers(0, 256, size=(h, w, c), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(F64)
    base = np.stack([96 + 80 * np.sin(x / (7.0 + 3 * k) + k) * np.cos(y / (11.0 + 2 * k)) for k in range(c)], -1)
    stripes = 40.0 * (((x.astype(np.int64) // 3 + y.astype(np.int64) // 5) % 2) - 0.5)
    img = base + stripes[:, :, None] + rng.normal(0, 2, size=(h, w, c))
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def _edge_k2(w, h, flen, px, py, axis, target, lo, hi):
    """Float k2 (k4 = 0) values on both sides of where ix (axis 0) or iy (axis 1) of pixel (px, py) crosses `target`."""
    def pos(k2):
        return float(source_positions(w, h, flen, k2, 0.0)[axis][py, px])
    flo = pos(lo) - target
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        if (pos(mid) - target > 0) == (flo > 0):
            lo = mid
        else:
            hi = mid
    k = F32(lo)
    return [float(np.nextafter(k, F32(-np.inf), dtype=F32)), float(k), float(np.nextafter(k, F32(np.inf), dtype=F32))]


def cases():
    """[(name, w, h, c, flen, k2, k4, seed)]: every size with every coefficient pair (channels and flen cycled; the 640x480
    image only with two pairs), then border cases whose source positions lie within 1e-4 px of -0.5 or w - 0.5."""
    out = []
    i = 0
    for (w, h) in SIZES:
        for pname, (k2, k4) in PAIRS.items():
            if (w, h) == (640, 480) and pname not in ("barrel", "strong"):
                continue
            c = 1 + i % 4
            flen = FLENS[i % 3]
            out.append(("%dx%d_%s_c%d_f%g" % (w, h, pname, c, flen), w, h, c, flen, k2, k4, 1000 + i))
            i += 1
    # corner and edge pixels crossing the borders: ix of pixel (0, 0) at -0.5 and of (w-1, 0) at w - 0.5, and likewise iy
    for (w, h, flen) in ((33, 9, 1.0), (31, 7, 0.6), (13, 17, 2.4)):
        for axis, px, py, target in ((0, 0, 0, -0.5), (0, w - 1, h // 2, w - 0.5), (1, 0, 0, -0.5), (1, w // 2, h - 1, h - 0.5)):
            for k2 in _edge_k2(w, h, flen, px, py, axis, target, 0.0, 4.0 * flen * flen):
                c = 1 + i % 4
                out.append(("%dx%d_edge%d_%d_%d_c%d_f%g" % (w, h, axis, px, py, c, flen), w, h, c, flen, k2, 0.0, 1000 + i))
                i += 1
    return out


# ---- the fixture's layout ----
FULL_PIXELS = 64 * 64         # results up to this many pixels are kept whole
N_SAMPLE = 2048               # pixels kept of a larger result, besides its digest


def _sample_index(h, w, seed):
    return np.random.default_rng(seed + 77).choice(h * w, size=min(N_SAMPLE, h * w), replace=False)


def digest(img: np.ndarray) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(img, np.uint8).tobytes()).digest(), np.uint8)


def fixture_entries(case, out: np.ndarray) -> dict:
    """The fixture's arrays for the reference result `out` of `case`."""
    name, w, h, c, flen, k2, k4, seed = case
    if w * h <= FULL_PIXELS:
        return {name: out}
    return {name + "__sha256": digest(out), name + "__shape": np.asarray(out.shape, np.int32),
            name + "__sample": out.reshape(h * w, c)[_sample_index(h, w, seed)]}


def check(golden, case, img: np.ndarray) -> None:
    """Asserts that `img` is the reference's result of `case` as the fixture holds it."""
    name, w, h, c, flen, k2, k4, seed = case
    img = np.asarray(img)
    if name in golden.files:
        np.testing.assert_array_equal(img, golden[name], err_msg=name)
        return
    assert img.shape == tuple(golden[name + "__shape"]), (name, img.shape)
    sample = img.reshape(h * w, c)[_sample_index(h, w, seed)]
    np.testing.assert_array_equal(sample, golden[name + "__sample"], err_msg=name)
    assert digest(img).tobytes() == golden[name + "__sha256"].tobytes(), name
