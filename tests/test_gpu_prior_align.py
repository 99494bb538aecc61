"""Relative priors (b200mvs_set_view_prior_relative[_device], Scene.set_view_prior_relative): planted maps give the planted
transform and the NumPy restatement's fit record; the installed prior is byte for byte set_view_prior of the restated
apply, on both routes, pitched, smaller than the view and under a mask; the routes agree; a failed fit leaves the
previous prior and the memory accounting alone; budgets change no map; a synthetic monocular prior keeps the quality of
the plain run; and the drop-in CLI installs the same prior."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import prior_align_reference as ref
from tests.test_gpu_prior import _fill_and_error, _run, _same
from tests.test_gpu_prior_state import _cuda
from tests.test_gpu_recon_mask import CLI, _map_size, _settings, _silhouettes
from tests.util import golden_scene

pytestmark = pytest.mark.gpu

KINDS = {"disparity": ref.DISPARITY, "depth": ref.DEPTH, "depth_scale": ref.DEPTH_SCALE}
PLANTED = {"disparity": (0.8, 0.05), "depth": (1.7, -0.3), "depth_scale": (0.6, 0.0)}


def _planted(s, v, kind, w, h, seed, dither=0.0):
    """A w x h map holding, at each pixel that exactly one feature of view v projects to, the planted transform of that
    feature's z, with 10 % of those pixels corrupted; other pixels NaN.  Returns (map, uncorrupted observation count)."""
    cam = ref.camera(s, v)
    X = ref.view_features(s, v)
    W0, H0 = cam[6], cam[7]
    ok, u, vv, z = ref.project(cam, X)
    with np.errstate(all="ignore"):
        px, py = np.floor(u * w / W0), np.floor(vv * h / H0)
    ok &= (px >= 0) & (px < w) & (py >= 0) & (py < h)
    px, py, z = px[ok].astype(int), py[ok].astype(int), z[ok]
    pix = py * w + px
    uniq, counts = np.unique(pix, return_counts=True)
    single = np.isin(pix, uniq[counts == 1])
    sc_, sh = PLANTED[kind]
    y = 1.0 / z if kind == "disparity" else z
    d = (y - sh) / sc_
    rng = np.random.default_rng(seed)
    d = d + dither * np.median(d) * rng.uniform(-1, 1, len(d))
    bad = rng.random(len(d)) < 0.1
    d[bad] *= rng.uniform(2.0, 4.0, bad.sum())
    m = np.full((h, w), np.nan, np.float32)
    m[py[single], px[single]] = d[single].astype(np.float32)
    return m, int((single & ~bad).sum())


def _close_fit(got, want):
    assert got["n_obs"] == want["n_obs"] and got["n_inliers"] == want["n_inliers"], (got, want)
    np.testing.assert_allclose(got["scale"], want["scale"], rtol=1e-12)
    np.testing.assert_allclose(got["shift"], want["shift"], rtol=1e-12, atol=1e-12 * abs(want["scale"]))
    np.testing.assert_allclose(got["median_rel_err"], want["median_rel_err"], rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("kind", list(KINDS))
def test_planted_maps(kind):
    from mve_b200 import dmrecon
    s = golden_scene("T1")
    sc = dmrecon.Scene.from_synth(s)
    for v in (0, 3):
        W0, H0 = s.size(v)
        for dither in (0.0, 1e-5):
            m, n_good = _planted(s, v, kind, W0, H0, seed=v, dither=dither)
            got = sc.set_view_prior_relative(v, m, 4, kind=kind)
            want, _ = ref.relative_prior(s, v, m, KINDS[kind])
            assert want["ok"]
            _close_fit(got, want)
            # exact values: the float32 rounding of the planted ones; dithered: the dither's least-squares error too
            tol = 1e-4 if dither else 1e-6
            np.testing.assert_allclose([got["scale"], got["shift"]], PLANTED[kind], rtol=tol, atol=tol)
            # Exact values differ from the model by their float32 rounding alone, which grows with d: the 3 sigma cut of
            # that near-zero spread drops some of the largest.  A uniform dither above the rounding keeps every one.
            print("%s view %d dither %g: n_obs %d n_inliers %d uncorrupted %d" % (
                kind, v, dither, got["n_obs"], got["n_inliers"], n_good))
            if dither:
                assert got["n_inliers"] == n_good
            else:
                assert 0.5 * n_good <= got["n_inliers"] <= n_good
    sc.close()


def _mono(s, v, size, seed=0):
    from mve_b200 import synth
    W0, H0 = s.size(v)
    w, h = size if isinstance(size, tuple) else (W0 // size, H0 // size)
    return synth.monocular(s, v, w, h, seed=seed)


@pytest.mark.parametrize("case", ["host", "device", "pitched", "view_size", "masked"])
def test_bit_exact_install(case):
    """The maps of a relative prior are those of set_view_prior(apply(values, fit)) with the returned s and t."""
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    if case == "masked":
        for v, m in _silhouettes(s, refs).items():
            sc.set_view_mask(v, m)
    fits, applied = {}, {}
    for v in refs:
        m = _mono(s, v, 1 if case == "view_size" else 4, seed=v)
        if case in ("device", "pitched"):
            fits[v] = sc.set_view_prior_relative(v, _cuda(m, case == "pitched"), 4, kind="disparity")
        else:
            fits[v] = sc.set_view_prior_relative(v, m, 4, kind="disparity")
        want, _ = ref.relative_prior(s, v, m, ref.DISPARITY)
        _close_fit(fits[v], want)
        applied[v] = ref.apply(ref.camera(s, v), m, ref.DISPARITY, fits[v]["scale"], fits[v]["shift"])
    got, gc = _run(sc, st, refs)
    for v in refs:
        sc.set_view_prior(v, applied[v], 4)
    want, wc = _run(sc, st, refs)
    _same(got, want)
    assert gc == wc
    sc.close()


@pytest.mark.parametrize("kind", list(KINDS))
def test_routes_agree(kind):
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    out = {}
    for route in ("host", "device"):
        sc = dmrecon.Scene.from_synth(s)
        fits = []
        for v in refs:
            m = _mono(s, v, 4, seed=v)
            if kind == "depth":                 # an affine depth map of the same scene
                with np.errstate(divide="ignore"):
                    m = np.where(m > 0, 1.0 / m, 0).astype(np.float32)
            fits.append(sc.set_view_prior_relative(v, m if route == "host" else torch.from_numpy(m).cuda(), 4, kind=kind))
        out[route] = (fits, _run(sc, st, refs))
        sc.close()
    assert out["host"][0] == out["device"][0]
    _same(out["host"][1][0], out["device"][1][0])
    assert out["host"][1][1] == out["device"][1][1]


def test_failures_leave_state_and_memory():
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    v = refs[0]
    m = _mono(s, v, 4)
    h, w = m.shape
    f0 = sc.memory_stats().fixed
    fit = sc.set_view_prior_relative(v, m, 4)
    installed = ref.apply(ref.camera(s, v), m, ref.DISPARITY, fit["scale"], fit["shift"])
    before, bc = _run(sc, st, refs)
    mem_rel = sc.memory_stats()            # after the run: its pyramids and workspace stay resident for the next call
    sc.set_view_prior(v, installed, 4)
    mem_abs = sc.memory_stats()
    assert mem_rel.fixed == mem_abs.fixed == f0 + 4 * w * h
    assert mem_rel.resident == mem_abs.resident
    # the same prior again, then failing fits of every kind of failure: the maps of that prior stay
    sc.set_view_prior_relative(v, m, 4)
    flat = np.full_like(m, 2.0)
    flat[0, 0] = 3.0
    fails = [(np.full_like(m, np.nan), "fewer than 16 usable feature observations", 0),
             (np.full_like(m, np.inf), "fewer than 16 usable feature observations", 0),
             (flat, "no spread", None),
             (m.max() + m.min() - m, "the scale is not positive", None)]
    for bad, why, n_obs in fails:
        for values in (bad, torch.from_numpy(bad).cuda()):
            with pytest.raises(dmrecon.B200MVSError) as e:
                sc.set_view_prior_relative(v, values, 4)
            assert e.value.code == dmrecon.ERR_INVALID_ARG and why in str(e.value), str(e.value)
            assert "b200mvs_set_view_prior_relative" in str(e.value)
            assert e.value.fit["n_obs"] == (n_obs if n_obs is not None else fit["n_obs"])
            assert e.value.fit["scale"] == 0 and e.value.fit["n_inliers"] == 0
    after, ac = _run(sc, st, refs)
    _same(after, before)
    assert ac == bc
    # scratch is released: repeated calls hold what one call holds
    res = sc.memory_stats().resident
    for _ in range(5):
        sc.set_view_prior_relative(v, torch.from_numpy(m).cuda(), 4)
    assert sc.memory_stats().resident == res and sc.memory_stats().fixed == mem_rel.fixed
    # it replaces a prior with dz and ids
    earlier, _ = sc.reconstruct(st, [v])
    sc.set_view_prior(v, earlier[0]["depth"], 4, dz=earlier[0]["dz"], view_ids=earlier[0]["view_ids"])
    sc.set_view_prior_relative(v, m, 4)
    assert sc.memory_stats().fixed == mem_rel.fixed
    again, _ = _run(sc, st, refs)
    _same(again, before)
    sc.close()


def test_budget_groups():
    from mve_b200 import dmrecon
    s = golden_scene("T2")
    st = _settings(s)
    refs = np.random.default_rng(5).permutation(s.n_views).tolist()
    priors = {v: _mono(s, v, 4, seed=v) for v in refs}
    plain = dmrecon.Scene.from_synth(s)
    for v in refs:
        plain.set_view_prior_relative(v, priors[v], 4)
    want, wc = _run(plain, st, refs)
    plain.close()
    lazy = dmrecon.Scene.from_synth(s, lazy=True)
    for v in refs:
        lazy.set_view_prior_relative(v, priors[v], 4)
    fixed = lazy.memory_stats().fixed
    single = max(lazy.working_set(st, [r]) for r in refs)
    total = lazy.working_set(st, refs)
    chosen = None
    for avail in np.linspace(single, total, 40).astype(np.int64).tolist():
        n, groups = lazy.plan_batches(st, refs, int(avail))
        if n >= 2:
            chosen = (avail, n)
            break
    assert chosen
    lazy.set_image_source(lambda v: s.images[v], fixed + chosen[0])
    got, c = _run(lazy, st, refs)
    mem = lazy.memory_stats()
    assert mem.n_groups == chosen[1] and mem.peak <= mem.budget
    _same(got, want)
    assert c["n_seeds_processed"] == wc["n_seeds_processed"]
    lazy.close()


@pytest.mark.parametrize("name", ["T1", "T2"])
def test_quality(name):
    """The noisy synthetic monocular prior at stride 4: fill at least the plain run's, median and p95 relative depth
    error within 5 % of the plain run's (SURVEY 8c); the analytic depth as the prior is printed beside it."""
    from mve_b200 import dmrecon, synth
    s = golden_scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    sc = dmrecon.Scene.from_synth(s)
    plain, pc = _run(sc, st, refs)
    for v in refs:
        sc.set_view_prior_relative(v, _mono(s, v, 4, seed=v), 4)
    mono, mc = _run(sc, st, refs)
    for v in refs:
        sc.set_view_prior(v, synth.depth(s, v, *_map_size(s, v)), 4)
    exact, ec = _run(sc, st, refs)
    rows = {k: _fill_and_error(s, m, refs) for k, m in (("plain", plain), ("mono", mono), ("depth", exact))}
    for k, c in (("plain", pc), ("mono", mc), ("depth", ec)):
        f, m, p = rows[k]
        print("%s %-5s fill %.4f median %.3e p95 %.3e rounds %d" % (name, k, f, m, p, c["n_rounds"]))
    f0, m0, p0 = rows["plain"]
    f1, m1, p1 = rows["mono"]
    assert f1 >= f0
    assert m1 <= 1.05 * m0 and p1 <= 1.05 * p0
    sc.close()


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli():
    """B200MVS_PRIOR_MONO=<embedding>,4,disparity: the maps Scene.set_view_prior_relative gives; a view without the
    embedding runs without a prior and says so; malformed values and B200MVS_PRIOR beside it are refused."""
    from mve_b200 import dmrecon, synth
    s = golden_scene("T1")
    views = [0, 4, 7]
    lvl = s.scale
    base = ["-s%d" % lvl, "--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--progress=silent", "--force",
            "-l" + ",".join(str(v) for v in views)]
    mono = {v: _mono(s, v, 4, seed=v) for v in views}
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        for v in views[:2]:
            synth.write_mvei(os.path.join(tmp, "views", "view_%04d.mve" % v, "mono.mvei"), mono[v][:, :, None])
        out = subprocess.run([CLI] + base + [tmp], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, B200MVS_PRIOR_MONO="mono,4,disparity"))
        assert out.returncode == 0, out.stdout + out.stderr
        assert 'Prior not found for image "0007", skipping.' in out.stdout, out.stdout
        sc = dmrecon.Scene.from_synth(s)
        st = dmrecon.Settings(scale=lvl, nr_recon_neighbors=s.nr_recon_neighbors)
        for v in views:
            if v in views[:2]:
                fit = sc.set_view_prior_relative(v, mono[v], 4)
                assert ("Prior fit for image \"%04d\": s %.6g t %.6g, %u of %u inliers"
                        % (v, fit["scale"], fit["shift"], fit["n_inliers"], fit["n_obs"])) in out.stdout, out.stdout
            else:
                sc.set_view_prior(v, None, 4)
            want, _ = sc.reconstruct(st, [v])
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            depth = synth.read_mvei(os.path.join(vd, "depth-L%d.mvei" % lvl))[:, :, 0]
            assert depth.tobytes() == want[0]["depth"].tobytes(), v
        sc.close()
        for bad in ("mono,4", "mono,0,disparity", "mono,4,inverse", ",4,depth"):
            out = subprocess.run([CLI] + base + [tmp], capture_output=True, text=True, timeout=600,
                                 env=dict(os.environ, B200MVS_PRIOR_MONO=bad))
            assert "B200MVS_PRIOR_MONO: expected" in out.stderr, (bad, out.stderr)
        out = subprocess.run([CLI] + base + [tmp], capture_output=True, text=True, timeout=600,
                             env=dict(os.environ, B200MVS_PRIOR_MONO="mono,4,disparity", B200MVS_PRIOR="mono,4"))
        assert "B200MVS_PRIOR_MONO and B200MVS_PRIOR" in out.stderr, out.stderr
