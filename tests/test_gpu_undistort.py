"""Views given their original photos (-m gpu): b200mvs_set_view_distortion / Scene.set_view_distortion undistort every
image the view receives with k_undistort_k2k4, byte for byte sfmrecon's image_undistort_k2k4<uint8_t>.

Level 0 must equal the reference's result (converted as k_import_rgb converts an `undistorted` image) by host upload,
device upload and an image source that evicts and fetches again; the expected bytes are the NumPy restatement's, each
checked first against tests/golden/undistort_ref.npz.  Every level must equal a plain upload of those bytes; (0, 0)
must be the plain import; a changed value drops the pyramid; and on T0 and T5 the maps, point sets and the drop-in CLI's
files must equal those of the reference-undistorted scene.  The fixture's 1-wide and 1-high cases are left to the CPU
tests: the C ABI registers views of at least 2 x 2 pixels."""
import copy
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests import undistort_reference as UR
from tests.util import ROOT, golden_scene

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "dmrecon_b200")
CAM = dict(paspect=1.0, ppoint=(0.5, 0.5), rot=np.eye(3, dtype=np.float32), trans=np.zeros(3, np.float32))
MAPS = ("depth", "conf", "dz", "normal", "view_ids")


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(ROOT, "tests", "golden", "undistort_ref.npz"))


def _cases():
    return [c for c in UR.cases() if c[1] >= 2 and c[2] >= 2]


@pytest.fixture(scope="module")
def expected(golden):
    """The reference's result of every case: the restatement's, checked against the fixture."""
    out = {}
    for case in _cases():
        name, w, h, c, flen, k2, k4, seed = case
        out[name] = UR.undistort_k2k4(UR.make_image(w, h, c, seed), flen, k2, k4)
        UR.check(golden, case, out[name])
    return out


def _rgb(img):
    """What get_level returns for a level imported from `img` (alpha dropped, grey expanded: image_pyramid.cc:65-73)."""
    return np.ascontiguousarray(img[:, :, :3] if img.shape[2] >= 3 else np.repeat(img[:, :, :1], 3, axis=2))


def _levels(sc, v):
    return [sc.level(v, l) for l in range(sc.num_levels(v))]


def test_level0_host_upload(expected):
    from mve_b200 import dmrecon
    cases = _cases()
    sc = dmrecon.Scene(len(cases))
    for v, (name, w, h, c, flen, k2, k4, seed) in enumerate(cases):
        sc.set_view_distortion(v, k2, k4)
        sc.set_view(v, UR.make_image(w, h, c, seed), flen, **CAM)
    for v, (name, *_r) in enumerate(cases):
        assert sc.level(v, 0).tobytes() == _rgb(expected[name]).tobytes(), name
    sc.close()


def test_level0_device_upload(expected):
    """Device uploads take 3 channels: a grey photo is given as three equal channels, a 4-channel one without alpha (the
    undistortion works on each channel alone, so the expected bytes are the same)."""
    import torch
    from mve_b200 import dmrecon
    cases = _cases()
    sc = dmrecon.Scene(len(cases))
    keep = []
    for v, (name, w, h, c, flen, k2, k4, seed) in enumerate(cases):
        t = torch.from_numpy(_rgb(UR.make_image(w, h, c, seed))).cuda()
        keep.append(t)
        sc.set_view_distortion(v, k2, k4)
        sc.set_view_device(v, t.data_ptr(), w, h, flen, stream=torch.cuda.current_stream().cuda_stream, **CAM)
    for v, (name, *_r) in enumerate(cases):
        assert sc.level(v, 0).tobytes() == _rgb(expected[name]).tobytes(), name
        lvl = sc.level(v, 0, on_device=True)
        assert lvl.is_cuda and lvl.cpu().numpy().tobytes() == _rgb(expected[name]).tobytes(), name
    sc.close()


def test_level0_image_source_evicts_and_fetches_again(expected):
    from mve_b200 import dmrecon
    cases = _cases()
    sc = dmrecon.Scene(len(cases))
    for v, (name, w, h, c, flen, k2, k4, seed) in enumerate(cases):
        sc.set_view_camera(v, w, h, flen, **CAM)
        sc.set_view_distortion(v, k2, k4)
    fixed = sc.memory_stats().fixed
    # room for one 640x480 pyramid (20 bytes per texel at a pitch of 4, about 8.2 MB) with its staging, not for all
    sc.set_image_source(lambda v: UR.make_image(*cases[v][1:4], cases[v][7]), fixed + (14 << 20))
    for _ in range(2):
        for v, (name, *_r) in enumerate(cases):
            assert sc.level(v, 0).tobytes() == _rgb(expected[name]).tobytes(), name
    m = sc.memory_stats()
    assert m.n_loads > len(cases) and m.n_evictions > 0 and m.peak <= m.budget, m.as_dict()
    sc.close()


def test_every_level_equals_plain_upload_of_reference_bytes(expected):
    from mve_b200 import dmrecon
    cases = [c for c in _cases() if c[1] * c[2] >= 900]
    a, b = dmrecon.Scene(len(cases)), dmrecon.Scene(len(cases))
    for v, (name, w, h, c, flen, k2, k4, seed) in enumerate(cases):
        a.set_view_distortion(v, k2, k4)
        a.set_view(v, UR.make_image(w, h, c, seed), flen, **CAM)
        b.set_view(v, expected[name], flen, **CAM)
    for v, (name, *_r) in enumerate(cases):
        la, lb = _levels(a, v), _levels(b, v)
        assert len(la) == len(lb) > 1
        for l, (x, y) in enumerate(zip(la, lb)):
            assert x.tobytes() == y.tobytes(), (name, l)
    a.close()
    b.close()


def test_zero_coefficients_are_the_plain_import():
    from mve_b200 import dmrecon
    img = UR.make_image(101, 135, 3, 7)
    a, b = dmrecon.Scene(1), dmrecon.Scene(1)
    a.set_view_distortion(0, 0.0, -0.0)
    a.set_view(0, img, 1.0, **CAM)
    b.set_view(0, img, 1.0, **CAM)
    assert [x.tobytes() for x in _levels(a, 0)] == [x.tobytes() for x in _levels(b, 0)]
    assert a.level(0, 0).tobytes() == img.tobytes()
    assert a.memory_stats().as_dict() == b.memory_stats().as_dict()
    a.close()
    b.close()


def test_changed_value_drops_and_rebuilds():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    photo = s.images[0]
    und = {k: UR.undistort_k2k4(photo, s.flen[0], k, 0.0) for k in (0.1, 0.2)}
    sc = dmrecon.Scene.from_synth(s)
    fixed = sc.memory_stats().fixed
    ws = sc.working_set(st, [0])
    sc.set_view_distortion(0, 0.1, 0.0)
    assert sc.memory_stats().fixed == fixed and sc.working_set(st, [0]) == ws
    # no source: the view is not loaded until it is uploaded again
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.reconstruct(st, [0])
    assert e.value.code == dmrecon.ERR_INVALID_ARG and "color image of view 0 is not loaded" in str(e.value)
    sc.set_view(0, photo, s.flen[0], s.paspect[0], s.ppoint[0], s.rot[0], s.trans[0])
    assert sc.level(0, 0).tobytes() == _rgb(und[0.1]).tobytes()
    sc.set_view_distortion(0, 0.1, 0.0)                      # unchanged: the pyramid stays
    assert sc.level(0, 0).tobytes() == _rgb(und[0.1]).tobytes()
    # with a source: fetched again with the new value
    sc.set_image_source(lambda v: s.images[v])
    n0 = sc.memory_stats().n_loads
    sc.set_view_distortion(0, 0.2, 0.0)
    assert sc.level(0, 0).tobytes() == _rgb(und[0.2]).tobytes()
    assert sc.memory_stats().n_loads == n0 + 1
    sc.set_view_distortion(0, 0.0, 0.0)
    assert sc.level(0, 0).tobytes() == _rgb(photo).tobytes()
    assert sc.memory_stats().n_loads == n0 + 2 and sc.memory_stats().fixed == fixed
    sc.close()


def _coefficients(s):
    """Per-view coefficients: barrel, pincushion and strong pairs."""
    pairs = [(0.08, 0.0), (-0.06, 0.01), (0.25, -0.1), (0.02, 0.003)]
    return [pairs[v % len(pairs)] for v in range(s.n_views)]


def _undistorted_scene(s, ks):
    u = copy.copy(s)
    u.images = [UR.undistort_k2k4(s.images[v], s.flen[v], *ks[v]) for v in range(s.n_views)]
    return u


@pytest.mark.parametrize("name", ["T0", "T5"])
def test_reconstruction_equals_reference_undistorted_scene(name):
    from mve_b200 import dmrecon
    s = golden_scene(name)
    ks = _coefficients(s)
    want = dmrecon.Scene.from_synth(_undistorted_scene(s, ks))
    got = dmrecon.Scene(s.n_views)
    for v in range(s.n_views):
        got.set_view_distortion(v, *ks[v])
        got.set_view(v, s.images[v], s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    got.set_features(s.feat_pos, s.feat_refs)
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))
    ma, sa = want.reconstruct(st, refs)
    mb, sb = got.reconstruct(st, refs)
    assert sa.n_filled == sb.n_filled > 0
    for j in range(len(refs)):
        for k in MAPS:
            assert ma[j][k].tobytes() == mb[j][k].tobytes(), (name, refs[j], k)
    opts = dict(with_normals=True, with_conf=True, with_scale=True)
    pa, _ = want.reconstruct_pointset(st, refs, opts)
    pb, _ = got.reconstruct_pointset(st, refs, opts)
    assert len(pa["colors"]) > 0
    for k in ("vertices", "normals", "colors", "values", "confidences"):
        assert pa[k].tobytes() == pb[k].tobytes(), (name, k)
    want.close()
    got.close()


def _add_photos(s, ks, scene_dir):
    """The `original` embedding and camera.radial_distortion of every view, as sfmrecon leaves them."""
    from mve_b200 import synth
    for v in range(s.n_views):
        vd = os.path.join(scene_dir, "views", "view_%04d.mve" % v)
        synth.write_mvei(os.path.join(vd, "original.mvei"), s.images[v])
        meta = os.path.join(vd, "meta.ini")
        txt = open(meta).read().replace("[camera]\n", "[camera]\nradial_distortion = %s %s\n" %
                                        tuple(repr(float(np.float32(k))) for k in ks[v]), 1)
        open(meta, "w").write(txt)


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built (needs the reference sources at build time)")
@pytest.mark.parametrize("name", ["T0", "T5"])
def test_cli_undistorts_original_photos(name):
    from mve_b200 import synth
    s = golden_scene(name)
    ks = _coefficients(s)
    with tempfile.TemporaryDirectory() as a, tempfile.TemporaryDirectory() as b:
        synth.write_mve_scene(_undistorted_scene(s, ks), a)
        synth.write_mve_scene(s, b)
        _add_photos(s, ks, b)
        common = ["-s%d" % s.scale, "--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--keep-dz",
                  "--progress=silent", "--force"]
        env = dict(os.environ)
        env.pop("B200MVS_UNDISTORT", None)
        r = subprocess.run([CLI] + common + [a], capture_output=True, text=True, timeout=600, env=env)
        assert r.returncode == 0, r.stdout + r.stderr
        r = subprocess.run([CLI] + common + ["-i", "original", b], capture_output=True, text=True, timeout=600,
                           env=dict(env, B200MVS_UNDISTORT="1"))
        assert r.returncode == 0, r.stdout + r.stderr
        n = 0
        for v in range(s.n_views):
            files = ["depth-L%d.mvei" % s.scale, "conf-L%d.mvei" % s.scale, "dz-L%d.mvei" % s.scale]
            va, vb = (os.path.join(d, "views", "view_%04d.mve" % v) for d in (a, b))
            if s.scale:
                files += [f for f in os.listdir(va) if f.startswith("undist-L%d" % s.scale)]
            for f in files:
                assert open(os.path.join(va, f), "rb").read() == open(os.path.join(vb, f), "rb").read(), (name, v, f)
                n += 1
        assert n >= 3 * s.n_views
