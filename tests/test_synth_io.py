"""On-disk layout the path must not change (SURVEY.md §8b): MVEI container, view directory, bundle file."""
import os
import struct
import tempfile

import numpy as np

from mve_b200 import synth


def test_mvei_header_and_roundtrip():
    """tests/mve/gtest_image_io.cc:301-344 (byte/float round trip + headers) restated for our writer."""
    with tempfile.TemporaryDirectory() as tmp:
        for arr in (np.arange(2 * 3 * 3, dtype=np.uint8).reshape(2, 3, 3), np.linspace(0, 1, 10, dtype=np.float32).reshape(5, 2, 1)):
            p = os.path.join(tmp, "x.mvei")
            synth.write_mvei(p, arr)
            raw = open(p, "rb").read()
            assert raw[:11] == b"\x89MVE_IMAGE\n"
            w, h, c, t = struct.unpack("<4i", raw[11:27])
            assert (h, w, c) == arr.shape and t == (1 if arr.dtype == np.uint8 else 9)
            assert (synth.read_mvei(p) == arr).all()


def test_scene_layout_and_determinism():
    s = synth.make_scene("T0")
    s2 = synth.make_scene("T0")
    assert all((a == b).all() for a, b in zip(s.images, s2.images))
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        assert os.path.exists(os.path.join(tmp, "synth_0.out"))
        for v in range(s.n_views):
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            assert os.path.exists(os.path.join(vd, "meta.ini")) and os.path.exists(os.path.join(vd, "undistorted.mvei"))
        hdr = open(os.path.join(tmp, "synth_0.out")).read().split("\n")
        assert hdr[0] == "drews 1.0" and hdr[1] == "%d %d" % (s.n_views, len(s.feat_pos))
    # cameras: rotation orthonormal, K K^-1 = I (tests/mve/gtest_camera.cc:9-30)
    for v in range(s.n_views):
        R = s.rot[v].reshape(3, 3).astype(np.float64)
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-6)


def test_npz_roundtrip():
    s = synth.make_scene("T0")
    with tempfile.TemporaryDirectory() as tmp:
        p = os.path.join(tmp, "s.npz")
        synth.save_scene_npz(s, p)
        t = synth.load_scene_npz(p)
    assert all((a == b).all() for a, b in zip(s.images, t.images))
    assert (s.rot == t.rot).all() and (s.trans == t.trans).all() and (s.feat_pos == t.feat_pos).all()
    assert all((a == b).all() for a, b in zip(s.feat_refs, t.feat_refs))


def test_npz_roundtrip_mixed_sizes():
    """T6 has views of two sizes: they are stored one by one and each keeps its own size; a scene of one size keeps the
    stacked `images` array."""
    s = synth.make_scene("T6")
    with tempfile.TemporaryDirectory() as tmp:
        p = os.path.join(tmp, "s.npz")
        synth.save_scene_npz(s, p)
        t = synth.load_scene_npz(p)
        assert "images" not in np.load(p).files
        synth.save_scene_npz(synth.make_scene("T0"), p)
        assert "images" in np.load(p).files
    assert all(a.shape == b.shape and (a == b).all() for a, b in zip(s.images, t.images))
    assert (s.width, s.height) == (t.width, t.height)
    assert [s.size(v) for v in range(s.n_views)] == [t.size(v) for v in range(t.n_views)]
    assert [t.images[v].shape[1::-1] for v in range(t.n_views)] == [t.size(v) for v in range(t.n_views)]
    assert (s.flen == t.flen).all() and (s.paspect == t.paspect).all() and (s.ppoint == t.ppoint).all()
    assert (s.rot == t.rot).all() and (s.trans == t.trans).all() and (s.feat_pos == t.feat_pos).all()
    assert all((a == b).all() for a, b in zip(s.feat_refs, t.feat_refs))
