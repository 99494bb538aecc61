"""Reconstruction masks on the CPU (b200mvs_set_view_mask in planning contexts): a NumPy restatement of the pixel mapping
that tests/test_gpu_recon_mask.py holds the engine to, the argument checks, and the sizes a mask must leave alone
(b200mvs_working_set, b200mvs_plan_batches and global view selection)."""
from fractions import Fraction

import numpy as np
import pytest

from tests.test_device_budget import _levels
from tests.util import golden_scene


def mask_coords(n, m):
    """Mask column (row) under the centre of each of the n columns (rows) of a map, for a mask m wide (high):
    floor((2x+1) m / 2n) in integers."""
    x = np.arange(n, dtype=np.int64)
    return (2 * x + 1) * m // (2 * n)


def background_map(mask, W, H):
    """H x W bool: True where pixel (x, y) of a W x H map is background under `mask` (h x w uint8, 0 = background)."""
    mask = np.asarray(mask)
    mh, mw = mask.shape
    return mask[mask_coords(H, mh)[:, None], mask_coords(W, mw)[None, :]] == 0


def level_sizes(s, v):
    """(width, height) of every pyramid level of view v: (w+1)/2 per level while min(w, h) >= 30 (image_pyramid.cc:46-47)."""
    return _levels(*s.size(v))


def _centre_pixel(x, n, m):
    """The mask pixel under the centre x + 1/2 of a map column, exactly: floor((x + 1/2) m / n)."""
    return int((Fraction(2 * x + 1, 2) * m / n).__floor__())


@pytest.mark.parametrize("name", ["T0", "T4", "T5", "T6"])
def test_mapping_at_every_level(name):
    """At every level size of every view, odd ones included: a mask of the map's size maps one to one, and a mask of the
    photo's size gives the photo pixel under the level pixel's centre."""
    s = golden_scene(name)
    for v in range(s.n_views):
        w0, h0 = s.size(v)
        for W, H in level_sizes(s, v):
            assert (mask_coords(W, W) == np.arange(W)).all() and (mask_coords(H, H) == np.arange(H)).all()
            cx, cy = mask_coords(W, w0), mask_coords(H, h0)
            assert cx.tolist() == [_centre_pixel(x, W, w0) for x in range(W)], (v, W)
            assert cy.tolist() == [_centre_pixel(y, H, h0) for y in range(H)], (v, H)


@pytest.mark.parametrize("W,H,mw,mh", [(101, 135, 1, 1), (51, 68, 101, 135), (13, 17, 7, 5), (13, 17, 1000, 3),
                                       (90, 90, 179, 180), (3, 2, 65535, 2), (1, 1, 4, 4), (40, 30, 41, 31)])
def test_mapping_masks_larger_and_smaller(W, H, mw, mh):
    """Any mask size: indices stay inside the mask, never decrease, cover both ends fairly and equal the exact centre rule."""
    for n, m in ((W, mw), (H, mh)):
        c = mask_coords(n, m)
        assert c.min() >= 0 and c.max() < m
        assert (np.diff(c) >= 0).all()
        assert c.tolist() == [_centre_pixel(x, n, m) for x in range(n)]
        if m >= n:
            assert len(set(c.tolist())) == n                  # a finer mask gives every map pixel its own mask pixel
        else:
            assert len(set(c.tolist())) == m                  # a coarser one uses every mask pixel


def test_background_map_follows_the_mask():
    rng = np.random.default_rng(3)
    mask = (rng.random((135, 101)) > 0.5).astype(np.uint8) * rng.integers(1, 256, (135, 101)).astype(np.uint8)
    assert (background_map(mask, 101, 135) == (mask == 0)).all()
    half = background_map(mask, 51, 68)
    assert (half == (mask[2 * np.arange(68)[:, None], 2 * np.arange(51)[None, :]] == 0)).all()
    assert not background_map(np.full((5, 5), 7, np.uint8), 33, 44).any()
    assert background_map(np.zeros((1, 1), np.uint8), 33, 44).all()


def _planning(s):
    from mve_b200 import dmrecon
    g = dmrecon.Scene(s.n_views, device=dmrecon.DEVICE_NONE)
    for v in range(s.n_views):
        g.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    g.set_features(s.feat_pos, s.feat_refs)
    return g


def test_set_view_mask_arguments_planning_context():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = _planning(s)
    sc.set_view_mask(0, np.ones((120, 160), np.uint8))        # stores: no device needed
    sc.set_view_mask(1, np.zeros((3, 7), np.uint8))
    sc.set_view_mask(1, None)
    sc.set_view_mask(5, np.ones((1, 1), np.uint8))
    for vid, m in ((-1, np.ones((4, 4), np.uint8)), (s.n_views, np.ones((4, 4), np.uint8)),
                   (0, np.ones((0, 4), np.uint8)), (0, np.ones((4, 0), np.uint8))):
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.set_view_mask(vid, m)
        assert e.value.code == dmrecon.ERR_INVALID_ARG and "b200mvs_set_view_mask: bad arguments" in str(e.value)
    with pytest.raises(dmrecon.B200MVSError):
        sc.set_view_mask(s.n_views, None)
    for bad in (np.ones((4, 4), np.float32), np.ones((4, 4, 1), np.uint8), np.ones(4, np.uint8)):
        with pytest.raises(ValueError):
            sc.set_view_mask(0, bad)
    L = dmrecon.lib()
    m = np.ones((4, 4), np.uint8)
    assert L.b200mvs_set_view_mask(None, 0, m.ctypes.data, 4, 4) == dmrecon.ERR_INVALID_ARG
    assert L.b200mvs_set_view_mask(sc._h, 0, m.ctypes.data, 0, 4) == dmrecon.ERR_INVALID_ARG
    assert L.b200mvs_set_view_mask(sc._h, 0, m.ctypes.data, 4, -1) == dmrecon.ERR_INVALID_ARG
    assert L.b200mvs_set_view_mask(sc._h, 0, None, 0, 0) == 0     # NULL clears; the size is not looked at
    sc.close()


def test_torch_mask_is_accepted():
    import torch
    s = golden_scene("T0")
    sc = _planning(s)
    sc.set_view_mask(0, torch.ones((120, 160), dtype=torch.uint8))
    sc.close()


@pytest.mark.parametrize("name", ["T0", "T2", "T6"])
def test_masks_leave_sizes_and_selection_alone(name):
    """A mask changes nothing a plan or a budget is made from: working sets, groups and the selected views are the same
    with no mask, all-background masks and half-plane masks."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    sc = _planning(s)
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = list(range(s.n_views))

    def sizes():
        ws = [sc.working_set(st, [r]) for r in refs] + [sc.working_set(st, refs)]
        single = max(ws[:-1])
        groups = [sc.plan_batches(st, refs, a)[1].tolist() for a in (single, (single + ws[-1]) // 2, ws[-1])]
        return ws, groups, [sc.global_view_selection(st, r) for r in refs]

    want = sizes()
    for kind in ("zero", "half"):
        for v in refs:
            w, h = s.size(v)
            m = np.zeros((h, w), np.uint8)
            if kind == "half":
                m[:, : w // 2] = 255
            sc.set_view_mask(v, m)
        assert sizes() == want, kind
    sc.close()
