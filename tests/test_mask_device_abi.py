"""The argument checks of b200mvs_set_view_mask_device and b200mvs_pset_clip_masks_device that come before any device call,
with their exact codes and messages from both error getters, on a machine without a GPU: the mask pointers are never
dereferenced.  A planning context (B200MVS_DEVICE_NONE) stands in for a context; a NULL mask clears either kind of mask
anywhere, and the host mask it clears is gone from the views' reconstruction."""
import ctypes as C

import numpy as np
import pytest

from tests.util import golden_scene

INVALID = -1
SV = "b200mvs_set_view_mask_device"
CM = "b200mvs_pset_clip_masks_device"
FAKE = 1 << 40                    # a fake device address; nothing at or after it is read


def _expect(L, rc, msg):
    from mve_b200 import depthmap as D
    D._lib()                      # the depth-map error getter's return type
    assert (rc, L.b200mvs_last_error(None).decode()) == (INVALID, msg)
    assert L.b200mvs_depthmap_last_error().decode() == msg


@pytest.fixture(scope="module")
def planning():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene(s.n_views, device=dmrecon.DEVICE_NONE)
    for v in range(s.n_views):
        sc.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    sc.set_features(s.feat_pos, s.feat_refs)
    yield s, sc
    sc.close()


def _set(L, h, view, ptr, w, h_, pitch):
    return L.b200mvs_set_view_mask_device(h, view, None if ptr is None else C.c_void_p(ptr), w, h_, pitch, None)


def test_symbols_exported():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    assert hasattr(L, SV) and hasattr(L, CM)


def test_set_view_mask_device_null_context():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    _expect(L, _set(L, None, 0, FAKE, 4, 4, 4), "%s: null context" % SV)


SET_CASES = [
    ("negative view", (-1, FAKE, 4, 4, 4), "view_id is -1, not in 0..%d"),
    ("view past the end", ("n", FAKE, 4, 4, 4), "view_id is %d, not in 0..%d"),
    ("null mask, bad view", ("n", None, 0, 0, 0), "view_id is %d, not in 0..%d"),
    ("width", (0, FAKE, 0, 4, 4), "w is 0, must be at least 1"),
    ("height", (1, FAKE, 4, -2, 4), "h is -2, must be at least 1"),
    ("pitch", (2, FAKE, 8, 3, 7), "row_pitch is 7, less than w (8)"),
    ("negative pitch", (2, FAKE, 1, 1, -1), "row_pitch is -1, less than w (1)"),
    ("planning context", (0, FAKE, 4, 4, 4),
     "mask_dev cannot be read by a planning context (B200MVS_DEVICE_NONE), which has no device"),
]


@pytest.mark.parametrize("name,args,msg", SET_CASES, ids=[c[0] for c in SET_CASES])
def test_set_view_mask_device_errors(planning, name, args, msg):
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    n = s.n_views
    view = n if args[0] == "n" else args[0]
    if "%d" in msg:
        msg = msg % ((n, n - 1) if msg.count("%d") == 2 else (n - 1,))
    _expect(L, _set(L, sc._h, view, *args[1:]), "%s: %s" % (SV, msg))


def test_null_mask_clears_either_call(planning):
    """NULL to the device call clears a host mask (no device needed), with the sizes not looked at; so does NULL to the host
    call.  A cleared mask leaves working sets as they were."""
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    want = sc.working_set(st, [0, 1])
    sc.set_view_mask(0, np.zeros((7, 5), np.uint8))
    assert _set(L, sc._h, 0, None, -5, 0, -9) == 0
    sc.set_view_mask(1, np.ones((3, 3), np.uint8))
    assert L.b200mvs_set_view_mask(sc._h, 1, None, 0, 0) == 0
    sc.set_view_mask(0, None, on_device=True)
    assert sc.working_set(st, [0, 1]) == want


def test_python_rejects_host_masks_on_device(planning):
    import torch
    s, sc = planning
    for bad in (np.ones((4, 4), np.uint8), torch.ones((4, 4), dtype=torch.uint8), [[1, 2], [3, 4]]):
        with pytest.raises(ValueError):
            sc.set_view_mask(0, bad, on_device=True)


def _clip(L, ps, n, masks, ws, hs, pitches, cams):
    nf = C.c_uint64(77)
    rc = L.b200mvs_pset_clip_masks_device(ps, n, masks, ws, hs, pitches, cams, None, C.byref(nf))
    assert nf.value == 77
    return rc


def test_clip_masks_device_null_arguments():
    """Without a handle (none can be made without a device), every call is rejected first for the handle, as the host
    call is; a negative count too."""
    from mve_b200 import depthmap as D
    L = D._pset_lib()
    ptrs = (C.c_void_p * 1)(FAKE)
    w = np.array([4], np.int32)
    p = np.array([4], np.int64)
    cams = (D._PsetCamera * 1)()
    cams[0].flen = 1.0
    for n, args in ((1, (ptrs, D._p(w), D._p(w), D._p(p), cams)), (-1, (None,) * 5), (0, (None,) * 5)):
        _expect(L, _clip(L, None, n, *args), "%s: null argument" % CM)
    rc = L.b200mvs_pset_clip_masks(None, 1, ptrs, D._p(w), D._p(w), cams, None)
    _expect(L, rc, "b200mvs_pset_clip_masks: null argument")


def test_python_rejects_mixed_masks_before_any_call():
    """scene_pointset with CUDA and host masks mixed raises ValueError before it makes a handle (which would need a
    device here)."""
    import torch
    from mve_b200 import depthmap as D

    class FakeCuda:
        is_cuda = True
        device = torch.device("cuda", 0)

    cam = dict(flen=1.0, paspect=1.0, ppoint=(0.5, 0.5), rot=np.eye(3), trans=np.zeros(3))
    masks = [dict(mask=np.ones((4, 4), np.uint8), camera=cam), dict(mask=FakeCuda(), camera=cam)]
    with pytest.raises(ValueError, match="not a mix"):
        D.scene_pointset([], masks=masks)
    with pytest.raises(ValueError, match="device"):
        D.scene_pointset([], masks=masks[1:], device=1)
