"""b200mvs_set_view_prior_state and b200mvs_set_view_prior_state_device without a GPU: the exported symbols and their
ctypes signatures, the argument checks a planning context (B200MVS_DEVICE_NONE) makes before anything is copied, with
the named messages, NULL clearing, and the ValueErrors of Scene.set_view_prior's dz and view_ids."""
import ctypes as C

import numpy as np
import pytest

from tests.util import golden_scene

INVALID = -1
SS = "b200mvs_set_view_prior_state"
SSD = "b200mvs_set_view_prior_state_device"
FAKE = 1 << 40                    # a fake device address; nothing at or after it is read


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


def test_symbols_and_signatures():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    assert SS in dmrecon.EXPORTS and SSD in dmrecon.EXPORTS
    assert L.b200mvs_set_view_prior_state.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                       C.c_int, C.c_int]
    assert L.b200mvs_set_view_prior_state_device.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                              C.c_int, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int,
                                                              C.c_void_p]


def _p(x):
    return None if x is None else C.c_void_p(x)


def _host(L, h, view, depth, dz, ids, w, hh, stride):
    return L.b200mvs_set_view_prior_state(h, view, _p(depth), _p(dz), _p(ids), w, hh, stride)


def _dev(L, h, view, depth, dz, ids, w, hh, stride):
    return L.b200mvs_set_view_prior_state_device(h, view, _p(depth), _p(dz), _p(ids), w, hh, 4 * w, 8 * w, 16 * w,
                                                 stride, None)


# (name, (view, depth, dz, ids, w, h, stride), message with {dz} / {ids} for the form's field names)
CASES = [
    ("negative view", (-1, FAKE, FAKE, FAKE, 4, 4, 1), "view_id is -1, not in 0..%d"),
    ("view past the end", ("n", FAKE, None, FAKE, 4, 4, 1), "view_id is %d, not in 0..%d"),
    ("null prior, bad view", ("n", None, None, None, 0, 0, 0), "view_id is %d, not in 0..%d"),
    ("width", (0, FAKE, FAKE, None, 0, 4, 1), "w is 0, must be at least 1"),
    ("height", (1, FAKE, None, None, 4, -2, 1), "h is -2, must be at least 1"),
    ("stride 0", (2, FAKE, FAKE, FAKE, 4, 4, 0), "stride is 0, not in 1..65535"),
    ("stride too large", (2, FAKE, FAKE, FAKE, 4, 4, 65536), "stride is 65536, not in 1..65535"),
    ("dz without depth", (0, None, FAKE, None, 4, 4, 1), "{dz} is given without a depth map"),
    ("ids without depth", (0, None, None, FAKE, 4, 4, 1), "{ids} is given without a depth map"),
    ("both without depth", (0, None, FAKE, FAKE, 4, 4, 1), "{dz} is given without a depth map"),
    ("planning context", (0, FAKE, FAKE, FAKE, 4, 4, 65535),
     "depth cannot be stored by a planning context (B200MVS_DEVICE_NONE), which has no device"),
]


@pytest.mark.parametrize("form", ["host", "device"])
@pytest.mark.parametrize("name,args,msg", CASES, ids=[c[0] for c in CASES])
def test_checks_name_the_function_and_field(planning, form, name, args, msg):
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    n = s.n_views
    view = n if args[0] == "n" else args[0]
    if "%d" in msg:
        msg = msg % ((n, n - 1) if msg.count("%d") == 2 else (n - 1,))
    msg = msg.format(dz="dz" if form == "host" else "dz_dev", ids="view_ids" if form == "host" else "view_ids_dev")
    rc = (_host if form == "host" else _dev)(L, sc._h, view, *args[1:])
    assert (rc, L.b200mvs_last_error(sc._h).decode()) == (INVALID, "%s: %s" % (SS if form == "host" else SSD, msg))


def test_null_context():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    assert _host(L, None, 0, FAKE, FAKE, FAKE, 4, 4, 1) == INVALID
    assert L.b200mvs_last_error(None).decode() == "%s: null context" % SS
    assert _dev(L, None, 0, FAKE, None, None, 4, 4, 1) == INVALID
    assert L.b200mvs_last_error(None).decode() == "%s: null context" % SSD


def test_null_clears_and_leaves_working_sets(planning):
    """NULL planes are accepted anywhere, with the sizes and pitches not looked at; the working set is unchanged."""
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    want = sc.working_set(st, [0, 1])
    assert _host(L, sc._h, 0, None, None, None, -5, 0, -9) == 0
    assert L.b200mvs_set_view_prior_state_device(sc._h, 1, None, None, None, -5, 0, -3, -1, 7, 0, None) == 0
    sc.set_view_prior(0, None, stride=4)
    assert sc.working_set(st, [0, 1]) == want
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.set_view_prior(0, np.ones((4, 4), np.float32), stride=4, dz=np.zeros((4, 4, 2), np.float32))
    assert e.value.code == dmrecon.ERR_INVALID_ARG and "planning context" in str(e.value) and SS in str(e.value)
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.set_view_prior(0, np.ones((4, 4), np.float32), stride=4, view_ids=np.full((4, 4, 4), -1, np.int32))
    assert SS in str(e.value)


def test_python_rejects_bad_planes(planning):
    import torch
    s, sc = planning
    d = np.ones((4, 5), np.float32)
    good_dz, good_ids = np.zeros((4, 5, 2), np.float32), np.full((4, 5, 4), -1, np.int32)
    for bad_dz in (np.zeros((4, 5, 2), np.float64), np.zeros((4, 5), np.float32), np.zeros((5, 4, 2), np.float32),
                   np.zeros((4, 5, 3), np.float32), np.zeros((4, 5, 2), np.int32)):
        with pytest.raises(ValueError):
            sc.set_view_prior(0, d, 2, dz=bad_dz, view_ids=good_ids)
    for bad_ids in (np.zeros((4, 5, 4), np.int64), np.zeros((4, 5, 4), np.float32), np.zeros((4, 5), np.int32),
                    np.zeros((4, 4, 4), np.int32), np.zeros((4, 5, 2), np.int32)):
        with pytest.raises(ValueError):
            sc.set_view_prior(0, d, 2, dz=good_dz, view_ids=bad_ids)
    # planes without a depth
    for kw in ({"dz": good_dz}, {"view_ids": good_ids}):
        with pytest.raises(ValueError):
            sc.set_view_prior(0, None, 2, **kw)
    # on the device every plane is a CUDA tensor: numpy arrays and CPU tensors are refused before any library call
    td = torch.ones((4, 5))
    for kw in ({"dz": good_dz}, {"view_ids": good_ids}, {"dz": torch.zeros((4, 5, 2))},
               {"view_ids": torch.full((4, 5, 4), -1, dtype=torch.int32)}):
        with pytest.raises(ValueError):
            sc.set_view_prior(0, td, 2, on_device=True, **kw)
