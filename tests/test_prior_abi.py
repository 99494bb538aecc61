"""b200mvs_set_view_prior and b200mvs_set_view_prior_device without a GPU: the exported symbols and their ctypes
signatures, the argument checks a planning context (B200MVS_DEVICE_NONE) makes before anything is copied, with the named
messages, and the seed rule of tests/prior_reference.py on edge shapes."""
import ctypes as C

import numpy as np
import pytest

from tests.prior_reference import prior_cells, prior_seeds
from tests.util import golden_scene

INVALID = -1
SV = "b200mvs_set_view_prior"
SD = "b200mvs_set_view_prior_device"
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
    assert SV in dmrecon.EXPORTS and SD in dmrecon.EXPORTS
    assert L.b200mvs_set_view_prior.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int]
    assert L.b200mvs_set_view_prior_device.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int64,
                                                        C.c_int, C.c_void_p]


def _host(L, h, view, ptr, w, hh, stride):
    return L.b200mvs_set_view_prior(h, view, None if ptr is None else C.c_void_p(ptr), w, hh, stride)


def _dev(L, h, view, ptr, w, hh, stride, pitch=None):
    return L.b200mvs_set_view_prior_device(h, view, None if ptr is None else C.c_void_p(ptr), w, hh,
                                           4 * w if pitch is None else pitch, stride, None)


CASES = [
    ("negative view", (-1, FAKE, 4, 4, 1), "view_id is -1, not in 0..%d"),
    ("view past the end", ("n", FAKE, 4, 4, 1), "view_id is %d, not in 0..%d"),
    ("null prior, bad view", ("n", None, 0, 0, 0), "view_id is %d, not in 0..%d"),
    ("width", (0, FAKE, 0, 4, 1), "w is 0, must be at least 1"),
    ("height", (1, FAKE, 4, -2, 1), "h is -2, must be at least 1"),
    ("stride 0", (2, FAKE, 4, 4, 0), "stride is 0, not in 1..65535"),
    ("stride too large", (2, FAKE, 4, 4, 65536), "stride is 65536, not in 1..65535"),
    ("planning context", (0, FAKE, 4, 4, 65535),
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
    rc = (_host if form == "host" else _dev)(L, sc._h, view, *args[1:])
    assert (rc, L.b200mvs_last_error(sc._h).decode()) == (INVALID, "%s: %s" % (SV if form == "host" else SD, msg))


def test_null_context():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    assert _host(L, None, 0, FAKE, 4, 4, 1) == INVALID
    assert L.b200mvs_last_error(None).decode() == "%s: null context" % SV
    assert _dev(L, None, 0, FAKE, 4, 4, 1) == INVALID
    assert L.b200mvs_last_error(None).decode() == "%s: null context" % SD


def test_null_prior_clears_and_leaves_working_sets(planning):
    """NULL is accepted anywhere, with the sizes not looked at; a view without a prior gives today's working set."""
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    want = sc.working_set(st, [0, 1])
    n, groups = sc.plan_batches(st, [0, 1], want)
    assert _host(L, sc._h, 0, None, -5, 0, -9) == 0
    assert _dev(L, sc._h, 1, None, -5, 0, 0, pitch=-3) == 0
    sc.set_view_prior(0, None, stride=4)
    assert sc.working_set(st, [0, 1]) == want
    n2, groups2 = sc.plan_batches(st, [0, 1], want)
    assert n2 == n and list(groups2) == list(groups)
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.set_view_prior(0, np.ones((4, 4), np.float32), stride=4)
    assert e.value.code == dmrecon.ERR_INVALID_ARG and "planning context" in str(e.value)


def test_python_rejects_bad_priors(planning):
    import torch
    s, sc = planning
    for bad in (np.ones((4, 4), np.float64), np.ones((2, 4, 4), np.float32), np.ones((4, 4), np.uint8)):
        with pytest.raises(ValueError):
            sc.set_view_prior(0, bad, stride=2)
    for bad in (np.ones((4, 4), np.float32), torch.ones((4, 4)), [[1.0, 2.0]]):
        with pytest.raises(ValueError):
            sc.set_view_prior(0, bad, stride=2, on_device=True)


@pytest.mark.parametrize("n,stride,want", [(0, 1, 0), (4, 1, 0), (5, 1, 1), (5, 7, 1), (6, 1, 2), (9, 2, 3), (10, 2, 3),
                                           (11, 3, 3), (100, 200, 1), (65535, 1, 65531)])
def test_candidate_cells(n, stride, want):
    assert prior_cells(n, stride) == want


def test_reference_edge_shapes():
    one = np.full((1, 1), 3.5, np.float32)
    # maps below 5 px have no candidate in that direction
    assert prior_seeds(4, 100, one, 1) == [] and prior_seeds(100, 4, one, 1) == []
    # a 1 x 1 prior gives every candidate its value
    got = prior_seeds(7, 6, one, 1)
    assert got == [(x, y, 3.5) for y in (2, 3) for x in (2, 3, 4)]
    # stride larger than the map: the one candidate (2, 2)
    assert prior_seeds(9, 13, one, 50) == [(2, 2, 3.5)]
    # odd sizes: the prior pixel under each candidate centre, by (2x+1) w // 2W
    rng = np.random.default_rng(3)
    prior = rng.uniform(1, 2, (5, 7)).astype(np.float32)
    got = prior_seeds(13, 11, prior, 3)
    assert [(x, y) for x, y, _ in got] == [(x, y) for y in (2, 5, 8) for x in (2, 5, 8)]
    for x, y, d in got:
        assert d == prior[(2 * y + 1) * 5 // 22, (2 * x + 1) * 7 // 26]
    # invalid values and masked pixels seed nothing
    bad = np.array([[0.0, -1.0], [np.nan, np.inf]], np.float32)
    assert prior_seeds(40, 40, bad, 1) == []
    mask = np.zeros((2, 2), np.uint8)
    mask[1, 1] = 255
    got = prior_seeds(10, 10, one, 1, mask)
    assert got and all(x >= 5 and y >= 5 for x, y, _ in got)
    # a prior of the map's size maps one to one
    full = rng.uniform(1, 2, (9, 11)).astype(np.float32)
    assert all(d == full[y, x] for x, y, d in prior_seeds(11, 9, full, 2))
