"""b200mvs_set_view_prior_relative and b200mvs_set_view_prior_relative_device without a GPU: the exported symbols and
their ctypes signatures, the argument checks a planning context (B200MVS_DEVICE_NONE) makes before anything is copied,
each naming the function and the field, a NULL context, and the errors of Scene.set_view_prior_relative."""
import ctypes as C

import numpy as np
import pytest

from tests.util import golden_scene

INVALID = -1
SR = "b200mvs_set_view_prior_relative"
SRD = "b200mvs_set_view_prior_relative_device"
FAKE = 1 << 40                    # a fake address; nothing at or after it is read


def _planning(n_extra=0, features=True):
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene(s.n_views + n_extra, device=dmrecon.DEVICE_NONE)
    for v in range(s.n_views):
        sc.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    if features:
        sc.set_features(s.feat_pos, s.feat_refs)
    return s, sc


@pytest.fixture(scope="module")
def planning():
    s, sc = _planning(n_extra=1)          # the last view has no camera
    s2, bare = _planning(features=False)
    yield s, sc, bare
    sc.close()
    bare.close()


def test_symbols_and_signatures():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    assert SR in dmrecon.EXPORTS and SRD in dmrecon.EXPORTS
    assert L.b200mvs_set_view_prior_relative.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                                          C.c_int, C.POINTER(dmrecon.PriorFit)]
    assert L.b200mvs_set_view_prior_relative_device.argtypes == [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                                                 C.c_int64, C.c_int, C.c_int, C.c_void_p,
                                                                 C.POINTER(dmrecon.PriorFit)]
    # b200mvs_prior_fit: two doubles, two uint32, a double
    assert C.sizeof(dmrecon.PriorFit) == 32 and dmrecon.PriorFit.n_obs.offset == 16
    assert dmrecon.PRIOR_KINDS == {"disparity": 0, "depth": 1, "depth_scale": 2}


def _call(L, form, h, view, values, w, hh, stride, kind, pitch=None, fit=None):
    fit = fit if fit is not None else _fit_struct()
    v = None if values is None else C.c_void_p(values)
    if form == "host":
        return L.b200mvs_set_view_prior_relative(h, view, v, w, hh, stride, kind, C.byref(fit))
    return L.b200mvs_set_view_prior_relative_device(h, view, v, w, hh, 4 * w if pitch is None else pitch, stride, kind,
                                                    None, C.byref(fit))


def _fit_struct():
    from mve_b200 import dmrecon
    return dmrecon.PriorFit(scale=7.0, shift=7.0, n_obs=7, n_inliers=7, median_rel_err=7.0)


# (name, context, (view, values, w, h, stride, kind, pitch), message with {values} for the form's field name)
CASES = [
    ("negative view", "sc", (-1, FAKE, 4, 4, 1, 0, None), "view_id is -1, not in 0..%d"),
    ("view past the end", "sc", ("n", FAKE, 4, 4, 1, 0, None), "view_id is %d, not in 0..%d"),
    ("width", "sc", (0, FAKE, 0, 4, 1, 0, None), "w is 0, must be at least 1"),
    ("height", "sc", (1, FAKE, 4, -2, 1, 1, None), "h is -2, must be at least 1"),
    ("stride 0", "sc", (2, FAKE, 4, 4, 0, 2, None), "stride is 0, not in 1..65535"),
    ("stride too large", "sc", (2, FAKE, 4, 4, 65536, 2, None), "stride is 65536, not in 1..65535"),
    ("null values", "sc", (0, None, 4, 4, 1, 0, None), "{values} is NULL"),
    ("kind 3", "sc", (0, FAKE, 4, 4, 1, 3, None), "kind is 3, not a B200MVS_PRIOR_* kind (0..2)"),
    ("kind -1", "sc", (0, FAKE, 4, 4, 1, -1, None), "kind is -1, not a B200MVS_PRIOR_* kind (0..2)"),
    ("view without a camera", "sc", ("last", FAKE, 4, 4, 1, 0, None), "view_id %d has no camera"),
    ("context without features", "bare", (0, FAKE, 4, 4, 1, 0, None),
     "the context has no features (b200mvs_set_features)"),
    ("planning context", "sc", (0, FAKE, 4, 4, 4, 1, None),
     "{values} cannot be read by a planning context (B200MVS_DEVICE_NONE), which has no device"),
]


@pytest.mark.parametrize("form", ["host", "device"])
@pytest.mark.parametrize("name,which,args,msg", CASES, ids=[c[0] for c in CASES])
def test_checks_name_the_function_and_field(planning, form, name, which, args, msg):
    from mve_b200 import dmrecon
    s, sc, bare = planning
    ctx = sc if which == "sc" else bare
    L = dmrecon.lib()
    n = ctx.n_views
    view = {"n": n, "last": n - 1}.get(args[0], args[0])
    if "%d" in msg:
        msg = msg % ((n, n - 1) if msg.count("%d") == 2 else ((n - 1,) if "not in" in msg else (view,)))
    msg = msg.format(values="values" if form == "host" else "values_dev")
    fit = _fit_struct()
    rc = _call(L, form, ctx._h, view, args[1], args[2], args[3], args[4], args[5], args[6], fit)
    assert rc == INVALID
    err = L.b200mvs_last_error(ctx._h).decode()
    fn = SR if form == "host" else SRD
    assert err == "%s: %s" % (fn, msg), err
    # fit_out is cleared before any check
    assert (fit.scale, fit.shift, fit.n_obs, fit.n_inliers, fit.median_rel_err) == (0.0, 0.0, 0, 0, 0.0)


@pytest.mark.parametrize("pitch", [15, 18, -4])
def test_device_row_pitch(planning, pitch):
    from mve_b200 import dmrecon
    s, sc, _ = planning
    L = dmrecon.lib()
    assert _call(L, "device", sc._h, 0, FAKE, 4, 4, 1, 0, pitch) == INVALID
    assert L.b200mvs_last_error(sc._h).decode() == (
        "%s: row_pitch is %d, not a multiple of 4 of at least 4 w (16)" % (SRD, pitch))


@pytest.mark.parametrize("form", ["host", "device"])
def test_null_context(form):
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    fit = _fit_struct()
    assert _call(L, form, None, 0, FAKE, 4, 4, 1, 0, None, fit) == INVALID
    assert L.b200mvs_last_error(None).decode() == "%s: null context" % (SR if form == "host" else SRD)
    # and a NULL fit_out is allowed
    f = L.b200mvs_set_view_prior_relative(None, 0, C.c_void_p(FAKE), 4, 4, 1, 0, None)
    assert f == INVALID


def test_python_errors(planning):
    from mve_b200 import dmrecon
    s, sc, _ = planning
    W, H = s.size(0)
    good = np.ones((H // 4, W // 4), np.float32)
    with pytest.raises(ValueError, match="kind is 'inverse'"):
        sc.set_view_prior_relative(0, good, 4, kind="inverse")
    for bad in (good.astype(np.float64), good[None], np.ones(5, np.float32)):
        with pytest.raises(ValueError, match="H x W float32 array"):
            sc.set_view_prior_relative(0, bad, 4)
    with pytest.raises(ValueError, match="torch.float32 tensor"):
        sc.set_view_prior_relative(0, [[1.0]], 4)
    import torch
    with pytest.raises(ValueError, match="torch.float32 tensor"):
        sc.set_view_prior_relative(0, torch.ones(4, 4), 4)            # a CPU tensor
    # through Python, a planning context's check raises B200MVSError naming the function, with the fit attached
    for kind in dmrecon.PRIOR_KINDS:
        with pytest.raises(dmrecon.B200MVSError, match="%s: values cannot be read by a planning context" % SR) as e:
            sc.set_view_prior_relative(0, good, 4, kind=kind)
        assert e.value.code == INVALID and e.value.fit["n_obs"] == 0
    with pytest.raises(dmrecon.B200MVSError, match="%s: view_id %d has no camera" % (SR, s.n_views)):
        sc.set_view_prior_relative(s.n_views, good, 4)
    with pytest.raises(dmrecon.B200MVSError, match="%s: stride is 0" % SR):
        sc.set_view_prior_relative(0, good, 0)
