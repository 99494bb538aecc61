"""Argument checks of the device-memory entry points that come before any device work, so they hold without a GPU: on a
planning context (B200MVS_DEVICE_NONE) b200mvs_reconstruct_device fails in require_device with B200MVS_ERR_CUDA,
b200mvs_get_level_device gives the level's size without a buffer and fails as b200mvs_get_level does with one, and a NULL
context, settings or maps_dev is B200MVS_ERR_INVALID_ARG."""
import ctypes as C

import numpy as np
import pytest

from tests.util import golden_scene


@pytest.fixture(scope="module")
def planning():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene(s.n_views, device=dmrecon.DEVICE_NONE)
    for v in range(s.n_views):
        sc.set_view_camera(v, s.width, s.height, s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    sc.set_features(s.feat_pos, s.feat_refs)
    yield s, sc
    sc.close()


def test_reconstruct_device_needs_a_device(planning):
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    st = dmrecon.Settings(scale=s.scale)
    refs = (C.c_int32 * 2)(0, 1)
    maps = (dmrecon._Maps * 2)()
    failed = C.c_int32(-1)
    rc = L.b200mvs_reconstruct_device(sc._h, C.byref(st), 2, refs, maps, None, None, None, C.byref(failed))
    msg = L.b200mvs_last_error(None).decode()
    assert rc == dmrecon.ERR_CUDA and "planning context" in msg, msg
    assert failed.value == -1 and maps[0].width == 0
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.reconstruct(st, [0, 1], on_device=True)
    assert e.value.code == dmrecon.ERR_CUDA


def test_null_arguments(planning):
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    st = dmrecon.Settings(scale=s.scale)
    refs = (C.c_int32 * 1)(0)
    maps = (dmrecon._Maps * 1)()
    assert L.b200mvs_reconstruct_device(None, C.byref(st), 1, refs, maps, None, None, None, None) == dmrecon.ERR_INVALID_ARG
    assert L.b200mvs_reconstruct_device(sc._h, None, 1, refs, maps, None, None, None, None) == dmrecon.ERR_INVALID_ARG
    assert "settings is NULL" in L.b200mvs_last_error(None).decode()
    assert L.b200mvs_reconstruct_device(sc._h, C.byref(st), 1, refs, None, None, None, None, None) == dmrecon.ERR_INVALID_ARG
    assert "maps_dev is NULL" in L.b200mvs_last_error(None).decode()


def test_get_level_device_on_planning_context(planning):
    from mve_b200 import dmrecon
    s, sc = planning
    L = dmrecon.lib()
    for level in range(sc.num_levels(0)):
        w, h, wd, hd = C.c_int(), C.c_int(), C.c_int(), C.c_int()
        assert L.b200mvs_get_level(sc._h, 0, level, C.byref(w), C.byref(h), None) == 0
        assert L.b200mvs_get_level_device(sc._h, 0, level, C.byref(wd), C.byref(hd), None, None) == 0
        assert (wd.value, hd.value) == (w.value, h.value) and w.value > 0
    buf = np.zeros(s.width * s.height * 3, np.uint8)
    rc_host = L.b200mvs_get_level(sc._h, 0, 0, None, None, buf.ctypes.data_as(C.c_void_p))
    msg_host = L.b200mvs_last_error(None).decode()
    rc_dev = L.b200mvs_get_level_device(sc._h, 0, 0, None, None, buf.ctypes.data_as(C.c_void_p), None)
    msg_dev = L.b200mvs_last_error(None).decode()
    assert rc_host < 0 and (rc_dev, msg_dev) == (rc_host, msg_host)
    assert not buf.any()
