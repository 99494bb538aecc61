"""Argument checks of b200mvs_pset_add_reconstruction that come before any device work, so they hold without a GPU: a
missing context and a planning context (B200MVS_DEVICE_NONE) are rejected with B200MVS_ERR_INVALID_ARG and a message."""
import ctypes as C

import pytest

from tests.util import golden_scene


def test_null_context_rejected():
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    L = D._pset_lib()
    assert L.b200mvs_pset_add_reconstruction(None, None, None, 0, None, None, None, None, None) == dmrecon.ERR_INVALID_ARG
    assert "null context" in L.b200mvs_last_error(None).decode()


@pytest.mark.parametrize("through", ["python", "abi"])
def test_planning_context_rejected(through):
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene(s.n_views, device=dmrecon.DEVICE_NONE)
    for v in range(s.n_views):
        sc.set_view_camera(v, s.width, s.height, s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    sc.set_features(s.feat_pos, s.feat_refs)
    st = dmrecon.Settings(scale=s.scale)
    if through == "python":
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.reconstruct_pointset(st, [0, 1])
        code, msg = e.value.code, str(e.value)
    else:
        L = D._pset_lib()
        refs = (C.c_int32 * 2)(0, 1)
        failed = C.c_int32(7)
        code = L.b200mvs_pset_add_reconstruction(None, sc._h, C.byref(st), 2, refs, None, None, C.byref(failed), None)
        msg = L.b200mvs_last_error(None).decode()
        assert failed.value == -1
    assert code == dmrecon.ERR_INVALID_ARG and "planning context" in msg, msg
    sc.close()
