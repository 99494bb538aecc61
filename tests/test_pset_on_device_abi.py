"""Checks of the device-resident point set's C ABI (b200mvs_pset_create_on_device, b200mvs_pset_read_device) that come
before any device work, so they hold without a GPU: both symbols are exported, create_on_device rejects every option set
that b200mvs_pset_create rejects with the same code and message (apart from the function it names), and read_device
rejects a NULL handle."""
import ctypes as C

import pytest

from tests import test_pset_abi

REJECTED = [p for m in test_pset_abi.test_pset_create_rejects.pytestmark if m.name == "parametrize" for p in m.args[1]]


def test_symbols_exported():
    from mve_b200 import depthmap as D
    L = D._pset_lib()
    assert hasattr(L, "b200mvs_pset_create_on_device") and hasattr(L, "b200mvs_pset_read_device")


@pytest.mark.parametrize("opts,msg", REJECTED)
def test_create_on_device_rejects_like_create(opts, msg):
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    L = D._pset_lib()
    _, opt = D._options(opts)
    got = []
    for fn in ("b200mvs_pset_create", "b200mvs_pset_create_on_device"):
        h = C.c_void_p(7)
        rc = getattr(L, fn)(0, C.byref(opt), C.byref(h))
        got.append((rc, L.b200mvs_depthmap_last_error().decode().replace(fn, "<fn>"), h.value))
    assert got[0] == got[1], got
    assert got[1][0] == dmrecon.ERR_INVALID_ARG and msg in got[1][1] and not got[1][2], got


def test_create_on_device_null_arguments():
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    L = D._pset_lib()
    _, opt = D._options(None)
    assert L.b200mvs_pset_create_on_device(0, None, None) == dmrecon.ERR_INVALID_ARG
    assert L.b200mvs_depthmap_last_error().decode() .startswith("b200mvs_pset_create_on_device: null argument")
    assert L.b200mvs_pset_create_on_device(0, C.byref(opt), None) == dmrecon.ERR_INVALID_ARG


def test_read_device_null_handle():
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    L = D._pset_lib()
    assert L.b200mvs_pset_read_device(None, None, None, None, None, None, None, None) == dmrecon.ERR_INVALID_ARG
    assert "b200mvs_pset_read_device: null handle" in L.b200mvs_depthmap_last_error().decode()
