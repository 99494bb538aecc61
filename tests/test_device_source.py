"""The device image source without a GPU: the C declarations and their ctypes bindings, the layout, pitch and overlap rules
of Scene.set_image_source(on_device=True) on shapes and strides alone, and the gather of mve_b200/csrc/undistort.cuh
compiled by g++ over packed, pitched and planar copies of every tests/golden/undistort_ref.npz case, which must give the
fixture's bytes."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest

from tests import undistort_reference as UR
from tests.util import ROOT


def _header():
    return re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200mvs.h")).read(), flags=re.S)


def test_header_declares_the_device_source():
    hdr = " ".join(_header().split())
    assert ("typedef struct b200mvs_device_image { const uint8_t* data; int32_t w, h, channels; int64_t row_pitch; "
            "int64_t plane_pitch; void* cuda_stream; } b200mvs_device_image;") in hdr
    assert "typedef int (*b200mvs_device_fetch_fn)(void* user, int32_t view_id, b200mvs_device_image* out);" in hdr
    assert ("int b200mvs_set_image_source_device(b200mvs_ctx* ctx, b200mvs_device_fetch_fn fetch, b200mvs_release_fn release, "
            "void* user, uint64_t budget_bytes);") in hdr


def test_bindings_match_the_header():
    from mve_b200 import dmrecon
    L = dmrecon.lib()
    assert "b200mvs_set_image_source_device" in dmrecon.EXPORTS
    f = L.b200mvs_set_image_source_device
    assert f.argtypes == [C.c_void_p, dmrecon._DEVICE_FETCH_FN, dmrecon._RELEASE_FN, C.c_void_p, C.c_uint64]
    assert f.argtypes[2] is L.b200mvs_set_image_source.argtypes[2]
    D = dmrecon._DeviceImage
    assert [n for n, _ in D._fields_] == ["data", "w", "h", "channels", "row_pitch", "plane_pitch", "cuda_stream"]
    assert (C.sizeof(D), D.row_pitch.offset, D.plane_pitch.offset, D.cuda_stream.offset) == (48, 24, 32, 40)
    assert dmrecon._DEVICE_FETCH_FN._argtypes_ == (C.c_void_p, C.c_int32, C.POINTER(D))
    assert dmrecon._DEVICE_FETCH_FN._restype_ is C.c_int


def test_layout_of_contiguous_and_pitched_images():
    from mve_b200.dmrecon import device_image_layout as lay
    assert lay((48, 64, 3), (192, 3, 1)) == (48, 64, 3, 192, 0)
    assert lay((48, 64), (64, 1)) == (48, 64, 1, 64, 0)                         # grey H x W
    assert lay((48, 64, 1), (64, 1, 1)) == (48, 64, 1, 64, 0)
    assert lay((48, 64, 4), (300, 4, 1)) == (48, 64, 4, 300, 0)                  # pitched rows
    assert lay((48, 64, 2), (200 * 64, 2, 1)) == (48, 64, 2, 200 * 64, 0)
    assert lay((3, 48, 64), (48 * 64, 64, 1), "chw") == (48, 64, 3, 64, 48 * 64)
    assert lay((3, 48, 64), (60 * 80, 80, 1), "chw") == (48, 64, 3, 80, 60 * 80)  # crop of a larger planar image
    assert lay((4, 48, 64), (48 * 80, 80, 1), "chw") == (48, 64, 4, 80, 48 * 80)
    # the stride of a dimension of size 1 is never used
    assert lay((1, 48, 64), (7, 64, 1), "chw") == (48, 64, 1, 64, 48 * 64)
    assert lay((48, 64, 1), (64, 1, 9)) == (48, 64, 1, 64, 0)
    assert lay((1, 64, 3), (5, 3, 1)) == (1, 64, 3, 192, 0)


@pytest.mark.parametrize("shape, strides, layout, what", [
    ((48, 64, 3), (192, 3, 2), "hwc", "channel stride"),
    ((48, 64, 3), (192, 4, 1), "hwc", "pixel stride"),
    ((48, 64, 3), (191, 3, 1), "hwc", "row stride 191"),
    ((48, 64, 3), (0, 3, 1), "hwc", "row stride 0"),
    ((48, 64), (32, 1), "hwc", "row stride 32"),
    ((48, 64, 3), (64, 3 * 48 * 64, 1), "hwc", "pixel stride"),                 # a CHW tensor permuted to HWC
    ((3, 48, 64), (48 * 64, 64, 2), "chw", "pixel stride"),
    ((3, 48, 64), (48 * 64, 63, 1), "chw", "row stride 63"),
    ((3, 48, 64), (47 * 64, 64, 1), "chw", "overlaps"),
    ((3, 48, 64), (0, 64, 1), "chw", "overlaps"),                                # expanded channels
    ((3, 48, 64), (1, 3 * 64, 3), "chw", "pixel stride"),                       # an HWC tensor permuted to CHW
    ((48, 64, 5), (320, 5, 1), "hwc", "1 to 4 channels, not 5"),
    ((48, 64, 0), (0, 0, 1), "hwc", "1 to 4 channels, not 0"),
    ((5, 48, 64), (48 * 64, 64, 1), "chw", "1 to 4 channels, not 5"),
    ((0, 48, 64), (48 * 64, 64, 1), "chw", "1 to 4 channels, not 0"),
    ((48, 64, 3, 1), (192, 3, 1, 1), "hwc", "H x W x C"),
    ((48, 64), (64, 1), "chw", "C x H x W"),
    ((48, 0, 3), (0, 3, 1), "hwc", "empty"),
    ((48, 64, 3), (192, 3, 1), "whc", "layout"),
])
def test_layout_rejections(shape, strides, layout, what):
    from mve_b200.dmrecon import device_image_layout
    with pytest.raises(ValueError, match=what):
        device_image_layout(shape, strides, layout)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("undistort_layout_emu") / "libundistort_layout_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared",
                           os.path.join(ROOT, "tests", "emu", "undistort_layout_emu.cc"), "-o", lib])
    L = C.CDLL(lib)
    L.emu_undistort_src.argtypes = [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                    C.c_float, C.c_void_p]
    return L


def layouts(img, seed):
    """The image as a device source may hold it: packed HWC, HWC with padded rows, and planar CHW with padded rows and
    planes, the padding filled with noise.  Yields (name, buffer, offset of the first texel, row pitch, plane pitch)."""
    h, w, c = img.shape
    rng = np.random.default_rng(seed)
    yield "packed", np.ascontiguousarray(img).reshape(-1), 0, w * c, 0
    row = w * c + 7
    buf = rng.integers(0, 256, 5 + h * row, dtype=np.uint8)
    buf[5:].reshape(h, row)[:, :w * c] = img.reshape(h, w * c)
    yield "pitched", buf, 5, row, 0
    row, plane = w + 5, (h + 3) * (w + 5) + 1
    buf = rng.integers(0, 256, 3 + c * plane, dtype=np.uint8)
    for k in range(c):
        buf[3 + k * plane:3 + k * plane + h * row].reshape(h, row)[:, :w] = img[:, :, k]
    yield "planar", buf, 3, row, plane


def test_gather_equals_reference_in_every_layout(emu):
    golden = np.load(os.path.join(ROOT, "tests", "golden", "undistort_ref.npz"))
    seen = set()
    for case in UR.cases():
        name, w, h, c, flen, k2, k4, seed = case
        img = UR.make_image(w, h, c, seed)
        for lname, buf, off, row, plane in layouts(img, seed):
            out = np.full_like(img, 0xA5)
            emu.emu_undistort_src(buf.ctypes.data + off, row, plane, w, h, c, flen, k2, k4, out.ctypes.data)
            if k2 == 0 and k4 == 0:
                assert out.tobytes() == img.tobytes(), (name, lname)
            UR.check(golden, case, out)
            seen.add((lname, c))
    assert seen == {(l, c) for l in ("packed", "pitched", "planar") for c in (1, 2, 3, 4)}
