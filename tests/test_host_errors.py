"""The error rules of the library's host code: every argument error of the depth-map consumers and the point-set handle
with its exact code and message, one message for b200mvs_last_error and b200mvs_depthmap_last_error, and device memory of
depthmap.cu taken and given back in one place.  The checks that come before any device work hold without a GPU; those
that need a handle or a context are marked gpu."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests.util import ROOT, golden_scene

INVALID = -1
OVERFLOW = -5


def _lib():
    from mve_b200 import depthmap as D
    return D._pset_lib()


def _messages(L):
    return L.b200mvs_last_error(None).decode(), L.b200mvs_depthmap_last_error().decode()


def _expect(L, rc, code, msg):
    ctx_msg, dm_msg = _messages(L)
    assert (rc, ctx_msg) == (code, msg)
    assert dm_msg == ctx_msg


def _pointset_args(depth=True, invproj=True, w=4, h=4, color=None, cch=0, counts=True, conf_iterations=4, cap=1 << 20):
    dm = np.ones((max(h, 1), max(w, 1)), np.float32)
    ip = np.eye(3, dtype=np.float32).reshape(9)
    nv, nf = C.c_uint64(0), C.c_uint64(0)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)          # noqa: E731
    return (0, p(dm) if depth else None, w, h, p(ip) if invproj else None, 5.0, None, p(color), cch,
            None, None, None, None, None, None, conf_iterations, None, 0.0, cap, cap,
            C.byref(nv) if counts else None, C.byref(nf) if counts else None, None), (dm, ip, nv, nf, color)


def _pointset(L, **kw):
    args, keep = _pointset_args(**kw)
    return L.b200mvs_depthmap_pointset(*args)


def _triangulate(L, **kw):
    args, keep = _pointset_args(**kw)
    # b200mvs_depthmap_triangulate: the arguments of b200mvs_depthmap_pointset without normals, confidences and scales
    return L.b200mvs_depthmap_triangulate(*(args[:13] + args[18:]))


_COLOR = np.zeros((4, 4, 5), np.uint8)
_DM = np.ones((4, 4), np.float32)
_P = lambda a: a.ctypes.data_as(C.c_void_p)                                    # noqa: E731

# (entry point call, code, message): every argument error that comes before a device call
HOST_ONLY = [
    ("confidence_clean null depth", lambda L: L.b200mvs_depthmap_confidence_clean(0, None, _P(_DM), 4, 4),
     INVALID, "Null depth or confidence map"),
    ("confidence_clean null conf", lambda L: L.b200mvs_depthmap_confidence_clean(0, _P(_DM), None, 4, 4),
     INVALID, "Null depth or confidence map"),
    ("confidence_clean width", lambda L: L.b200mvs_depthmap_confidence_clean(0, _P(_DM), _P(_DM), 0, 4),
     INVALID, "Image dimensions do not match"),
    ("confidence_clean height", lambda L: L.b200mvs_depthmap_confidence_clean(0, _P(_DM), _P(_DM), 4, 0),
     INVALID, "Image dimensions do not match"),
    ("cleanup null depth", lambda L: L.b200mvs_depthmap_cleanup(0, None, 4, 4, 1, _P(_DM)), INVALID, "depthmap_cleanup"),
    ("cleanup null out", lambda L: L.b200mvs_depthmap_cleanup(0, _P(_DM), 4, 4, 1, None), INVALID, "depthmap_cleanup"),
    ("cleanup width", lambda L: L.b200mvs_depthmap_cleanup(0, _P(_DM), 0, 4, 1, _P(_DM)), INVALID, "depthmap_cleanup"),
    ("cleanup height", lambda L: L.b200mvs_depthmap_cleanup(0, _P(_DM), 4, 0, 1, _P(_DM)), INVALID, "depthmap_cleanup"),
    ("cleanup too large", lambda L: L.b200mvs_depthmap_cleanup(0, _P(_DM), 65536, 65536, 1, _P(_DM)), INVALID, "depthmap_cleanup"),
    ("triangulate null depth", lambda L: _triangulate(L, depth=False), INVALID, "Null depthmap given"),
    ("triangulate null invproj", lambda L: _triangulate(L, invproj=False), INVALID, "depthmap_triangulate"),
    ("triangulate null counts", lambda L: _triangulate(L, counts=False), INVALID, "depthmap_triangulate"),
    ("triangulate width", lambda L: _triangulate(L, w=1), INVALID, "depthmap_triangulate"),
    ("triangulate height", lambda L: _triangulate(L, h=1), INVALID, "depthmap_triangulate"),
    ("triangulate colour channels 0", lambda L: _triangulate(L, color=_COLOR, cch=0), INVALID, "Color image dimension mismatch"),
    ("triangulate colour channels 5", lambda L: _triangulate(L, color=_COLOR, cch=5), INVALID, "Color image dimension mismatch"),
    ("pointset null depth", lambda L: _pointset(L, depth=False), INVALID, "Null depthmap given"),
    ("pointset null invproj", lambda L: _pointset(L, invproj=False), INVALID, "depthmap_triangulate"),
    ("pointset null counts", lambda L: _pointset(L, counts=False), INVALID, "depthmap_triangulate"),
    ("pointset width", lambda L: _pointset(L, w=1), INVALID, "depthmap_triangulate"),
    ("pointset height", lambda L: _pointset(L, h=1), INVALID, "depthmap_triangulate"),
    ("pointset colour channels", lambda L: _pointset(L, color=_COLOR, cch=5), INVALID, "Color image dimension mismatch"),
    ("add_view null handle", lambda L: L.b200mvs_pset_add_view(None, 0, _P(_DM), 4, 4, None, 0, None, None),
     INVALID, "b200mvs_pset_add_view: null handle or camera"),
    ("add_view_device null handle", lambda L: L.b200mvs_pset_add_view_device(None, 0, _P(_DM), 4, 4, None, 0, None, None, None),
     INVALID, "b200mvs_pset_add_view_device: null handle or camera"),
    ("clip_masks null handle", lambda L: L.b200mvs_pset_clip_masks(None, 0, None, None, None, None, None),
     INVALID, "b200mvs_pset_clip_masks: null argument"),
    ("get_info null handle", lambda L: L.b200mvs_pset_get_info(None, None), INVALID, "b200mvs_pset_get_info: null argument"),
    ("read null handle", lambda L: L.b200mvs_pset_read(None, None, None, None, None, None), INVALID, "b200mvs_pset_read: null handle"),
    ("read_correspondence null handle", lambda L: L.b200mvs_pset_read_correspondence(None, None, None),
     INVALID, "b200mvs_pset_read_correspondence: null handle"),
    ("read_device null handle", lambda L: L.b200mvs_pset_read_device(None, None, None, None, None, None, None, None),
     INVALID, "b200mvs_pset_read_device: null handle"),
    ("add_reconstruction null context", lambda L: L.b200mvs_pset_add_reconstruction(None, None, None, 0, None, None, None, None, None),
     INVALID, "b200mvs_pset_add_reconstruction: null context"),
]

CREATE_REJECTS = [
    (None, "<fn>: null argument"),
    (dict(with_normals=True, with_conf=True, poisson_normals=True, conf_iterations=0), "Invalid amount of iterations"),
    (dict(with_conf=True, conf_iterations=0), "Invalid amount of iterations"),
    (dict(with_conf=True, conf_iterations=-3), "Invalid amount of iterations"),
    (dict(poisson_normals=True, with_normals=True), "<fn>: poisson_normals needs with_normals and with_conf"),
    (dict(poisson_normals=True, with_conf=True), "<fn>: poisson_normals needs with_normals and with_conf"),
    (dict(correspondence=True, aabb=((0, 0, 0), (1, 1, 1))), "<fn>: correspondence needs every vertex of a view (no bounding box)"),
]


@pytest.mark.parametrize("name,call,code,msg", HOST_ONLY, ids=[c[0] for c in HOST_ONLY])
def test_argument_errors(name, call, code, msg):
    L = _lib()
    _expect(L, call(L), code, msg)


@pytest.mark.parametrize("fn", ["b200mvs_pset_create", "b200mvs_pset_create_on_device"])
@pytest.mark.parametrize("opts,msg", CREATE_REJECTS)
def test_create_rejects(fn, opts, msg):
    from mve_b200 import depthmap as D
    L = _lib()
    h = C.c_void_p(7)
    if opts is None:
        rc = getattr(L, fn)(0, None, C.byref(h))
        _expect(L, rc, INVALID, msg.replace("<fn>", fn))
        rc = getattr(L, fn)(0, C.byref(D._options(None)[1]), None)
        _expect(L, rc, INVALID, msg.replace("<fn>", fn))
        return
    rc = getattr(L, fn)(0, C.byref(D._options(opts)[1]), C.byref(h))
    _expect(L, rc, INVALID, msg.replace("<fn>", fn))
    assert not h.value


def test_planning_context_rejected():
    from mve_b200 import dmrecon
    L = _lib()
    sc = dmrecon.Scene(2, device=dmrecon.DEVICE_NONE)
    try:
        refs = (C.c_int32 * 1)(0)
        st = dmrecon.Settings()
        rc = L.b200mvs_pset_add_reconstruction(None, sc._h, C.byref(st), 1, refs, None, None, None, None)
        _expect(L, rc, INVALID, "b200mvs_pset_add_reconstruction: a planning context (B200MVS_DEVICE_NONE) cannot reconstruct")
    finally:
        sc.close()


def test_one_channel():
    from mve_b200 import dmrecon
    L = _lib()
    # a context call, then a depth-map call, then a context call again: both getters follow the last failing call
    h = C.c_void_p()
    assert L.b200mvs_create(0, 0, C.byref(h)) == dmrecon.ERR_INVALID_ARG
    first = _messages(L)
    assert first[0] == first[1] and first[0].startswith("b200mvs_create"), first
    assert L.b200mvs_pset_read(None, None, None, None, None, None) == dmrecon.ERR_INVALID_ARG
    assert _messages(L) == ("b200mvs_pset_read: null handle",) * 2
    assert L.b200mvs_create(0, 0, C.byref(h)) == dmrecon.ERR_INVALID_ARG
    assert _messages(L) == first


def _function_spans(src, heads):
    spans = []
    for head in heads:
        m = re.search(head, src)
        assert m, head
        depth, i = 1, m.end()
        while depth:
            depth += {"{": 1, "}": -1}.get(src[i], 0)
            i += 1
        spans.append((m.start(), i))
    return spans


def test_cuda_malloc_only_in_the_workspace_and_the_set_store():
    src = open(os.path.join(ROOT, "mve_b200", "csrc", "depthmap.cu")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    work = _function_spans(src, [r"struct Work\s*\{"])[0]
    spans = [(a + work[0], b + work[0]) for a, b in
             _function_spans(src[work[0]:work[1]], [r"cudaError_t need\([^)]*\)\s*\{", r"void drop\([^)]*\)\s*\{"])]
    spans += _function_spans(src, [r"cudaError_t store_alloc\([^)]*\)\s*\{", r"void store_free\([^)]*\)\s*\{"])
    calls = [m.start() for m in re.finditer(r"\bcuda(Malloc|Free)\w*\s*\(", src)]
    assert len(calls) == 4
    assert all(any(a <= c < b for a, b in spans) for c in calls)


# ---- messages that need a handle or a context on the device ----

def _camera(flen=1.0):
    from mve_b200 import depthmap as D
    return D._camera(dict(flen=flen, paspect=1.0, ppoint=(0.5, 0.5), rot=np.eye(3), trans=np.zeros(3)))


def _handle(L, **opts):
    from mve_b200 import depthmap as D
    h = C.c_void_p()
    assert L.b200mvs_pset_create(0, C.byref(D._options(opts)[1]), C.byref(h)) == 0
    return h


def _add_view(L, h, w=8, h_=8, depth=True, flen=1.0, color=None, cch=0):
    dm = np.ones((max(h_, 1), max(w, 1)), np.float32)
    cam = _camera(flen)
    return L.b200mvs_pset_add_view(h, 0, _P(dm) if depth else None, w, h_, None if color is None else _P(color), cch,
                                   C.byref(cam), None)


@pytest.mark.gpu
def test_handle_argument_errors():
    L = _lib()
    h = _handle(L)
    try:
        _expect(L, _add_view(L, h, depth=False), INVALID, "Null depthmap given")
        _expect(L, _add_view(L, h, flen=0.0), INVALID, "Invalid camera given")
        _expect(L, _add_view(L, h, w=1), INVALID, "b200mvs_pset_add_view: depth map size")
        _expect(L, _add_view(L, h, color=np.zeros((8, 8, 5), np.uint8), cch=5), INVALID, "Color image dimension mismatch")
        dm = np.ones((8, 8), np.float32)
        cam = _camera()
        rc = L.b200mvs_pset_add_view_device(h, 0, _P(dm), 8, 8, None, 0, C.byref(cam), None, None)
        _expect(L, rc, INVALID, "b200mvs_pset_add_view_device: depth_dev is pageable host memory, not device memory")
        _expect(L, L.b200mvs_pset_read_correspondence(h, None, None), INVALID,
                "b200mvs_pset_read_correspondence: handle made without correspondence")
        pix = np.zeros(2, np.uint32)
        _expect(L, L.b200mvs_pset_read_device(h, None, None, None, None, None, _P(pix), None), INVALID,
                "b200mvs_pset_read_device: pixels_xy given for a handle made without correspondence")
        nf = C.c_uint64(7)
        assert L.b200mvs_pset_clip_masks(h, 0, None, None, None, None, C.byref(nf)) == 0 and nf.value == 0
        _expect(L, _add_view(L, h), INVALID, "b200mvs_pset_add_view: the masks have been applied already")
        _expect(L, L.b200mvs_pset_clip_masks(h, 0, None, None, None, None, None), INVALID,
                "b200mvs_pset_clip_masks: the masks have been applied already")
    finally:
        L.b200mvs_pset_destroy(h)


@pytest.mark.gpu
def test_add_reconstruction_handle_errors():
    from mve_b200 import dmrecon
    L = _lib()
    s = golden_scene("T0")
    sc = dmrecon.Scene(s.n_views, device=0)
    h = _handle(L)
    try:
        refs = (C.c_int32 * 1)(0)
        st = dmrecon.Settings(scale=s.scale)
        failed = C.c_int32(7)
        rc = L.b200mvs_pset_add_reconstruction(None, sc._h, C.byref(st), 1, refs, None, None, C.byref(failed), None)
        _expect(L, rc, INVALID, "b200mvs_pset_add_reconstruction: null handle")
        assert failed.value == -1
        assert L.b200mvs_pset_clip_masks(h, 0, None, None, None, None, None) == 0
        rc = L.b200mvs_pset_add_reconstruction(h, sc._h, C.byref(st), 1, refs, None, None, None, None)
        _expect(L, rc, INVALID, "b200mvs_pset_add_reconstruction: the masks have been applied already")
    finally:
        L.b200mvs_pset_destroy(h)
        sc.close()


@pytest.mark.gpu
def test_pointset_device_errors():
    L = _lib()
    _expect(L, _pointset(L, conf_iterations=-1), INVALID, "Invalid amount of iterations")
    # a full 4 x 4 map has 16 vertices and 18 faces
    _expect(L, _triangulate(L, cap=15), OVERFLOW, "depthmap_triangulate: output capacity too small")
    _expect(L, _pointset(L, cap=15), OVERFLOW, "depthmap_triangulate: output capacity too small")
