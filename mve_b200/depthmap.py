"""Host-side mirror of the reference's depth-map consumers over the C ABI (include/b200mvs.h):
mve::image::depthmap_confidence_clean / depthmap_cleanup and mve::geom::depthmap_triangulate (libs/mve/depthmap.{h,cc}),
the per-view work of apps/scene2pset, and (scene_pointset) its whole-scene point set.  No CPU fallback: the calls fail without a CUDA device."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import dmrecon

DD_FACTOR_DEFAULT = 5.0      # mve::geom::DD_FACTOR_DEFAULT (libs/mve/depthmap.h)


def _lib():
    L = dmrecon.lib()
    if not getattr(L, "_dm_ready", False):
        L.b200mvs_depthmap_last_error.restype = C.c_char_p
        L.b200mvs_depthmap_confidence_clean.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.b200mvs_depthmap_cleanup.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p]
        L.b200mvs_depthmap_confidence_clean_device.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                               C.c_void_p]
        L.b200mvs_depthmap_cleanup_device.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                      C.c_void_p]
        L.b200mvs_depthmap_triangulate.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int,
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]
        L.b200mvs_depthmap_pointset.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p, C.c_int,
                                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                C.c_float, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200mvs_depthmap_pointset_device.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_int, C.c_float, C.c_void_p]
        L._dm_ready = True
    return L


def _check(rc):
    if rc < 0:
        raise dmrecon.B200MVSError(rc, _lib().b200mvs_depthmap_last_error().decode())


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def depthmap_confidence_clean(dm: np.ndarray, cm: np.ndarray, device: int = 0) -> None:
    """In place: dm = 0 where cm <= 0 (depthmap.cc:118-131).  dm and cm may be torch CUDA tensors (float32, contiguous, on
    one device; `device` is then theirs): see depthmap_confidence_clean_maps."""
    if _is_cuda(dm) or _is_cuda(cm):
        depthmap_confidence_clean_maps([dm], [cm])
        return
    if dm.shape != cm.shape:
        raise ValueError("Image dimensions do not match")
    assert dm.dtype == np.float32 and dm.flags["C_CONTIGUOUS"]
    cm = np.ascontiguousarray(cm, np.float32)
    _check(_lib().b200mvs_depthmap_confidence_clean(device, _p(dm), _p(cm), dm.shape[1], dm.shape[0]))


def depthmap_cleanup(dm: np.ndarray, thres: int, device: int = 0) -> np.ndarray:
    """Islands of dm != 0 smaller than thres pixels removed (depthmap.cc:25-113).  dm may be a torch CUDA tensor (float32,
    contiguous; `device` is then its own): the result is a new CUDA tensor, see depthmap_cleanup_maps."""
    if _is_cuda(dm):
        import torch
        out = torch.empty_like(dm)
        depthmap_cleanup_maps([dm], thres, out=[out])
        return out
    dm = np.ascontiguousarray(dm, np.float32)
    out = np.empty_like(dm)
    _check(_lib().b200mvs_depthmap_cleanup(device, _p(dm), dm.shape[1], dm.shape[0], int(thres), _p(out)))
    return out


def _device_maps(what, maps, dev=None):
    """The device of a sequence of 2-D float32 contiguous CUDA tensors (`dev` if given, else the first one's), else
    ValueError naming `what`[j]."""
    import torch
    for j, t in enumerate(maps):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("%s[%d] must be a CUDA tensor" % (what, j))
        if t.dtype != torch.float32 or t.dim() != 2 or not t.is_contiguous():
            raise ValueError("%s[%d] must be a contiguous 2-D float32 tensor" % (what, j))
        if dev is None:
            dev = t.device
        elif t.device != dev:
            raise ValueError("%s[%d] is on %s, the maps on %s" % (what, j, t.device, dev))
    return dev


def _batch(maps, dev):
    """(device index, map pointers, widths, heights, stream) of a batch of CUDA tensors; the stream is dev's current one."""
    import torch
    if dev is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    ptrs = (C.c_void_p * max(len(maps), 1))(*[t.data_ptr() for t in maps])
    ws = np.array([t.shape[1] for t in maps] or [0], np.int32)
    hs = np.array([t.shape[0] for t in maps] or [0], np.int32)
    return dev.index, ptrs, ws, hs, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def depthmap_confidence_clean_maps(dms, cms) -> None:
    """depthmap_confidence_clean in place on each map of a batch of torch CUDA tensors, e.g. the depth and conf maps of
    Scene.reconstruct(on_device=True): float32, contiguous, H x W, all on one device.  One library call
    (b200mvs_depthmap_confidence_clean_device), ordered after the work of that device's current stream; the maps are
    written when it returns."""
    dms, cms = list(dms), list(cms)
    if len(dms) != len(cms):
        raise ValueError("%d depth maps and %d confidence maps" % (len(dms), len(cms)))
    dev = _device_maps("cms", cms, _device_maps("dms", dms))
    for j, (d, c) in enumerate(zip(dms, cms)):
        if d.shape != c.shape:
            raise ValueError("Image dimensions do not match (map %d)" % j)
    index, dp, ws, hs, stream = _batch(dms, dev)
    cp = (C.c_void_p * max(len(cms), 1))(*[t.data_ptr() for t in cms])
    _check(_lib().b200mvs_depthmap_confidence_clean_device(index, len(dms), dp, cp, _p(ws), _p(hs), stream))


def depthmap_cleanup_maps(dms, thres, out=None):
    """depthmap_cleanup on each map of a batch of torch CUDA tensors (as depthmap_confidence_clean_maps), with thres an int
    or one per map.  out: None (new tensors), or one tensor per map of the same shape on the same device; out=dms cleans
    in place.  One library call (b200mvs_depthmap_cleanup_device) on the device's current stream.  Returns the outputs."""
    import torch
    dms = list(dms)
    dev = _device_maps("dms", dms)
    th = list(thres) if isinstance(thres, (list, tuple, np.ndarray, torch.Tensor)) else [thres] * len(dms)
    if len(th) != len(dms):
        raise ValueError("%d thresholds for %d maps" % (len(th), len(dms)))
    th = np.array([int(t) for t in th] or [0], np.int64)
    outs = [torch.empty_like(d) for d in dms] if out is None else list(out)
    if len(outs) != len(dms):
        raise ValueError("%d outputs for %d maps" % (len(outs), len(dms)))
    _device_maps("out", outs, dev)
    for j, (d, o) in enumerate(zip(dms, outs)):
        if d.shape != o.shape:
            raise ValueError("out[%d] has shape %s, the map %s" % (j, tuple(o.shape), tuple(d.shape)))
    index, dp, ws, hs, stream = _batch(dms, dev)
    op = (C.c_void_p * max(len(outs), 1))(*[t.data_ptr() for t in outs])
    _check(_lib().b200mvs_depthmap_cleanup_device(index, len(dms), dp, _p(ws), _p(hs), _p(th), op, stream))
    return outs


class DmMesh(C.Structure):
    """b200mvs_dm_mesh (include/b200mvs.h): one map of b200mvs_depthmap_pointset_device."""
    _fields_ = [("depth_dev", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("invproj", C.c_float * 9),
                ("cam_to_world", C.c_void_p), ("color_dev", C.c_void_p), ("color_channels", C.c_int32),
                ("vertex_ids", C.c_void_p), ("vertices", C.c_void_p), ("colors", C.c_void_p), ("faces", C.c_void_p),
                ("normals", C.c_void_p), ("confidences", C.c_void_p), ("scales", C.c_void_p),
                ("cap_vertices", C.c_uint64), ("cap_faces", C.c_uint64), ("n_vertices", C.c_uint64), ("n_faces", C.c_uint64)]


def _per_map(what, v, n):
    v = [None] * n if v is None else list(v)
    if len(v) != n:
        raise ValueError("%d %s for %d maps" % (len(v), what, n))
    return v


def depthmap_pointset_maps(dms, invprojs, colors=None, cam_to_world=None, dd_factor: float = DD_FACTOR_DEFAULT,
                           with_normals: bool = False, conf_iterations: int = 0, scale_factor: Optional[float] = None):
    """depthmap_pointset on each map of a batch of torch CUDA tensors, e.g. the depth maps of
    Scene.reconstruct(on_device=True): float32, contiguous, H x W, all on one device.  invprojs: one 3x3 (or 9) inverse
    projection per map.  colors: None, or one uint8 H x W or H x W x C CUDA tensor (or None) per map, e.g.
    Scene.level(v, s, on_device=True).  cam_to_world: None, or one 4x4 host matrix (or None) per map.
    Two library calls (b200mvs_depthmap_pointset_device) on the device's current stream: one counts, one fills new,
    exactly sized tensors.  Returns one dict per map with the keys of depthmap_pointset but device_ms, each value a CUDA
    tensor or None when skipped; vertex_ids and faces are torch.uint32 (torch.int32 with the same bits on a torch
    without uint32)."""
    import torch
    dms = list(dms)
    dev = _device_maps("dms", dms)
    n = len(dms)
    ips = np.ascontiguousarray(invprojs, np.float32)
    if ips.size != 9 * n:
        raise ValueError("invprojs must hold one 3x3 matrix per map (%d maps)" % n)
    ips = ips.reshape(n, 9)
    cols = _per_map("colour images", colors, n)
    ctws = [None if c is None else np.ascontiguousarray(c, np.float32).reshape(16) for c in _per_map("cam_to_world", cam_to_world, n)]
    meshes = (DmMesh * max(n, 1))()
    for j, (d, c) in enumerate(zip(dms, cols)):
        m = meshes[j]
        m.depth_dev, m.height, m.width = d.data_ptr(), d.shape[0], d.shape[1]
        m.invproj[:] = [float(x) for x in ips[j]]
        m.cam_to_world = None if ctws[j] is None else ctws[j].ctypes.data
        if c is not None:
            if not _is_cuda(c) or c.device != dev or c.dtype != torch.uint8 or c.dim() not in (2, 3) or not c.is_contiguous():
                raise ValueError("colors[%d] must be a contiguous uint8 CUDA tensor on %s" % (j, dev))
            if tuple(c.shape[:2]) != tuple(d.shape):
                raise ValueError("Color image dimension mismatch (map %d)" % j)
            m.color_dev, m.color_channels = c.data_ptr(), 1 if c.dim() == 2 else c.shape[2]
    index, _, _, _, stream = _batch(dms, dev)
    L = _lib()

    def call():
        _check(L.b200mvs_depthmap_pointset_device(index, n, meshes, float(dd_factor), int(conf_iterations),
                                                  float(scale_factor if scale_factor is not None else 0.0), stream))
    call()
    u32 = getattr(torch, "uint32", torch.int32)
    out = []
    for j, (d, c) in enumerate(zip(dms, cols)):
        m = meshes[j]
        nv, nf = int(m.n_vertices), int(m.n_faces)
        f32 = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)      # noqa: E731
        r = dict(vertex_ids=torch.empty(tuple(d.shape), dtype=u32, device=dev), vertices=f32(nv, 3),
                 colors=None if c is None else f32(nv, 4), faces=torch.empty((nf, 3), dtype=u32, device=dev),
                 normals=f32(nv, 3) if with_normals else None, confidences=f32(nv) if conf_iterations > 0 else None,
                 scales=f32(nv) if scale_factor is not None else None)
        for k, t in r.items():
            setattr(m, k, None if t is None else t.data_ptr())
        m.cap_vertices, m.cap_faces = nv, nf
        out.append(r)
    call()
    return out


def depthmap_triangulate_maps(dms, invprojs, colors=None, cam_to_world=None, dd_factor: float = DD_FACTOR_DEFAULT):
    """depthmap_triangulate on each map of a batch of torch CUDA tensors: depthmap_pointset_maps without the per-vertex
    attributes.  Returns one dict per map with vertex_ids, vertices, colors (or None) and faces."""
    keys = ("vertex_ids", "vertices", "colors", "faces")
    return [{k: r[k] for k in keys} for r in depthmap_pointset_maps(dms, invprojs, colors, cam_to_world, dd_factor)]


def depthmap_triangulate(dm: np.ndarray, invproj: np.ndarray, dd_factor: float = DD_FACTOR_DEFAULT,
                         cam_to_world: Optional[np.ndarray] = None, color: Optional[np.ndarray] = None, device: int = 0):
    """mve::geom::depthmap_triangulate (depthmap.cc:196-375). Returns dict(vertex_ids [H,W] uint32, vertices [V,3], colors [V,4]
    or None, faces [F,3] uint32, device_ms).  dm (and color) may be torch CUDA tensors (`device` is then theirs): the
    result is the dict of depthmap_triangulate_maps, CUDA tensors without device_ms."""
    if _is_cuda(dm):
        return depthmap_triangulate_maps([dm], [invproj], [color], [cam_to_world], dd_factor)[0]
    dm = np.ascontiguousarray(dm, np.float32)
    h, w = dm.shape
    ip = np.ascontiguousarray(invproj, np.float32).reshape(9)
    ctw = None if cam_to_world is None else np.ascontiguousarray(cam_to_world, np.float32).reshape(16)
    cch = 0
    if color is not None:
        color = np.ascontiguousarray(color, np.uint8)
        if color.shape[:2] != (h, w):
            raise ValueError("Color image dimension mismatch")
        cch = 1 if color.ndim == 2 else color.shape[2]
    cap_v, cap_f = w * h, 2 * (w - 1) * (h - 1)
    vids = np.empty((h, w), np.uint32)
    verts = np.empty((cap_v, 3), np.float32)
    cols = np.empty((cap_v, 4), np.float32) if color is not None else None
    faces = np.empty((cap_f, 3), np.uint32)
    nv, nf, ms = C.c_uint64(0), C.c_uint64(0), C.c_double(0)
    _check(_lib().b200mvs_depthmap_triangulate(device, _p(dm), w, h, _p(ip), float(dd_factor), _p(ctw), _p(color), cch, _p(vids), _p(verts),
                                               _p(cols), _p(faces), cap_v, cap_f, C.byref(nv), C.byref(nf), C.byref(ms)))
    return dict(vertex_ids=vids, vertices=verts[:nv.value].copy(), colors=None if cols is None else cols[:nv.value].copy(),
                faces=faces[:nf.value].copy(), device_ms=ms.value)


def depthmap_pointset(dm: np.ndarray, invproj: np.ndarray, dd_factor: float = DD_FACTOR_DEFAULT,
                      cam_to_world: Optional[np.ndarray] = None, color: Optional[np.ndarray] = None,
                      with_normals: bool = True, conf_iterations: int = 4, scale_factor: Optional[float] = 2.5, device: int = 0):
    """The per-view work of apps/scene2pset (scene2pset.cc:264-358): triangulation + vertex normals + boundary confidences +
    scale values. Returns the dict of depthmap_triangulate plus normals [V,3], confidences [V], scales [V] (None when skipped).
    dm (and color) may be torch CUDA tensors (`device` is then theirs): the result is the dict of depthmap_pointset_maps."""
    if _is_cuda(dm):
        return depthmap_pointset_maps([dm], [invproj], [color], [cam_to_world], dd_factor, with_normals, conf_iterations,
                                      scale_factor)[0]
    dm = np.ascontiguousarray(dm, np.float32)
    h, w = dm.shape
    ip = np.ascontiguousarray(invproj, np.float32).reshape(9)
    ctw = None if cam_to_world is None else np.ascontiguousarray(cam_to_world, np.float32).reshape(16)
    cch = 0
    if color is not None:
        color = np.ascontiguousarray(color, np.uint8)
        cch = 1 if color.ndim == 2 else color.shape[2]
    cap_v, cap_f = w * h, 2 * (w - 1) * (h - 1)
    vids = np.empty((h, w), np.uint32)
    verts = np.empty((cap_v, 3), np.float32)
    cols = np.empty((cap_v, 4), np.float32) if color is not None else None
    faces = np.empty((cap_f, 3), np.uint32)
    nrm = np.empty((cap_v, 3), np.float32) if with_normals else None
    cf = np.empty(cap_v, np.float32) if conf_iterations > 0 else None
    sc = np.empty(cap_v, np.float32) if scale_factor is not None else None
    nv, nf, ms = C.c_uint64(0), C.c_uint64(0), C.c_double(0)
    _check(_lib().b200mvs_depthmap_pointset(device, _p(dm), w, h, _p(ip), float(dd_factor), _p(ctw), _p(color), cch, _p(vids), _p(verts),
                                            _p(cols), _p(faces), _p(nrm), _p(cf), int(conf_iterations), _p(sc),
                                            float(scale_factor if scale_factor is not None else 0.0), cap_v, cap_f,
                                            C.byref(nv), C.byref(nf), C.byref(ms)))
    n = nv.value
    return dict(vertex_ids=vids, vertices=verts[:n].copy(), colors=None if cols is None else cols[:n].copy(), faces=faces[:nf.value].copy(),
                normals=None if nrm is None else nrm[:n].copy(), confidences=None if cf is None else cf[:n].copy(),
                scales=None if sc is None else sc[:n].copy(), device_ms=ms.value)


class _PsetOptions(C.Structure):
    _fields_ = [("with_normals", C.c_int32), ("with_conf", C.c_int32), ("with_scale", C.c_int32), ("poisson_normals", C.c_int32),
                ("correspondence", C.c_int32), ("use_aabb", C.c_int32), ("aabb_min", C.c_float * 3), ("aabb_max", C.c_float * 3),
                ("min_valid_fraction", C.c_float), ("scale_factor", C.c_float), ("dd_factor", C.c_float), ("conf_iterations", C.c_int32)]


class _PsetCamera(C.Structure):
    _fields_ = [("flen", C.c_float), ("paspect", C.c_float), ("ppoint", C.c_float * 2), ("rot", C.c_float * 9), ("trans", C.c_float * 3)]


class _PsetView(C.Structure):
    _fields_ = [("added", C.c_int32), ("fraction", C.c_float), ("n_points", C.c_uint64), ("first_index", C.c_uint64)]


class _PsetInfo(C.Structure):
    _fields_ = [("n_points", C.c_uint64), ("n_colors", C.c_uint64), ("n_views", C.c_uint64), ("device_bytes", C.c_uint64),
                ("peak_device_bytes", C.c_uint64), ("ms_pointset", C.c_double), ("ms_filter", C.c_double), ("ms_mask", C.c_double)]


class _PsetCorrView(C.Structure):
    _fields_ = [("view_id", C.c_uint32), ("width", C.c_uint32), ("height", C.c_uint32), ("first_index", C.c_uint64)]


def _pset_lib():
    L = _lib()
    if not getattr(L, "_pset_ready", False):
        L.b200mvs_pset_create.argtypes = [C.c_int, C.POINTER(_PsetOptions), C.POINTER(C.c_void_p)]
        L.b200mvs_pset_create_on_device.argtypes = [C.c_int, C.POINTER(_PsetOptions), C.POINTER(C.c_void_p)]
        L.b200mvs_pset_read_device.argtypes = [C.c_void_p] + [C.c_void_p] * 7
        L.b200mvs_pset_destroy.argtypes = [C.c_void_p]
        L.b200mvs_pset_destroy.restype = None
        L.b200mvs_pset_add_view.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(_PsetCamera),
                                            C.POINTER(_PsetView)]
        L.b200mvs_pset_add_view_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                   C.POINTER(_PsetCamera), C.c_void_p, C.POINTER(_PsetView)]
        L.b200mvs_pset_clip_masks.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64)]
        L.b200mvs_pset_clip_masks_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                     C.c_void_p, C.POINTER(C.c_uint64)]
        L.b200mvs_pset_get_info.argtypes = [C.c_void_p, C.POINTER(_PsetInfo)]
        L.b200mvs_pset_read.argtypes = [C.c_void_p] + [C.c_void_p] * 5
        L.b200mvs_pset_read_correspondence.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200mvs_pset_add_reconstruction.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                                      C.c_void_p, C.c_void_p, C.c_void_p]
        L.b200mvs_pset_add_reconstruction_levels.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L._pset_ready = True
    return L


def _camera(cam) -> _PsetCamera:
    c = _PsetCamera()
    c.flen, c.paspect = float(cam["flen"]), float(cam["paspect"])
    c.ppoint[:] = [float(x) for x in np.asarray(cam["ppoint"], np.float32).reshape(2)]
    c.rot[:] = [float(x) for x in np.asarray(cam["rot"], np.float32).reshape(9)]
    c.trans[:] = [float(x) for x in np.asarray(cam["trans"], np.float32).reshape(3)]
    return c


def _options(options):
    o = dict(with_normals=False, with_conf=False, with_scale=False, poisson_normals=False, correspondence=False, aabb=None,
             min_valid_fraction=0.0, scale_factor=2.5, dd_factor=DD_FACTOR_DEFAULT, conf_iterations=4)
    o.update(options or {})
    opt = _PsetOptions()
    opt.with_normals, opt.with_conf, opt.with_scale = int(o["with_normals"]), int(o["with_conf"]), int(o["with_scale"])
    opt.poisson_normals, opt.correspondence = int(o["poisson_normals"]), int(o["correspondence"])
    opt.use_aabb = int(o["aabb"] is not None)
    if o["aabb"] is not None:
        opt.aabb_min[:] = [float(np.float32(x)) for x in o["aabb"][0]]
        opt.aabb_max[:] = [float(np.float32(x)) for x in o["aabb"][1]]
    opt.min_valid_fraction, opt.scale_factor = float(o["min_valid_fraction"]), float(o["scale_factor"])
    opt.dd_factor, opt.conf_iterations = float(o["dd_factor"]), int(o["conf_iterations"])
    return o, opt


def _view_record(view_id, r):
    return dict(id=int(view_id), added=bool(r.added), fraction=float(r.fraction), n_points=int(r.n_points),
                first_index=int(r.first_index))


def _cuda_masks(masks, device):
    """Whether the masks of scene_pointset are CUDA tensors (on the handle's `device`, else ValueError) or all host
    arrays; a mix raises ValueError.  Checked before any library call."""
    if not masks:
        return False
    cuda = [_is_cuda(m["mask"]) for m in masks]
    if any(cuda) and not all(cuda):
        raise ValueError("masks must be all CUDA tensors or all host arrays, not a mix")
    if cuda[0]:
        import torch
        dev = torch.device("cuda", device) if device >= 0 else None
        for m in masks:
            if m["mask"].device != dev:
                raise ValueError("a CUDA mask must be on the point set's device %s, not %s" % (dev, m["mask"].device))
    return cuda[0]


def _clip_device_masks(L, h, masks, device):
    """b200mvs_pset_clip_masks_device with CUDA tensor masks, read in place after the work of the current stream."""
    import torch
    ts = []
    for m in masks:
        t = m["mask"]
        if t.dim() != 2:
            raise ValueError("masks must have one channel")
        t = t.to(torch.uint8)
        if (t.shape[1] > 1 and t.stride(1) != 1) or (t.shape[0] > 1 and t.stride(0) < t.shape[1]):
            t = t.contiguous()
        ts.append(t)
    ptrs = (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    ws = np.array([t.shape[1] for t in ts], np.int32)
    hs = np.array([t.shape[0] for t in ts], np.int32)
    pitches = np.array([t.stride(0) if t.shape[0] > 1 else t.shape[1] for t in ts], np.int64)
    cams = (_PsetCamera * len(ts))(*[_camera(m["camera"]) for m in masks])
    stream = torch.cuda.current_stream(torch.device("cuda", device)).cuda_stream
    nf = C.c_uint64(0)
    _check(L.b200mvs_pset_clip_masks_device(h, len(ts), ptrs, _p(ws), _p(hs), _p(pitches), cams, C.c_void_p(stream), C.byref(nf)))
    return int(nf.value)


def _finish(L, h, o, masks, per_view, device=None, mask_device=None):
    """Clips the handle's points with `masks` and reads the point set out (the result of scene_pointset): numpy arrays, or
    with `device` (a handle's device index) torch CUDA tensors on that device, read on its current stream.  mask_device:
    the handle's device when the masks are CUDA tensors (_cuda_masks)."""
    num_filtered = 0
    if masks and mask_device is not None:
        num_filtered = _clip_device_masks(L, h, masks, mask_device)
    elif masks:
        ms = [np.ascontiguousarray(m["mask"], np.uint8) for m in masks]
        if any(m.ndim != 2 for m in ms):
            raise ValueError("masks must have one channel")
        ptrs = (C.c_void_p * len(ms))(*[m.ctypes.data for m in ms])
        ws = np.array([m.shape[1] for m in ms], np.int32)
        hs = np.array([m.shape[0] for m in ms], np.int32)
        cams = (_PsetCamera * len(ms))(*[_camera(m["camera"]) for m in masks])
        nf = C.c_uint64(0)
        _check(L.b200mvs_pset_clip_masks(h, len(ms), ptrs, _p(ws), _p(hs), cams, C.byref(nf)))
        num_filtered = int(nf.value)
    info = _PsetInfo()
    _check(L.b200mvs_pset_get_info(h, C.byref(info)))
    n, nc = int(info.n_points), int(info.n_colors)
    if device is None:
        empty, f32, u32, ptr = np.empty, np.float32, np.uint32, _p
    else:
        import torch
        dev = torch.device("cuda", device)
        # uint32 where torch has the dtype (it copies and converts to numpy; few kernels take it), else the same bits as int32
        empty, f32, u32 = (lambda shape, dt: torch.empty(shape, dtype=dt, device=dev)), torch.float32, getattr(torch, "uint32", torch.int32)
        ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())             # noqa: E731
    verts = empty((n, 3), f32)
    nrm = empty((n, 3), f32) if o["with_normals"] else None
    cols = empty((nc, 4), f32)
    vals = empty(n, f32) if o["with_scale"] else None
    cfs = empty(n, f32) if o["with_conf"] else None
    pix = empty((n, 2), u32) if o["correspondence"] else None
    if device is None:
        _check(L.b200mvs_pset_read(h, _p(verts), _p(nrm), _p(cols), _p(vals), _p(cfs)))
    else:
        stream = torch.cuda.current_stream(dev).cuda_stream
        _check(L.b200mvs_pset_read_device(h, ptr(verts), ptr(nrm), ptr(cols), ptr(vals), ptr(cfs), ptr(pix), C.c_void_p(stream)))
    corr = None
    if o["correspondence"]:
        meta = (_PsetCorrView * max(1, int(info.n_views)))()
        _check(L.b200mvs_pset_read_correspondence(h, _p(pix) if device is None else None, meta))
        corr = dict(pixels=pix, views=[(int(m.view_id), int(m.width), int(m.height), int(m.first_index))
                                       for m in meta[:int(info.n_views)]])
    return dict(vertices=verts, normals=nrm, colors=cols, values=vals, confidences=cfs, views=per_view, correspondence=corr,
                num_filtered=num_filtered,
                info=dict(peak_device_bytes=int(info.peak_device_bytes), device_bytes=int(info.device_bytes),
                          ms_pointset=info.ms_pointset, ms_filter=info.ms_filter, ms_mask=info.ms_mask))


def _create(L, device, opt, on_device):
    h = C.c_void_p()
    create = L.b200mvs_pset_create_on_device if on_device else L.b200mvs_pset_create
    _check(create(device, C.byref(opt), C.byref(h)))
    return h


def scene_pointset(views, options=None, masks=None, device: int = 0, on_device: bool = False):
    """The whole-scene point set of apps/scene2pset (scene2pset.cc:247-464) on the device, through b200mvs_pset_*.

    views: dicts with id, depth [H, W] float32, camera (dict of flen, paspect, ppoint, rot, trans as in mve::CameraInfo) and
    optionally color [H, W] or [H, W, C] uint8 (None: the view adds no colours), in output order.  depth and color may be
    torch CUDA tensors on `device` (both, or depth alone without colours): such a view is read where it is
    (b200mvs_pset_add_view_device, after the work of the current stream) and gives the same points as its host copy.
    options: with_normals, with_conf, with_scale, poisson_normals, correspondence, aabb ((min xyz), (max xyz)) or None,
    min_valid_fraction (0), scale_factor (2.5), dd_factor (5), conf_iterations (4).
    masks: dicts with mask [H, W] uint8 (one channel) and camera; the points any of them marks 0 are deleted.  The masks
    may be torch CUDA tensors on `device`, all of them or none: they are read in place after the work of the current
    stream (b200mvs_pset_clip_masks_device), with either value of on_device and the same results.

    Returns dict(vertices [N, 3], normals [N, 3] or None, colors [M, 4] (M < N when a view had no colour image),
    values [N] or None, confidences [N] or None, views (per input view: id, added, fraction, n_points, first_index),
    correspondence (pixels [N, 2] uint32, views [(view_id, width, height, first_index)]) or None, num_filtered,
    info (peak_device_bytes, device_bytes, ms_pointset, ms_filter, ms_mask)).

    on_device: the set is built and clipped in device memory (b200mvs_pset_create_on_device) and vertices, normals,
    colors, values, confidences and correspondence pixels are torch CUDA tensors on `device`, read on its current stream
    (b200mvs_pset_read_device), with the shapes and dtypes above; the pixels are torch.uint32 (torch.int32 with the same
    bits on a torch without uint32).  views, correspondence views, num_filtered and info stay host values."""
    o, opt = _options(options)
    cuda_masks = _cuda_masks(masks, device)
    L = _pset_lib()
    h = _create(L, device, opt, on_device)
    try:
        per_view = []
        for v in views:
            if _is_cuda(v["depth"]):
                per_view.append(_add_device_view(L, h, v))
                continue
            dm = np.ascontiguousarray(v["depth"], np.float32)
            col = v.get("color")
            cch = 0
            if col is not None:
                col = np.ascontiguousarray(col, np.uint8)
                if col.shape[:2] != dm.shape:
                    raise ValueError("Color image dimension mismatch")
                cch = 1 if col.ndim == 2 else col.shape[2]
            r = _PsetView()
            cam = _camera(v["camera"])
            _check(L.b200mvs_pset_add_view(h, int(v["id"]), _p(dm), dm.shape[1], dm.shape[0], _p(col), cch, C.byref(cam), C.byref(r)))
            per_view.append(_view_record(v["id"], r))
        return _finish(L, h, o, masks, per_view, device if on_device else None, device if cuda_masks else None)
    finally:
        L.b200mvs_pset_destroy(h)


def _is_cuda(a):
    return getattr(a, "is_cuda", False) is True


def _add_device_view(L, h, v):
    """One view of scene_pointset whose depth map (and colour image) are CUDA tensors."""
    import torch
    dm = v["depth"].to(torch.float32).contiguous()
    if dm.dim() != 2:
        raise ValueError("depth must be H x W")
    col = v.get("color")
    cch = 0
    if col is not None:
        if not _is_cuda(col):
            raise ValueError("color must be a CUDA tensor when depth is one")
        col = col.to(torch.uint8).contiguous()
        if tuple(col.shape[:2]) != tuple(dm.shape):
            raise ValueError("Color image dimension mismatch")
        cch = 1 if col.dim() == 2 else col.shape[2]
    r = _PsetView()
    cam = _camera(v["camera"])
    stream = torch.cuda.current_stream(dm.device).cuda_stream
    _check(L.b200mvs_pset_add_view_device(h, int(v["id"]), C.c_void_p(dm.data_ptr()), dm.shape[1], dm.shape[0],
                                          None if col is None else C.c_void_p(col.data_ptr()), cch, C.byref(cam),
                                          C.c_void_p(stream), C.byref(r)))
    return _view_record(v["id"], r)


def reconstruct_pointset(scene, settings, ref_views, options=None, masks=None, progress=None, on_device: bool = False,
                         scales=None):
    """dmrecon and scene2pset in one call (b200mvs_pset_add_reconstruction): reconstructs the reference views of
    `scene` (a dmrecon.Scene) and builds their point set on the device, each view's depth map and colours (its pyramid
    level settings.scale) staying on the device.  Equal to scene.reconstruct(...) followed by scene_pointset of the maps
    with the level images and the registered cameras, in ref_views order.  options, masks and on_device as for
    scene_pointset (on_device: the set never leaves the scene's device); progress as for Scene.reconstruct.
    scales: one pyramid level per reference view instead of settings.scale (b200mvs_pset_add_reconstruction_levels);
    a view may appear at several levels, and each entry adds the points of its map and its level image.  Returns
    (the dict of scene_pointset, dmrecon.Stats)."""
    o, opt = _options(options)
    cuda_masks = _cuda_masks(masks, scene.device)
    L = _pset_lib()
    refs = np.asarray(ref_views, np.int32)
    levels = dmrecon.levels_array(scales, len(refs))
    h = C.c_void_p()
    # a planning context has no device to make a handle on: the call itself rejects the context
    if scene.device != dmrecon.DEVICE_NONE:
        h = _create(L, scene.device, opt, on_device)
    try:
        recs = (_PsetView * max(1, len(refs)))()
        stats = dmrecon.Stats()
        failed = C.c_int32(-1)
        if levels is None:
            rc = L.b200mvs_pset_add_reconstruction(h, scene._h, C.byref(settings), len(refs), _p(refs), progress,
                                                   C.byref(stats), C.byref(failed), recs)
        else:
            rc = L.b200mvs_pset_add_reconstruction_levels(h, scene._h, C.byref(settings), len(refs), _p(refs), _p(levels),
                                                          progress, C.byref(stats), C.byref(failed), recs)
        if rc != 0:
            msg = L.b200mvs_last_error(None).decode()
            if failed.value >= 0:
                msg += " (view %d)" % failed.value
            raise dmrecon.B200MVSError(rc, msg, failed.value)
        per_view = [_view_record(v, recs[j]) for j, v in enumerate(refs.tolist())]
        return _finish(L, h, o, masks, per_view, scene.device if on_device else None,
                       scene.device if cuda_masks else None), stats
    finally:
        if h.value:
            L.b200mvs_pset_destroy(h)
