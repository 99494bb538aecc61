"""Host-side mirror of the reference's dmrecon interface over the C ABI of libb200mvs.so.

The reference's boundary for this path is the C++ class `mvs::DMRecon(scene, settings).start()`
(libs/dmrecon/dmrecon.h:40-68) fed by `mve::Scene`/`mve::View`; the compiled drop-in for that is
shim/ (see INTEGRATION.md).  This module is the same surface for Python callers (tests, bench.py):

    Settings  <-> mvs::Settings           (libs/dmrecon/settings.h:22-52, same names and defaults)
    Scene     <-> mve::Scene              (views with `undistorted` images + cameras, bundle features)
    DMRecon   <-> mvs::DMRecon            (ctor validation messages of dmrecon.cc:30-87; start())

There is no CPU fallback: importing works without a GPU, creating a Scene does not.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Sequence

import numpy as np

from . import build as _build

_LIB = None


class B200MVSError(RuntimeError):
    def __init__(self, code: int, msg: str, failed_view: int = -1):
        super().__init__("b200mvs error %d: %s" % (code, msg))
        self.code = code
        self.failed_view = failed_view


class Settings(C.Structure):
    """mvs::Settings (settings.h:22-52). Field names follow the C ABI (snake case of the reference's)."""
    _fields_ = [("filter_width", C.c_uint32), ("min_ncc", C.c_float), ("min_parallax", C.c_float),
                ("accept_ncc", C.c_float), ("min_refine_diff", C.c_float), ("max_iterations", C.c_uint32),
                ("nr_recon_neighbors", C.c_uint32), ("global_vs_max", C.c_uint32), ("scale", C.c_int32),
                ("use_color_scale", C.c_int32), ("aabb_min", C.c_float * 3), ("aabb_max", C.c_float * 3),
                ("frontier_band", C.c_float), ("frontier_topk", C.c_uint32)]

    def __init__(self, **kw):
        super().__init__()
        lib().b200mvs_default_settings(C.byref(self))
        for k, v in kw.items():
            if not hasattr(self, k):
                raise AttributeError(k)
            setattr(self, k, v)


class _Maps(C.Structure):
    _fields_ = [("depth", C.c_void_p), ("conf", C.c_void_p), ("dz", C.c_void_p), ("normal", C.c_void_p),
                ("view_ids", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32)]


# The maps of a reference view of H x W pixels: name -> (trailing shape after (H, W), numpy dtype, torch dtype name)
_MAP_LAYOUT = dict(depth=((), np.float32, "float32"), conf=((), np.float32, "float32"), dz=((2,), np.float32, "float32"),
                   normal=((3,), np.float32, "float32"), view_ids=((4,), np.int32, "int32"))


class Progress(C.Structure):
    """mvs::Progress (progress.h:27-43)."""
    _fields_ = [("status", C.c_int32), ("cancelled", C.c_int32), ("filled", C.c_uint64),
                ("queue_size", C.c_uint64), ("start_time", C.c_uint64)]


class Stats(C.Structure):
    _fields_ = [("n_opt", C.c_uint64), ("n_sample_sets", C.c_uint64), ("n_rounds", C.c_uint64),
                ("n_filled", C.c_uint64), ("n_seeds_processed", C.c_uint64), ("n_seeds_success", C.c_uint64),
                ("n_entries_peak", C.c_uint64), ("ms_patch_kernel", C.c_double), ("ms_total_device", C.c_double),
                ("n_patch_launches", C.c_uint64), ("n_kernel_launches", C.c_uint64),
                ("ms_optimise_phases", C.c_double), ("n_grid_barriers", C.c_uint64),
                ("ms_optimise_thread_phases", C.c_double), ("ms_sort_phases", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


PATCH_IN = np.dtype([("x", "<i4"), ("y", "<i4"), ("depth", "<f4"), ("dz_i", "<f4"), ("dz_j", "<f4"),
                     ("n_local", "<i4"), ("local_ids", "<i4", (4,))])
PATCH_OUT = np.dtype([("conf", "<f4"), ("depth", "<f4"), ("dz_i", "<f4"), ("dz_j", "<f4"),
                      ("normal", "<f4", (3,)), ("n_local", "<i4"), ("local_ids", "<i4", (4,)),
                      ("iterations", "<i4"), ("converged", "<i4"), ("opti_success", "<i4")])

EXPORTS = ["b200mvs_default_settings", "b200mvs_create", "b200mvs_destroy", "b200mvs_last_error", "b200mvs_version",
           "b200mvs_upload_view", "b200mvs_upload_view_device", "b200mvs_set_view_camera", "b200mvs_set_features", "b200mvs_num_levels",
           "b200mvs_get_level", "b200mvs_global_view_selection", "b200mvs_optimize_patches", "b200mvs_reconstruct",
           "b200mvs_plan_views", "b200mvs_set_patch_mode", "b200mvs_depthmap_last_error", "b200mvs_depthmap_confidence_clean",
           "b200mvs_depthmap_cleanup", "b200mvs_depthmap_triangulate", "b200mvs_depthmap_pointset",
           "b200mvs_depthmap_confidence_clean_device", "b200mvs_depthmap_cleanup_device", "b200mvs_depthmap_pointset_device",
           "b200mvs_set_image_source", "b200mvs_memory_stats", "b200mvs_working_set", "b200mvs_plan_batches",
           "b200mvs_set_frontier_capacity", "b200mvs_frontier_info", "b200mvs_plan_stats", "b200mvs_pset_create", "b200mvs_pset_destroy",
           "b200mvs_pset_add_view", "b200mvs_pset_clip_masks", "b200mvs_pset_get_info", "b200mvs_pset_read",
           "b200mvs_pset_read_correspondence", "b200mvs_pset_add_reconstruction", "b200mvs_reconstruct_device",
           "b200mvs_get_level_device", "b200mvs_pset_add_view_device", "b200mvs_pset_create_on_device", "b200mvs_pset_read_device",
           "b200mvs_set_view_distortion", "b200mvs_set_image_source_device", "b200mvs_set_view_mask",
           "b200mvs_set_view_mask_device", "b200mvs_pset_clip_masks_device", "b200mvs_reconstruct_levels",
           "b200mvs_reconstruct_levels_device", "b200mvs_pset_add_reconstruction_levels", "b200mvs_working_set_levels",
           "b200mvs_plan_batches_levels", "b200mvs_set_view_prior", "b200mvs_set_view_prior_device",
           "b200mvs_set_view_prior_state", "b200mvs_set_view_prior_state_device", "b200mvs_set_view_prior_relative",
           "b200mvs_set_view_prior_relative_device"]

ERR_INVALID_ARG = -1
ERR_CUDA = -2
ERR_GLOBAL_VS = -3
ERR_CANCELLED = -4
ERR_OVERFLOW = -5
ERR_NO_MEMORY = -7
DEVICE_NONE = -1             # B200MVS_DEVICE_NONE: a planning context (cameras, features, view selection; no images)


PRIOR_KINDS = {"disparity": 0, "depth": 1, "depth_scale": 2}    # B200MVS_PRIOR_* (include/b200mvs.h)


class PriorFit(C.Structure):
    """b200mvs_prior_fit (include/b200mvs.h)."""
    _fields_ = [("scale", C.c_double), ("shift", C.c_double), ("n_obs", C.c_uint32), ("n_inliers", C.c_uint32),
                ("median_rel_err", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class _Image(C.Structure):
    _fields_ = [("rgb", C.c_void_p), ("w", C.c_int32), ("h", C.c_int32), ("channels", C.c_int32)]


class _DeviceImage(C.Structure):
    """b200mvs_device_image (include/b200mvs.h)."""
    _fields_ = [("data", C.c_void_p), ("w", C.c_int32), ("h", C.c_int32), ("channels", C.c_int32),
                ("row_pitch", C.c_int64), ("plane_pitch", C.c_int64), ("cuda_stream", C.c_void_p)]


_FETCH_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int32, C.POINTER(_Image))
_DEVICE_FETCH_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_int32, C.POINTER(_DeviceImage))
_RELEASE_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_int32)


def device_image_layout(shape: Sequence[int], strides: Sequence[int], layout: str = "hwc"):
    """The b200mvs_device_image fields (h, w, channels, row_pitch, plane_pitch) of a uint8 image of this shape and these
    strides (in elements = bytes): layout "hwc" takes H x W x C or H x W (grey), "chw" takes C x H x W.  The element
    stride must be 1, the pixel stride C (hwc) or 1 (chw), the row stride at least the bytes of a row and the plane stride
    at least h * row stride (planes that do not overlap the rows of another).  The stride of a dimension of size 1 is never
    used and is not checked.  Anything else raises ValueError."""
    shape, strides = tuple(int(v) for v in shape), tuple(int(v) for v in strides)
    if layout == "hwc":
        if len(shape) == 2:
            shape, strides = shape + (1,), strides + (1,)
        if len(shape) != 3:
            raise ValueError("an hwc image is H x W x C or H x W, not %s" % (shape,))
        h, w, c = shape
        row, px, el = strides
        plane = 0
    elif layout == "chw":
        if len(shape) != 3:
            raise ValueError("a chw image is C x H x W, not %s" % (shape,))
        c, h, w = shape
        plane, row, px = strides
        el = 1
    else:
        raise ValueError("layout must be 'hwc' or 'chw', not %r" % (layout,))
    if not 1 <= c <= 4:
        raise ValueError("an image has 1 to 4 channels, not %d" % c)
    if h < 1 or w < 1:
        raise ValueError("empty image %s" % (shape,))
    if c == 1 and layout == "hwc":
        el = 1
    if layout == "hwc":
        if el != 1 or (w > 1 and px != c):
            raise ValueError("an hwc image needs channel stride 1 and pixel stride C, not strides %s" % (strides,))
        row = row if h > 1 else w * c
        if row < w * c:
            raise ValueError("hwc row stride %d is less than W * C = %d" % (row, w * c))
        return h, w, c, row, 0
    if w > 1 and px != 1:
        raise ValueError("a chw image needs pixel stride 1, not strides %s" % (strides,))
    row = row if h > 1 else w
    if row < w:
        raise ValueError("chw row stride %d is less than W = %d" % (row, w))
    plane = plane if c > 1 else h * row
    if plane < h * row:
        raise ValueError("chw plane stride %d overlaps the rows of a plane: it must be at least H * row stride = %d"
                         % (plane, h * row))
    return h, w, c, row, plane


class Memory(C.Structure):
    """b200mvs_memory: device budget and accounting of one context (include/b200mvs.h)."""
    _fields_ = [("budget", C.c_uint64), ("fixed", C.c_uint64), ("resident", C.c_uint64), ("peak", C.c_uint64),
                ("n_loads", C.c_uint64), ("bytes_loaded", C.c_uint64), ("n_evictions", C.c_uint64), ("n_groups", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class PlanInfo(C.Structure):
    """b200mvs_plan_info: how the last reconstruction planned its views (include/b200mvs.h)."""
    _fields_ = [("n_prepared", C.c_uint64), ("n_device", C.c_uint64), ("n_host", C.c_uint64), ("ms_plan", C.c_double),
                ("ms_device", C.c_double), ("peak_bytes", C.c_uint64)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def lib():
    """Loads libb200mvs.so (building it when sources are newer). Fails loudly when it cannot."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.environ.get("B200MVS_LIB") or _build.LIB      # B200MVS_LIB: kernel-variant experiments (tools/kbench.py)
    if path == _build.LIB and _build.needs_build():
        path = _build.build()
    L = C.CDLL(path)
    L.b200mvs_last_error.restype = C.c_char_p
    L.b200mvs_last_error.argtypes = [C.c_void_p]
    L.b200mvs_version.restype = C.c_char_p
    L.b200mvs_default_settings.argtypes = [C.c_void_p]
    L.b200mvs_create.argtypes = [C.c_int, C.c_int, C.c_void_p]
    L.b200mvs_destroy.argtypes = [C.c_void_p]
    L.b200mvs_upload_view.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float,
                                      C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_upload_view_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_set_features.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_set_view_distortion.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float]
    L.b200mvs_set_view_mask.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.b200mvs_set_view_mask_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_void_p]
    L.b200mvs_set_view_prior.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.b200mvs_set_view_prior_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int64, C.c_int,
                                                C.c_void_p]
    L.b200mvs_set_view_prior_state.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                               C.c_int]
    L.b200mvs_set_view_prior_state_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                      C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_void_p]
    L.b200mvs_set_view_prior_relative.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                                  C.POINTER(PriorFit)]
    L.b200mvs_set_view_prior_relative_device.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int64,
                                                         C.c_int, C.c_int, C.c_void_p, C.POINTER(PriorFit)]
    L.b200mvs_set_view_camera.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_num_levels.argtypes = [C.c_void_p, C.c_int]
    L.b200mvs_get_level.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_get_level_device.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_global_view_selection.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    L.b200mvs_optimize_patches.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                           C.c_void_p, C.c_void_p]
    L.b200mvs_reconstruct.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    L.b200mvs_reconstruct_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
    L.b200mvs_reconstruct_levels.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]
    L.b200mvs_reconstruct_levels_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_working_set_levels.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_plan_batches_levels.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p,
                                              C.c_void_p]
    L.b200mvs_plan_views.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    L.b200mvs_set_patch_mode.argtypes = [C.c_void_p, C.c_int, C.c_int64]
    L.b200mvs_set_image_source.argtypes = [C.c_void_p, _FETCH_FN, _RELEASE_FN, C.c_void_p, C.c_uint64]
    L.b200mvs_set_image_source_device.argtypes = [C.c_void_p, _DEVICE_FETCH_FN, _RELEASE_FN, C.c_void_p, C.c_uint64]
    L.b200mvs_memory_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.b200mvs_working_set.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.b200mvs_plan_batches.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    L.b200mvs_set_frontier_capacity.argtypes = [C.c_void_p, C.c_double, C.c_uint64]
    L.b200mvs_frontier_info.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.b200mvs_plan_stats.argtypes = [C.c_void_p, C.c_void_p]
    _LIB = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def levels_array(scales, n: int):
    """The int32 level array of the *_levels entry points for `scales` (one pyramid level per reference view), or None
    for scales=None (the entry points without levels, at settings.scale).  A length other than n raises ValueError."""
    if scales is None:
        return None
    levels = np.ascontiguousarray(scales, np.int32).reshape(-1)
    if len(levels) != n:
        raise ValueError("scales has %d entries for %d reference views" % (len(levels), n))
    return levels


def _torch():
    """torch, imported only by the calls that return CUDA tensors."""
    import torch
    return torch


class Scene:
    """Device-resident counterpart of mve::Scene for this path: views (image + camera) and bundle features."""

    def __init__(self, n_views: int, device: int = 0):
        self._lib = lib()
        self.n_views = n_views
        self.device = device
        h = C.c_void_p()
        rc = self._lib.b200mvs_create(device, n_views, C.byref(h))
        if rc != 0:
            raise B200MVSError(rc, self._lib.b200mvs_last_error(None).decode())
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b200mvs_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc < 0:
            self._raise_fetch_error()
            raise B200MVSError(rc, self._lib.b200mvs_last_error(self._h).decode())
        return rc

    def _raise_fetch_error(self):
        """A device source's fetch returned a tensor that does not fit b200mvs_device_image: the failed call raises that
        ValueError (the fetch itself could only return failure to the library)."""
        errors = getattr(self, "_fetch_errors", None)
        if errors:
            err = errors[-1]
            errors.clear()
            raise err

    @classmethod
    def from_synth(cls, s, device: int = 0, views: Optional[Sequence[int]] = None, lazy: bool = False,
                   budget_bytes: int = 0) -> "Scene":
        """Uploads a mve_b200.synth.Scene (host images -> device, pyramids built on the device).
        lazy: register cameras only and install an image source over the scene's images (loaded when a call needs them,
        evicted to stay within budget_bytes; 0 = 90 % of the free device memory)."""
        sc = cls(s.n_views, device)
        for v in (range(s.n_views) if views is None else views):
            if lazy:
                sc.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
            else:
                sc.set_view(v, s.images[v], s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
        sc.set_features(s.feat_pos, s.feat_refs)
        if lazy:
            sc.set_image_source(lambda v: s.images[v], budget_bytes)
        return sc

    def set_image_source(self, fetch, budget_bytes: int = 0, on_device: bool = False, layout: str = "hwc"):
        """Loads images on demand: fetch(view_id) returns the view's H x W x C uint8 image (the size registered for the view).
        budget_bytes bounds the device memory of this context (0 = 90 % of the free bytes now); pyramids no running call
        needs are evicted and fetched again when needed.  fetch=None removes the source.
        on_device: fetch returns a torch.uint8 CUDA tensor on cuda:<device> instead (b200mvs_set_image_source_device):
        H x W x C or H x W with layout "hwc", C x H x W with layout "chw", with any strides device_image_layout accepts.
        The pyramid is built from the tensor in place, after the work enqueued on the current stream when fetch returns;
        the tensor is held until the library releases it.  A tensor that does not fit makes the call that fetched it
        raise ValueError."""
        if on_device and fetch is not None:
            self._set_device_source(fetch, budget_bytes, layout)
            return
        held = {}

        def _fetch(_user, view_id, out):
            try:
                img = np.ascontiguousarray(fetch(int(view_id)), dtype=np.uint8)
                if img.ndim == 2:
                    img = img[:, :, None]
                held[int(view_id)] = img
                out.contents.rgb = img.ctypes.data
                out.contents.h, out.contents.w, out.contents.channels = img.shape
                return 0
            except Exception:
                return 1

        def _release(_user, view_id):
            held.pop(int(view_id), None)

        if fetch is None:
            self._source = None
            self._check(self._lib.b200mvs_set_image_source(self._h, _FETCH_FN(), _RELEASE_FN(), None, 0))
            return
        cbs = (_FETCH_FN(_fetch), _RELEASE_FN(_release), held)
        self._check(self._lib.b200mvs_set_image_source(self._h, cbs[0], cbs[1], None, int(budget_bytes)))
        self._source = cbs                       # the C side keeps the function pointers: keep the ctypes objects alive

    def _set_device_source(self, fetch, budget_bytes: int, layout: str):
        if layout not in ("hwc", "chw"):
            raise ValueError("layout must be 'hwc' or 'chw', not %r" % (layout,))
        torch = _torch()
        dev = torch.device(self._torch_device())
        held = {}
        errors = []

        def _fetch(_user, view_id, out):
            try:
                t = fetch(int(view_id))
                if not isinstance(t, torch.Tensor) or t.dtype != torch.uint8 or t.device != dev:
                    raise ValueError("fetch(%d) must return a torch.uint8 tensor on %s" % (view_id, dev))
                h, w, c, row, plane = device_image_layout(t.shape, t.stride(), layout)
                held[int(view_id)] = t
                o = out.contents
                o.data, o.w, o.h, o.channels, o.row_pitch, o.plane_pitch = t.data_ptr(), w, h, c, row, plane
                o.cuda_stream = torch.cuda.current_stream(dev).cuda_stream
                return 0
            except ValueError as e:
                errors.append(e)
                return 1
            except Exception:
                return 1

        def _release(_user, view_id):
            held.pop(int(view_id), None)

        cbs = (_DEVICE_FETCH_FN(_fetch), _RELEASE_FN(_release), held)
        self._check(self._lib.b200mvs_set_image_source_device(self._h, cbs[0], cbs[1], None, int(budget_bytes)))
        self._source = cbs                       # the C side keeps the function pointers: keep the ctypes objects alive
        self._fetch_errors = errors

    def memory_stats(self) -> Memory:
        m = Memory()
        self._check(self._lib.b200mvs_memory_stats(self._h, C.byref(m)))
        return m

    def working_set(self, settings: Settings, ref_views: Sequence[int], scales=None) -> int:
        """Device bytes one launch of these reference views needs beyond the fixed allocations.  scales: one pyramid
        level per reference view instead of settings.scale (b200mvs_working_set_levels)."""
        refs = np.asarray(ref_views, np.int32)
        levels = levels_array(scales, len(refs))
        out = C.c_uint64()
        if levels is None:
            self._check(self._lib.b200mvs_working_set(self._h, C.byref(settings), len(refs), _p(refs), C.byref(out)))
        else:
            self._check(self._lib.b200mvs_working_set_levels(self._h, C.byref(settings), len(refs), _p(refs), _p(levels),
                                                             C.byref(out)))
        return out.value

    def plan_batches(self, settings: Settings, ref_views: Sequence[int], available: int, scales=None):
        """Groups of these reference views whose working sets fit `available` bytes: (n_groups, group of each view).
        scales: one pyramid level per reference view instead of settings.scale (b200mvs_plan_batches_levels)."""
        refs = np.asarray(ref_views, np.int32)
        levels = levels_array(scales, len(refs))
        groups = np.full(len(refs), -1, np.int32)
        failed = C.c_int32(-1)
        if levels is None:
            rc = self._lib.b200mvs_plan_batches(self._h, C.byref(settings), len(refs), _p(refs), int(available), _p(groups),
                                                C.byref(failed))
        else:
            rc = self._lib.b200mvs_plan_batches_levels(self._h, C.byref(settings), len(refs), _p(refs), _p(levels),
                                                       int(available), _p(groups), C.byref(failed))
        if rc < 0:
            raise B200MVSError(rc, self._lib.b200mvs_last_error(self._h).decode(), failed.value)
        return rc, groups

    def set_view(self, view_id: int, image: np.ndarray, flen, paspect, ppoint, rot, trans):
        """mve::View with an `undistorted` uint8 image + mve::CameraInfo (camera.h:23-170)."""
        img = np.ascontiguousarray(image, dtype=np.uint8)
        if img.ndim == 2:
            img = img[:, :, None]
        h, w, ch = img.shape
        pp = np.ascontiguousarray(ppoint, np.float32)
        r = np.ascontiguousarray(rot, np.float32).reshape(9)
        t = np.ascontiguousarray(trans, np.float32).reshape(3)
        self._check(self._lib.b200mvs_upload_view(self._h, view_id, _p(img), w, h, ch, float(flen), float(paspect),
                                                  _p(pp), _p(r), _p(t)))

    def set_view_device(self, view_id: int, dev_ptr: int, w: int, h: int, flen, paspect, ppoint, rot, trans, stream: int = 0):
        """Same, the image (h x w x 3 uint8) already being in this device's memory (e.g. a torch tensor's data_ptr())."""
        pp = np.ascontiguousarray(ppoint, np.float32)
        r = np.ascontiguousarray(rot, np.float32).reshape(9)
        t = np.ascontiguousarray(trans, np.float32).reshape(3)
        self._check(self._lib.b200mvs_upload_view_device(self._h, view_id, C.c_void_p(dev_ptr), w, h, float(flen),
                                                         float(paspect), _p(pp), _p(r), _p(t), C.c_void_p(stream)))

    def set_view_camera(self, view_id: int, w: int, h: int, flen, paspect, ppoint, rot, trans):
        """SingleView::create: camera + image size, the colour image is loaded later (or never, if not needed)."""
        pp = np.ascontiguousarray(ppoint, np.float32)
        r = np.ascontiguousarray(rot, np.float32).reshape(9)
        t = np.ascontiguousarray(trans, np.float32).reshape(3)
        self._check(self._lib.b200mvs_set_view_camera(self._h, view_id, w, h, float(flen), float(paspect), _p(pp), _p(r), _p(t)))

    def set_view_distortion(self, view_id: int, k2: float, k4: float):
        """Radial distortion (mve::CameraInfo::dist, meta.ini camera.radial_distortion) of the images this view is given
        from now on: set_view, set_view_device and image-source fetches take the distorted photo, and level(view, 0) is
        sfmrecon's undistortion of it (mve::image::image_undistort_k2k4 with the view's flen).  (0, 0), the default,
        imports images unchanged.  A changed value drops the view's resident pyramid; cameras are unchanged."""
        self._check(self._lib.b200mvs_set_view_distortion(self._h, view_id, float(k2), float(k4)))

    def set_view_mask(self, view_id: int, mask, on_device: bool = False):
        """Reconstruction mask of a reference view (b200mvs_set_view_mask): an H x W uint8 array, 0 = background, the
        convention of scene2pset -m; a numpy array or a torch tensor (a CUDA tensor is copied to the host).  None clears it.
        reconstruct(), reconstruct(on_device=True) and reconstruct_pointset() then never seed, queue or optimise a
        background pixel: it ends unfilled (depth, conf, dz, normal 0, view ids -1) and yields no point.  Pixel (x, y) of a
        W x H map is background when mask pixel ((2x+1) * mask_w // 2W, (2y+1) * mask_h // 2H) is 0, so the mask may have
        the photo's size or any level's.  This differs from the `masks=` of reconstruct_pointset(), which deletes points of
        the finished point set (scene2pset -m) after every pixel has been reconstructed.
        on_device: the mask is an H x W torch.uint8 CUDA tensor on the scene's device, copied on the device after the
        work of its current stream (b200mvs_set_view_mask_device), with the same results.  Its rows may be pitched (a
        tensor whose rows are not dense is made contiguous first); the copy is kept in device memory, counted in
        memory_stats().fixed, until the mask is cleared or replaced.  Anything else raises ValueError."""
        if mask is None:
            self._check(self._lib.b200mvs_set_view_mask(self._h, view_id, None, 0, 0))
            return
        if on_device:
            self._set_view_mask_device(view_id, mask)
            return
        if hasattr(mask, "detach"):                  # a torch tensor, on the host or a device
            mask = mask.detach().cpu().numpy()
        m = np.asarray(mask)
        if m.ndim != 2 or m.dtype != np.uint8:
            raise ValueError("a view mask is an H x W uint8 array, not %s %s" % (m.dtype, m.shape))
        m = np.ascontiguousarray(m)
        self._check(self._lib.b200mvs_set_view_mask(self._h, view_id, _p(m), m.shape[1], m.shape[0]))

    def _set_view_mask_device(self, view_id: int, mask):
        torch = _torch()
        if (not isinstance(mask, torch.Tensor) or mask.dtype != torch.uint8 or mask.dim() != 2 or not mask.is_cuda
                or (self.device != DEVICE_NONE and mask.device != torch.device(self._torch_device()))):
            where = "the scene's device" if self.device == DEVICE_NONE else self._torch_device()
            raise ValueError("an on-device view mask is an H x W torch.uint8 tensor on %s, not %s" % (
                where, "%s %s on %s" % (mask.dtype, tuple(mask.shape), mask.device) if isinstance(mask, torch.Tensor)
                else type(mask).__name__))
        h, w = mask.shape
        if h < 1 or w < 1:
            raise ValueError("an on-device view mask must not be empty, not %d x %d" % (h, w))
        if (w > 1 and mask.stride(1) != 1) or (h > 1 and mask.stride(0) < w):
            mask = mask.contiguous()
        pitch = mask.stride(0) if h > 1 else w
        stream = torch.cuda.current_stream(mask.device).cuda_stream
        self._check(self._lib.b200mvs_set_view_mask_device(self._h, view_id, C.c_void_p(mask.data_ptr()), w, h, pitch,
                                                           C.c_void_p(stream)))

    def set_view_prior(self, view_id: int, depth, stride: int, on_device: bool = False, dz=None, view_ids=None):
        """Prior depth map of a reference view (b200mvs_set_view_prior): an H x W float32 array of depths in MVE's
        convention (distance from the camera centre along the pixel's ray, as in depth-L<s>), a numpy array or a torch
        tensor (a CUDA tensor is copied to the host).  None clears it.  Every reconstruction then also seeds, after the
        SfM features, the pixels x = 2 + stride i <= W - 3, y = 2 + stride k <= H - 3 of each W x H map whose prior pixel
        ((2x+1) * prior_w // 2W, (2y+1) * prior_h // 2H) holds a finite depth > 0 and that are not masked out, so the
        prior may have the photo's size or any level's.  The copy is kept in device memory, counted in
        memory_stats().fixed, until the prior is cleared or replaced.
        on_device: the prior is an H x W torch.float32 CUDA tensor on the scene's device, at any row stride, copied on the
        device after the work of its current stream (b200mvs_set_view_prior_device), with the same results.  Anything
        else raises ValueError.
        dz (H x W x 2 float32) and view_ids (H x W x 4 int32), optional and of depth's H x W: the rest of each seed's
        state (b200mvs_set_view_prior_state[_device]).  A seed's dz is the prior's, scaled to the map's pixel size, and
        its local views are the prior's ids in the entry's global selection when there are exactly nr_recon_neighbors of
        them, so the maps of an earlier reconstruct go straight in:
        set_view_prior(v, m["depth"], 4, dz=m["dz"], view_ids=m["view_ids"]).  With on_device, every plane given is a
        CUDA tensor on the scene's device."""
        if depth is None:
            if dz is not None or view_ids is not None:
                raise ValueError("dz and view_ids of a view prior need its depth")
            self._check(self._lib.b200mvs_set_view_prior(self._h, view_id, None, 0, 0, 0))
            return
        if on_device:
            self._set_view_prior_device(view_id, depth, stride, dz, view_ids)
            return
        planes = []
        for name, t, tail, dt in (("depth", depth, (), np.float32), ("dz", dz, (2,), np.float32),
                                  ("view_ids", view_ids, (4,), np.int32)):
            if t is None:
                planes.append(None)
                continue
            if hasattr(t, "detach"):                 # a torch tensor, on the host or a device
                t = t.detach().cpu().numpy()
            a = np.asarray(t)
            shape = a.shape[:2] if not planes else planes[0].shape
            if a.ndim != 2 + len(tail) or a.shape[2:] != tail or a.shape[:2] != shape or a.dtype != dt:
                raise ValueError("a view prior's %s is an H x W%s %s array%s, not %s %s" % (
                    name, "".join(" x %d" % n for n in tail), np.dtype(dt).name,
                    " of the depth's H x W %s" % (shape,) if planes else "", a.dtype, a.shape))
            planes.append(np.ascontiguousarray(a))
        d, z, ids = planes
        h, w = d.shape
        if z is None and ids is None:
            self._check(self._lib.b200mvs_set_view_prior(self._h, view_id, _p(d), w, h, int(stride)))
        else:
            self._check(self._lib.b200mvs_set_view_prior_state(self._h, view_id, _p(d), None if z is None else _p(z),
                                                               None if ids is None else _p(ids), w, h, int(stride)))

    def _set_view_prior_device(self, view_id: int, depth, stride: int, dz=None, view_ids=None):
        torch = _torch()
        planes, pitches = [], []
        for name, t, tail, dt in (("depth", depth, (), torch.float32), ("dz", dz, (2,), torch.float32),
                                  ("view_ids", view_ids, (4,), torch.int32)):
            if t is None:
                planes.append(None)
                pitches.append(0)
                continue
            shape = (tuple(t.shape[:2]) if isinstance(t, torch.Tensor) else None) if not planes else tuple(planes[0].shape)
            if (not isinstance(t, torch.Tensor) or t.dtype != dt or t.dim() != 2 + len(tail) or not t.is_cuda
                    or tuple(t.shape[2:]) != tail or tuple(t.shape[:2]) != shape
                    or (self.device != DEVICE_NONE and t.device != torch.device(self._torch_device()))):
                where = "the scene's device" if self.device == DEVICE_NONE else self._torch_device()
                raise ValueError("an on-device view prior's %s is an H x W%s %s tensor%s on %s, not %s" % (
                    name, "".join(" x %d" % n for n in tail), dt, " of the depth's H x W" if planes else "", where,
                    "%s %s on %s" % (t.dtype, tuple(t.shape), t.device) if isinstance(t, torch.Tensor)
                    else type(t).__name__))
            h, w = t.shape[:2]
            if h < 1 or w < 1:
                raise ValueError("an on-device view prior must not be empty, not %d x %d" % (h, w))
            row = w * (tail[0] if tail else 1)           # elements of a packed row
            if not t[0].is_contiguous() or (h > 1 and t.stride(0) < row):
                t = t.contiguous()
            planes.append(t)
            pitches.append(t.element_size() * (t.stride(0) if h > 1 else row))
        d, z, ids = planes
        h, w = d.shape
        stream = C.c_void_p(torch.cuda.current_stream(d.device).cuda_stream)
        ptr = [None if t is None else C.c_void_p(t.data_ptr()) for t in planes]
        if z is None and ids is None:
            self._check(self._lib.b200mvs_set_view_prior_device(self._h, view_id, ptr[0], w, h, pitches[0], int(stride),
                                                                stream))
        else:
            self._check(self._lib.b200mvs_set_view_prior_state_device(self._h, view_id, ptr[0], ptr[1], ptr[2], w, h,
                                                                      *pitches, int(stride), stream))

    def set_view_prior_relative(self, view_id: int, values, stride: int, kind: str = "disparity") -> dict:
        """Prior from a map known up to a transform (b200mvs_set_view_prior_relative[_device]), such as a monocular
        network's output: kind "disparity" (1/z = s d + t), "depth" (z = s d + t) or "depth_scale" (z = s d), with z the
        planar depth.  The view's registered features fix s and t on the device, robustly, and the map becomes a depth
        prior in MVE's convention, installed as set_view_prior installs one.  values is an H x W float32 numpy array (the
        host route) or a torch.float32 CUDA tensor on the scene's device at any row stride (the device route, after the
        work of its current stream).  Returns the fit: scale, shift, n_obs, n_inliers, median_rel_err.  A failed fit
        raises B200MVSError with the fit dict as .fit, and leaves the view's previous prior in place; a bad kind, shape,
        dtype or device raises ValueError."""
        if kind not in PRIOR_KINDS:
            raise ValueError("kind is %r, not one of %s" % (kind, ", ".join(PRIOR_KINDS)))
        fit = PriorFit()
        if isinstance(values, np.ndarray):
            if values.ndim != 2 or values.dtype != np.float32:
                raise ValueError("a relative view prior is an H x W float32 array, not %s %s" % (values.dtype, values.shape))
            v = np.ascontiguousarray(values)
            h, w = v.shape
            rc = self._lib.b200mvs_set_view_prior_relative(self._h, view_id, _p(v), w, h, int(stride), PRIOR_KINDS[kind],
                                                           C.byref(fit))
        else:
            torch = _torch()
            if (not isinstance(values, torch.Tensor) or values.dtype != torch.float32 or values.dim() != 2
                    or not values.is_cuda
                    or (self.device != DEVICE_NONE and values.device != torch.device(self._torch_device()))):
                where = "the scene's device" if self.device == DEVICE_NONE else self._torch_device()
                raise ValueError("a relative view prior is an H x W float32 numpy array or torch.float32 tensor on %s, "
                                 "not %s" % (where, "%s %s on %s" % (values.dtype, tuple(values.shape), values.device)
                                             if isinstance(values, torch.Tensor) else type(values).__name__))
            h, w = values.shape
            if h < 1 or w < 1:
                raise ValueError("a relative view prior must not be empty, not %d x %d" % (h, w))
            if not values[0].is_contiguous() or (h > 1 and values.stride(0) < w):
                values = values.contiguous()
            pitch = 4 * (values.stride(0) if h > 1 else w)
            stream = torch.cuda.current_stream(values.device).cuda_stream
            rc = self._lib.b200mvs_set_view_prior_relative_device(self._h, view_id, C.c_void_p(values.data_ptr()), w, h,
                                                                  pitch, int(stride), PRIOR_KINDS[kind],
                                                                  C.c_void_p(stream), C.byref(fit))
        try:
            self._check(rc)
        except B200MVSError as e:
            e.fit = fit.as_dict()
            raise
        return fit.as_dict()

    def set_features(self, pos: np.ndarray, refs: Sequence[np.ndarray]):
        """mve::Bundle::Features (bundle.h:51-60)."""
        off = np.zeros(len(refs) + 1, np.int32)
        if len(refs):
            off[1:] = np.cumsum([len(r) for r in refs])
        ids = np.concatenate(refs).astype(np.int32) if len(refs) else np.zeros(0, np.int32)
        p = np.ascontiguousarray(pos, np.float32)
        self._check(self._lib.b200mvs_set_features(self._h, len(refs), _p(p), _p(off), _p(ids)))

    def num_levels(self, view_id: int) -> int:
        return self._check(self._lib.b200mvs_num_levels(self._h, view_id))

    def level(self, view_id: int, level: int, on_device: bool = False):
        """The level's packed RGB bytes, H x W x 3: a numpy array, or with on_device a torch uint8 tensor on cuda:<device>
        (b200mvs_get_level_device, ordered after the current stream's work)."""
        w, h = C.c_int(), C.c_int()
        self._check(self._lib.b200mvs_get_level(self._h, view_id, level, C.byref(w), C.byref(h), None))
        if on_device:
            torch = _torch()
            out = torch.empty((h.value, w.value, 3), dtype=torch.uint8, device=self._torch_device())
            stream = torch.cuda.current_stream(out.device).cuda_stream
            self._check(self._lib.b200mvs_get_level_device(self._h, view_id, level, C.byref(w), C.byref(h),
                                                           C.c_void_p(out.data_ptr()), C.c_void_p(stream)))
            return out
        out = np.empty((h.value, w.value, 3), np.uint8)
        self._check(self._lib.b200mvs_get_level(self._h, view_id, level, C.byref(w), C.byref(h), _p(out)))
        return out

    def _torch_device(self):
        if self.device == DEVICE_NONE:
            raise B200MVSError(ERR_CUDA, "planning context (B200MVS_DEVICE_NONE): no CUDA device, b200mvs has no CPU fallback")
        return "cuda:%d" % self.device

    def global_view_selection(self, settings: Settings, ref_view: int) -> List[int]:
        """DMRecon::globalViewSelection (dmrecon.cc:211-241)."""
        out = np.empty(64, np.int32)
        n = self._check(self._lib.b200mvs_global_view_selection(self._h, C.byref(settings), ref_view, _p(out), 64))
        return out[:n].tolist()

    def set_patch_mode(self, mode: int = 0, thread_min: int = -1):
        """Engine knob: 1 = one warp per patch, 2 = one thread per patch, 0 = by size (see include/b200mvs.h)."""
        self._check(self._lib.b200mvs_set_patch_mode(self._h, mode, thread_min))

    def set_frontier_capacity(self, entries_per_px: float = 2.0, min_entries: int = 65536):
        """Initial frontier capacity of a launch: max(ceil(entries_per_px * pixels), seeds, min_entries) entries; a launch
        that needs more grows its frontier and resumes (see include/b200mvs.h).  Also sizes working_set / plan_batches."""
        if min_entries < 0:
            raise B200MVSError(ERR_INVALID_ARG, "frontier capacity: min_entries must not be negative")
        self._check(self._lib.b200mvs_set_frontier_capacity(self._h, float(entries_per_px), int(min_entries)))

    def frontier_info(self) -> dict:
        """Frontier of the last reconstruct(): initial and final capacity in entries, number of resumes."""
        v = [C.c_uint64() for _ in range(3)]
        self._check(self._lib.b200mvs_frontier_info(self._h, *(C.byref(x) for x in v)))
        return dict(initial=v[0].value, final=v[1].value, resumes=v[2].value)

    def plan_info(self) -> dict:
        """How the last reconstruct(), reconstruct(on_device=True) or reconstruct_pointset() planned its views: prepared by
        plan_views(), on the device or on host threads, with the planning phase's wall and kernel times and its largest
        device allocation."""
        p = PlanInfo()
        self._check(self._lib.b200mvs_plan_stats(self._h, C.byref(p)))
        return p.as_dict()

    def plan_views(self, settings: Settings, ref_views: Sequence[int]):
        """Global view selection + seed lists of these reference views ahead of their reconstruct() call; safe to call from
        another thread while a reconstruct() of a previous batch is running (ctypes releases the GIL)."""
        refs = np.asarray(ref_views, np.int32)
        self._check(self._lib.b200mvs_plan_views(self._h, C.byref(settings), len(refs), _p(refs)))

    def optimize_patches(self, settings: Settings, ref_view: int, global_ids: Sequence[int], patches: np.ndarray,
                         stats: Optional[Stats] = None) -> np.ndarray:
        """Batch of independent mvs::PatchOptimization runs (patch-level parity entry)."""
        patches = np.ascontiguousarray(patches, dtype=PATCH_IN)
        out = np.zeros(len(patches), PATCH_OUT)
        g = np.asarray(global_ids, np.int32)
        self._check(self._lib.b200mvs_optimize_patches(self._h, C.byref(settings), ref_view, _p(g), len(g), _p(patches),
                                                       len(patches), _p(out), C.byref(stats) if stats is not None else None))
        return out

    def reconstruct(self, settings: Settings, ref_views: Sequence[int], download: bool = True,
                    want=("depth", "conf", "dz", "normal", "view_ids"), out=None, progress=None, on_device: bool = False,
                    stream=None, scales=None):
        """DMRecon::start for a batch of reference views. Returns (list of map dicts or None, Stats).
        The maps: depth, conf [H, W] float32, dz [H, W, 2], normal [H, W, 3] float32, view_ids [H, W, 4] int32.
        out: optional list (one dict per view) of preallocated C-contiguous host arrays (e.g. pinned) of those dtypes and
        shapes to receive the maps, else ValueError.
        progress: optional (Progress * n) array, updated live; setting .cancelled from another thread cancels the run.
        on_device: the maps as torch CUDA tensors on cuda:<device> (b200mvs_reconstruct_device), without leaving the
        device.  They are allocated by torch, or taken from `out` (contiguous CUDA tensors of those dtypes, shapes and
        device, else ValueError).  The call's work is ordered after what `stream` (a torch.cuda.Stream; default: the
        current stream of the scene's device) has enqueued, and the maps are complete when it returns.
        scales: one pyramid level per reference view instead of settings.scale (b200mvs_reconstruct_levels and
        b200mvs_reconstruct_levels_device): view ref_views[j] is reconstructed at level scales[j], and its maps have
        that level's size.  A view may appear at several levels, a (view, level) pair once."""
        refs = np.asarray(ref_views, np.int32)
        levels = levels_array(scales, len(refs))
        if download and on_device:
            return self._reconstruct_device(settings, refs, want, out, progress, stream, levels)
        stats = Stats()
        failed = C.c_int32(-1)
        maps_arr, results = None, None
        sizes = self._map_sizes(refs, settings.scale if levels is None else levels) if download else None
        if sizes is not None:
            maps_arr, results = self._map_buffers(sizes, want, out)
        if levels is None:
            rc = self._lib.b200mvs_reconstruct(self._h, C.byref(settings), len(refs), _p(refs), maps_arr, progress,
                                               C.byref(stats), C.byref(failed))
        else:
            rc = self._lib.b200mvs_reconstruct_levels(self._h, C.byref(settings), len(refs), _p(refs), _p(levels), maps_arr,
                                                      progress, C.byref(stats), C.byref(failed))
        self._raise(rc, failed)
        return results, stats

    def _map_sizes(self, refs, scale):
        """(H, W) of each reference view at level `scale` (an int, or one level per view), or None when a view has no
        such level: the reconstruct call then reports it with the reference's own message (dmrecon.cc:37-75), before it
        looks at any buffer."""
        sizes = []
        for j, r in enumerate(refs):
            w, h = C.c_int(), C.c_int()
            level = int(scale) if np.ndim(scale) == 0 else int(scale[j])
            if level < 0 or self._lib.b200mvs_get_level(self._h, int(r), level, C.byref(w), C.byref(h), None) != 0:
                return None
            sizes.append((h.value, w.value))
        return sizes

    @staticmethod
    def _map_buffers(sizes, want, out, dev=None):
        """The maps of views of these (H, W) sizes and the b200mvs_maps array that points at them: out[j]'s arrays,
        checked against _MAP_LAYOUT (else ValueError), or new ones for depth and the maps in `want`.  Host arrays, or
        with `dev` CUDA tensors on that device."""
        torch = _torch() if dev is not None else None
        maps_arr = (_Maps * max(len(sizes), 1))()
        results = []
        for j, (H, W) in enumerate(sizes):
            if out is None:
                d = {k: np.empty((H, W) + tail, nd) if dev is None else
                     torch.empty((H, W) + tail, dtype=getattr(torch, td), device=dev)
                     for k, (tail, nd, td) in _MAP_LAYOUT.items() if k == "depth" or k in want}
            else:
                d = out[j]
                for k, a in d.items():
                    if k not in _MAP_LAYOUT:
                        raise ValueError("out[%d] has an unknown map %r" % (j, k))
                    tail, nd, td = _MAP_LAYOUT[k]
                    shape = (H, W) + tail
                    if dev is None:
                        if a.shape != shape or a.dtype != nd or not a.flags["C_CONTIGUOUS"]:
                            raise ValueError("out[%d][%s] has the wrong shape" % (j, k))
                    elif (not isinstance(a, torch.Tensor) or a.device != dev or a.dtype != getattr(torch, td)
                          or tuple(a.shape) != shape or not a.is_contiguous()):
                        raise ValueError("out[%d][%s] must be a contiguous %s tensor of shape %s on %s"
                                         % (j, k, getattr(torch, td), shape, dev))
            results.append(d)
            for k in _MAP_LAYOUT:
                setattr(maps_arr[j], k, (d[k].ctypes.data if dev is None else d[k].data_ptr()) if k in d else None)
        return maps_arr, results

    def _raise(self, rc: int, failed):
        if rc != 0:
            self._raise_fetch_error()
            msg = self._lib.b200mvs_last_error(self._h).decode()
            if failed.value >= 0:
                msg += " (view %d)" % failed.value
            raise B200MVSError(rc, msg, failed.value)

    def _reconstruct_device(self, settings, refs, want, out, progress, stream, levels=None):
        stats = Stats()
        failed = C.c_int32(-1)
        # without sizes or a device, empty buffers: b200mvs_reconstruct_device reports the error before it looks at them
        maps_arr, results, cuda_stream = (_Maps * max(len(refs), 1))(), None, None
        sizes = self._map_sizes(refs, settings.scale if levels is None else levels)
        if sizes is not None and self.device != DEVICE_NONE:
            torch = _torch()
            dev = torch.device(self._torch_device())
            maps_arr, results = self._map_buffers(sizes, want, out, dev)
            cuda_stream = (stream if stream is not None else torch.cuda.current_stream(dev)).cuda_stream
        if levels is None:
            rc = self._lib.b200mvs_reconstruct_device(self._h, C.byref(settings), len(refs), _p(refs), maps_arr,
                                                      C.c_void_p(cuda_stream), progress, C.byref(stats), C.byref(failed))
        else:
            rc = self._lib.b200mvs_reconstruct_levels_device(self._h, C.byref(settings), len(refs), _p(refs), _p(levels),
                                                             maps_arr, C.c_void_p(cuda_stream), progress, C.byref(stats),
                                                             C.byref(failed))
        self._raise(rc, failed)
        return results, stats

    def reconstruct_pointset(self, settings: Settings, ref_views: Sequence[int], options=None, masks=None, progress=None,
                             on_device: bool = False, scales=None):
        """DMRecon::start for a batch of reference views and scene2pset of their maps, without the maps leaving the device
        (b200mvs_pset_add_reconstruction).  options / masks / on_device: as for mve_b200.depthmap.scene_pointset (the masks
        are applied after the reconstruction, unlike set_view_mask, which keeps background pixels from being reconstructed
        at all; on_device keeps the point set on the device and returns CUDA tensors);
        progress and scales: as for reconstruct().  Returns (the dict of depthmap.scene_pointset, Stats)."""
        from . import depthmap
        return depthmap.reconstruct_pointset(self, settings, ref_views, options, masks, progress, on_device, scales)


class DMRecon:
    """mvs::DMRecon (dmrecon.h:40-68): construct with a scene and settings, call start()."""

    def __init__(self, scene: Scene, settings: Settings, ref_view_nr: int):
        if ref_view_nr < 0 or ref_view_nr >= scene.n_views:
            raise ValueError("Master view index out of bounds")          # dmrecon.cc:37-38
        if settings.scale < 0:
            raise ValueError("Invalid scale factor")                     # dmrecon.cc:41-42
        self.scene, self.settings, self.ref_view_nr = scene, settings, ref_view_nr
        self.maps = None
        self.stats = None

    def getRefViewNr(self) -> int:
        return self.ref_view_nr

    def start(self):
        maps, stats = self.scene.reconstruct(self.settings, [self.ref_view_nr])
        self.maps, self.stats = maps[0], stats
        return self.maps
