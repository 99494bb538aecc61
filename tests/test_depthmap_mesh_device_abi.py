"""The argument checks of b200mvs_depthmap_pointset_device that come before any device call, with their exact codes and
messages from both error getters, on a machine without a GPU: the pointers are never dereferenced.  An empty batch
returns 0 without touching anything, a NULL array included."""
import ctypes as C

import pytest

INVALID = -1
FN = "b200mvs_depthmap_pointset_device"
BASE = 1 << 40                    # a fake, 4-byte aligned address; nothing at or after it is read
MB = 1 << 20


def _lib():
    from mve_b200 import depthmap as D
    return D._lib()


def _mesh(**kw):
    """One 8 x 4 map at BASE + slot MB, all outputs wanted, capacities of a vertex per pixel and two faces per block."""
    from mve_b200.depthmap import DmMesh
    m = DmMesh()
    m.width, m.height = 8, 4
    m.invproj[:] = [1, 0, 0, 0, 1, 0, 0, 0, 1]
    m.cap_vertices, m.cap_faces = 32, 42
    m.n_vertices = m.n_faces = 7
    slot = kw.pop("slot", 0)
    at = BASE + slot * 16 * MB
    m.depth_dev = at
    for k, name in enumerate(("vertex_ids", "vertices", "colors", "faces", "normals", "confidences", "scales")):
        setattr(m, name, at + (k + 1) * MB)
    for k, v in kw.items():
        setattr(m, k, v)
    return m


def _call(L, meshes, conf_iterations=4):
    arr = (type(meshes[0]) * len(meshes))(*meshes)
    return L.b200mvs_depthmap_pointset_device(0, len(meshes), arr, 5.0, conf_iterations, 2.5, None), arr


def _expect(L, rc, msg):
    assert (rc, L.b200mvs_last_error(None).decode()) == (INVALID, "%s: %s" % (FN, msg))
    assert L.b200mvs_depthmap_last_error().decode() == "%s: %s" % (FN, msg)


def test_empty_batch_touches_nothing():
    L = _lib()
    assert L.b200mvs_depthmap_pointset_device(0, 0, None, 5.0, 4, 2.5, None) == 0
    # with a device that does not exist and a negative conf_iterations: nothing is looked at
    assert L.b200mvs_depthmap_pointset_device(999, 0, None, 5.0, -1, 2.5, None) == 0


def test_negative_count_and_null_maps():
    L = _lib()
    _expect(L, L.b200mvs_depthmap_pointset_device(0, -1, None, 5.0, 4, 2.5, None), "n_maps is -1, must not be negative")
    _expect(L, L.b200mvs_depthmap_pointset_device(0, 2, None, 5.0, 4, 2.5, None), "maps is NULL")


X = BASE + 64 * MB                 # far from every buffer of slots 0 and 1

CASES = [
    ("conf_iterations", dict(), -1, "conf_iterations is -1: Invalid amount of iterations"),
    ("null depth", dict(m1=dict(depth_dev=None)), 4, "maps[1].depth_dev is NULL"),
    ("width", dict(m0=dict(width=1)), 4, "maps[0].width is 1, must be at least 2"),
    ("height", dict(m1=dict(height=-5)), 4, "maps[1].height is -5, must be at least 2"),
    ("too large", dict(m1=dict(width=65536, height=65536)), 4,
     "maps[1] has 4294967296 pixels (width x height), more than 2147483646"),
    # the smallest square map above 2^31 - 2 pixels: its faces would not count in the 32 bits of the scan
    ("too large for the scan", dict(m0=dict(width=46341, height=46341)), 4,
     "maps[0] has 2147488281 pixels (width x height), more than 2147483646"),
    ("colour channels", dict(m0=dict(color_dev=X, color_channels=5)), 4, "maps[0].color_channels is 5, must be 1 to 4"),
    ("no colour channels", dict(m1=dict(color_dev=X, color_channels=0)), 4, "maps[1].color_channels is 0, must be 1 to 4"),
    ("capacity wraps", dict(m1=dict(cap_vertices=1 << 62)), 4,
     "maps[1].vertices: 4611686018427387904 x 12 bytes from 0x10001200000 wrap the address space (cap_vertices)"),
    ("faces wrap", dict(m0=dict(cap_faces=(1 << 64) - 1)), 4,
     "maps[0].faces: 18446744073709551615 x 12 bytes from 0x10000400000 wrap the address space (cap_faces)"),
    ("outputs overlap", dict(m0=dict(cap_vertices=MB)), 4, "maps[0].vertices overlaps maps[0].colors"),
    ("output on a depth map", dict(m1=dict(scales=BASE)), 4, "maps[1].scales overlaps maps[0].depth_dev"),
    ("output on a colour image", dict(m0=dict(color_dev=X, color_channels=3), m1=dict(faces=X + 88)), 4,
     "maps[1].faces overlaps maps[0].color_dev"),
    ("same output twice", dict(m1=dict(normals=BASE + 5 * MB)), 4, "maps[0].normals overlaps maps[1].normals"),
    ("vertex ids on a later map's output", dict(m0=dict(vertex_ids=BASE + 16 * MB + 2 * MB + 64)), 4,
     "maps[0].vertex_ids overlaps maps[1].vertices"),
]


@pytest.mark.parametrize("name,mods,iters,msg", CASES, ids=[c[0] for c in CASES])
def test_argument_errors(name, mods, iters, msg):
    L = _lib()
    meshes = [_mesh(slot=0, **mods.get("m0", {})), _mesh(slot=1, **mods.get("m1", {}))]
    rc, arr = _call(L, meshes, conf_iterations=iters)
    _expect(L, rc, msg)
    # nothing is written back before the checks pass
    assert [(m.n_vertices, m.n_faces) for m in arr] == [(7, 7), (7, 7)]


def test_count_only_maps_skip_output_checks():
    L = _lib()
    # map 1 wants nothing: its capacities are not checked, so the call goes on to the device (none here) and fails there,
    # not on the capacity; map 0's bad capacity is still found
    bare = dict(vertex_ids=None, vertices=None, colors=None, faces=None, normals=None, confidences=None, scales=None)
    rc, _ = _call(L, [_mesh(slot=0, cap_faces=(1 << 64) - 1), _mesh(slot=1, cap_vertices=1 << 62, **bare)])
    _expect(L, rc, "maps[0].faces: 18446744073709551615 x 12 bytes from 0x10000400000 wrap the address space (cap_faces)")
    rc, _ = _call(L, [_mesh(slot=0, **bare), _mesh(slot=1, cap_vertices=1 << 62, **bare)])
    assert rc != 0 and "cap_vertices" not in L.b200mvs_last_error(None).decode()


def test_map_checks_come_before_overlaps():
    L = _lib()
    # map 0 writes onto map 1's depth, and map 1 has no height: the maps' own fields are checked first
    rc, _ = _call(L, [_mesh(slot=0, vertices=BASE + 16 * MB), _mesh(slot=1, height=0)])
    _expect(L, rc, "maps[1].height is 0, must be at least 2")
