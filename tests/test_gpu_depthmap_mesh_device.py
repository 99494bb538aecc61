"""depthmap_triangulate and the per-view point set on batches of maps in device memory (-m gpu):
b200mvs_depthmap_pointset_device through depthmap_pointset_maps and depthmap_triangulate_maps.

Every map's outputs are byte for byte the host entry points' on that map alone (which test_gpu_depthmap_ops and
test_gpu_depthmap_edges pin to the reference): every triangulation case of depthmap_edges_ref.npz and depthmap_ops_ref.npz
in one shuffled batch of mixed sizes under several settings, and the cleaned maps and level images of real
reconstructions.  Also covered: batches split into chunks (more than 2^28 pixels, and one map larger than that),
count-only maps, overflow and rejections that leave every buffer untouched, the order after the caller's stream, and
no device memory kept after a call."""
import ctypes as C

import numpy as np
import pytest

from tests import pset_reference as S
from tests.test_gpu_depthmap_edges import DD_EDGE, tri_cases
from tests.test_gpu_depthmap_ops import TRI_CASES, tri_inputs
from tests.util import golden_scene

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID, OVERFLOW = -1, -5
FN = "b200mvs_depthmap_pointset_device"
KEYS = ("vertex_ids", "vertices", "colors", "faces", "normals", "confidences", "scales")
CTW = np.array([[0.36, 0.48, -0.8, 1.5], [-0.8, 0.6, 0.0, -2.0], [0.48, 0.64, 0.6, 0.25], [0, 0, 0, 1]], F32)


def _torch():
    import torch
    return torch


def _cuda(a):
    return None if a is None else _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _bytes(t):
    """The bytes of a host array or CUDA tensor (uint32 tensors through their int32 bits)."""
    torch = _torch()
    if isinstance(t, torch.Tensor):
        if t.dtype not in (torch.float32, torch.int32, torch.uint8):
            t = t.view(torch.int32)
        return t.cpu().numpy().tobytes()
    return np.ascontiguousarray(t).tobytes()


def _same(got, want, what):
    for k in KEYS:
        if k not in want:
            continue
        assert (got[k] is None) == (want[k] is None), (what, k)
        if want[k] is not None:
            g = got[k]
            assert g.is_cuda and tuple(g.shape) == want[k].shape, (what, k, tuple(g.shape), want[k].shape)
            assert _bytes(g) == _bytes(want[k]), (what, k)


def fixture_maps():
    """(name, depth, invproj, colour or None, cam_to_world or None): every case of the two fixtures, a camera-to-world
    matrix on every third map"""
    out = [(n, c["dm"], c["invproj"], c["color"]) for n, c in tri_cases().items()]
    for kind, _, color in TRI_CASES:
        dm, ip, ci = tri_inputs(kind, color)
        out.append(("ops_%s_%d" % (kind, int(color)), dm, ip, ci))
    return [(n, d, ip, c, CTW if j % 3 == 1 else None) for j, (n, d, ip, c) in enumerate(out)]


@pytest.fixture(scope="module")
def fixtures():
    maps = fixture_maps()
    order = np.random.default_rng(5).permutation(len(maps))
    return [maps[j] for j in order]


# (dd_factor, conf_iterations, scale_factor): the app's, the edge fixtures' thresholds and depths, dd off
SETTINGS = [(5.0, 4, 2.5), (float(DD_EDGE[1]), 1, 0.0), (float(DD_EDGE[2]), 300, 1.0), (0.0, 7, 2.5), (2.0, 256, 2.5)]


# ---------------------------------------------------------------- 1. the fixture cases in one shuffled batch
@pytest.mark.parametrize("dd,iters,scale", SETTINGS)
def test_fixture_cases_batched(fixtures, dd, iters, scale):
    from mve_b200 import depthmap as D
    names = [f[0] for f in fixtures]
    dms = [_cuda(f[1]) for f in fixtures]
    got = D.depthmap_pointset_maps(dms, [f[2] for f in fixtures], [_cuda(f[3]) for f in fixtures], [f[4] for f in fixtures],
                                   dd_factor=dd, with_normals=True, conf_iterations=iters, scale_factor=scale)
    assert len({d.shape for d in dms}) > 10
    for n, (_, dm, ip, ci, ctw), g in zip(names, fixtures, got):
        want = D.depthmap_pointset(dm, ip, dd_factor=dd, cam_to_world=ctw, color=ci, with_normals=True, conf_iterations=iters,
                                   scale_factor=scale)
        _same(g, want, n)


def test_triangulate_and_single_map_forms(fixtures):
    from mve_b200 import depthmap as D
    dms = [_cuda(f[1]) for f in fixtures]
    cols = [_cuda(f[3]) for f in fixtures]
    tri = D.depthmap_triangulate_maps(dms, [f[2] for f in fixtures], cols, [f[4] for f in fixtures])
    for (n, dm, ip, ci, ctw), t, d, c in zip(fixtures, tri, dms, cols):
        want = D.depthmap_triangulate(dm, ip, cam_to_world=ctw, color=ci)
        assert set(t) == {"vertex_ids", "vertices", "colors", "faces"}
        _same(t, want, n)
        # the single-map forms take CUDA tensors
        _same(D.depthmap_triangulate(d, ip, cam_to_world=ctw, color=c), want, n)
        if n in ("complex", "special", "ops_golden_1"):
            _same(D.depthmap_pointset(d, ip, color=c, cam_to_world=ctw),
                  D.depthmap_pointset(dm, ip, color=ci, cam_to_world=ctw), n)
    # the host forms are unchanged: numpy in, numpy out
    assert isinstance(D.depthmap_triangulate(fixtures[0][1], fixtures[0][2])["faces"], np.ndarray)


# ---------------------------------------------------------------- 2. real reconstructions
@pytest.mark.parametrize("name", ["T0", "T5"])
def test_reconstruction_maps(name):
    from mve_b200 import depthmap as D, dmrecon
    s = golden_scene(name)
    sc = dmrecon.Scene.from_synth(s)
    try:
        st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
        refs = list(range(s.n_views))
        maps, _ = sc.reconstruct(st, refs, want=("depth", "conf"), on_device=True)
        levels = [sc.level(v, st.scale, on_device=True) for v in refs]
    finally:
        sc.close()
    dms = [m["depth"] for m in maps]
    D.depthmap_confidence_clean_maps(dms, [m["conf"] for m in maps])
    D.depthmap_cleanup_maps(dms, 100, out=dms)
    ips, ctws = [], []
    for j, (v, d) in enumerate(zip(refs, dms)):
        h, w = d.shape
        ips.append(np.linalg.inv(S.calibration(S.camera_of(s, v), w, h).reshape(3, 3).astype(np.float64)).astype(F32))
        ctws.append(CTW if j % 2 else None)
    got = D.depthmap_pointset_maps(dms, ips, levels, ctws, with_normals=True, conf_iterations=4, scale_factor=2.5)
    total = 0
    for j, (d, lv, g) in enumerate(zip(dms, levels, got)):
        want = D.depthmap_pointset(d.cpu().numpy(), ips[j], cam_to_world=ctws[j], color=lv.cpu().numpy(), with_normals=True,
                                   conf_iterations=4, scale_factor=2.5)
        _same(g, want, (name, j))
        total += len(want["faces"])
    assert total > 1000


# ---------------------------------------------------------------- 3. chunks
def _sparse(h, w, seed, keep):
    """A mostly-zero map: a few random pixels and one smooth square patch are non-zero, so the meshes stay small"""
    torch = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = torch.zeros((h, w), device="cuda")
    d[torch.rand((h, w), generator=g, device="cuda") < keep] = 3.0
    y0, x0 = (seed * 997) % (h - 300), (seed * 1531) % (w - 300)
    d[y0:y0 + 256, x0:x0 + 256] = 2.0 + torch.rand((256, 256), generator=g, device="cuda") * 0.01
    return d


def _ip(h, w):
    ax = float(max(w, h))
    return np.array([1 / ax, 0, -0.5 * w / ax, 0, 1 / ax, -0.5 * h / ax, 0, 0, 1], F32)


def test_chunks_equal_one_call_per_map():
    from mve_b200 import depthmap as D
    torch = _torch()
    # five 8192 x 8192 maps: 5 * 2^26 pixels, chunks of four maps and of one
    dms = [_sparse(8192, 8192, seed=j, keep=0.002) for j in range(5)]
    ips = [_ip(8192, 8192)] * 5
    kw = dict(with_normals=True, conf_iterations=4, scale_factor=2.5)
    batch = D.depthmap_pointset_maps(dms, ips, **kw)
    assert all(len(b["faces"]) > 1000 for b in batch)
    for j, d in enumerate(dms):
        one = D.depthmap_pointset_maps([d], [ips[j]], **kw)[0]
        for k in KEYS:
            assert (batch[j][k] is None) == (one[k] is None), (j, k)
            if one[k] is not None:
                assert batch[j][k].shape == one[k].shape and torch.equal(batch[j][k].view(torch.int32), one[k].view(torch.int32)), (j, k)
    del batch, one, dms
    torch.cuda.empty_cache()
    # a single map larger than 2^28 pixels is a chunk of its own, against the host entry point
    big = _sparse(16384, 16400, seed=9, keep=0.001)
    got = D.depthmap_pointset_maps([big], [_ip(16384, 16400)], **kw)[0]
    want = D.depthmap_pointset(big.cpu().numpy(), _ip(16384, 16400), **kw)
    _same(got, want, "big")


# ---------------------------------------------------------------- 4. count-only maps, overflow and rejections
def _lib():
    from mve_b200 import depthmap as D
    return D._lib()


def _meshes(dms, ips):
    from mve_b200.depthmap import DmMesh
    arr = (DmMesh * len(dms))()
    for m, d, ip in zip(arr, dms, ips):
        m.depth_dev, m.height, m.width = d.data_ptr(), d.shape[0], d.shape[1]
        m.invproj[:] = [float(x) for x in ip]
    return arr


def _outputs(torch, h, w, nv, nf, fill):
    """Every output of one map, at sentinel bytes"""
    return dict(vertex_ids=torch.full((h, w), fill, dtype=torch.int32, device="cuda"),
                vertices=torch.full((nv, 3), fill, dtype=torch.int32, device="cuda"),
                faces=torch.full((nf, 3), fill, dtype=torch.int32, device="cuda"),
                normals=torch.full((nv, 3), fill, dtype=torch.int32, device="cuda"),
                confidences=torch.full((nv,), fill, dtype=torch.int32, device="cuda"),
                scales=torch.full((nv,), fill, dtype=torch.int32, device="cuda"))


def _run(arr, iters=4):
    L = _lib()
    stream = _torch().cuda.current_stream().cuda_stream
    rc = L.b200mvs_depthmap_pointset_device(0, len(arr), arr, 5.0, iters, 2.5, C.c_void_p(stream))
    return rc, L.b200mvs_last_error(None).decode()


@pytest.fixture(scope="module")
def three():
    """Three edge-case maps of different sizes, their host results"""
    from mve_b200 import depthmap as D
    cases = tri_cases()
    picks = [cases[n] for n in ("257x131", "complex", "ragged")]
    want = [D.depthmap_pointset(c["dm"], c["invproj"], with_normals=True, conf_iterations=4, scale_factor=2.5) for c in picks]
    return [_cuda(c["dm"]) for c in picks], [c["invproj"] for c in picks], want


def test_count_only_maps_in_a_mixed_batch(three):
    torch = _torch()
    dms, ips, want = three
    arr = _meshes(dms, ips)
    outs = {}
    for j in (0, 2):                                    # map 1 is only counted
        nv, nf = len(want[j]["vertices"]), len(want[j]["faces"])
        outs[j] = _outputs(torch, *dms[j].shape, nv, nf, 0)
        for k, t in outs[j].items():
            setattr(arr[j], k, t.data_ptr())
        arr[j].cap_vertices, arr[j].cap_faces = nv, nf
    arr[1].cap_vertices = arr[1].cap_faces = 0
    assert _run(arr)[0] == 0
    assert [(m.n_vertices, m.n_faces) for m in arr] == [(len(w["vertices"]), len(w["faces"])) for w in want]
    for j in (0, 2):
        for k, t in outs[j].items():
            assert _bytes(t) == _bytes(want[j][k]), (j, k)


def test_maps_without_a_vertex_buffer(three):
    """Maps with outputs but no vertices buffer: vertex ids and faces only, colours only, confidences only.  The call
    computes their vertices in its workspace, and each output equals the host entry point's."""
    from mve_b200 import depthmap as D
    torch = _torch()
    dms, ips, _ = three
    h1, w1 = dms[1].shape
    ci = np.random.default_rng(7).integers(0, 256, size=(h1, w1, 3), dtype=np.uint8)
    want = [D.depthmap_triangulate(dms[0].cpu().numpy(), ips[0]),
            D.depthmap_triangulate(dms[1].cpu().numpy(), ips[1], color=ci),
            D.depthmap_pointset(dms[2].cpu().numpy(), ips[2], with_normals=False, conf_iterations=4, scale_factor=None)]
    wanted = [("vertex_ids", "faces"), ("colors",), ("confidences",)]
    shapes = dict(vertex_ids=lambda j, nv, nf: tuple(dms[j].shape), faces=lambda j, nv, nf: (nf, 3),
                  colors=lambda j, nv, nf: (nv, 4), confidences=lambda j, nv, nf: (nv,))
    col = _cuda(ci)
    arr = _meshes(dms, ips)
    arr[1].color_dev, arr[1].color_channels = col.data_ptr(), 3
    outs = []
    for j, keys in enumerate(wanted):
        nv, nf = len(want[j]["vertices"]), len(want[j]["faces"])
        o = {k: torch.full(shapes[k](j, nv, nf), 0x7F7F7F7F, dtype=torch.int32, device="cuda") for k in keys}
        for k, t in o.items():
            setattr(arr[j], k, t.data_ptr())
        arr[j].cap_vertices, arr[j].cap_faces = nv, nf
        outs.append(o)
    assert _run(arr)[0] == 0
    assert [(m.n_vertices, m.n_faces) for m in arr] == [(len(w["vertices"]), len(w["faces"])) for w in want]
    for j, o in enumerate(outs):
        for k, t in o.items():
            assert _bytes(t) == _bytes(want[j][k]), (j, k)


def test_overflow_writes_counts_and_no_output(three):
    torch = _torch()
    dms, ips, want = three
    for k_over in (0, 2):
        arr = _meshes(dms, ips)
        outs = []
        for j in range(3):
            nv, nf = len(want[j]["vertices"]), len(want[j]["faces"])
            o = _outputs(torch, *dms[j].shape, nv, nf, 0x7F7F7F7F)
            for k, t in o.items():
                setattr(arr[j], k, t.data_ptr())
            arr[j].cap_vertices, arr[j].cap_faces = nv, nf - (j == k_over)
            outs.append(o)
        rc, msg = _run(arr)
        nv, nf = len(want[k_over]["vertices"]), len(want[k_over]["faces"])
        assert (rc, msg) == (OVERFLOW, "%s: maps[%d] has %d vertices and %d faces, cap_vertices is %d and cap_faces %d"
                             % (FN, k_over, nv, nf, nv, nf - 1))
        assert [(m.n_vertices, m.n_faces) for m in arr] == [(len(w["vertices"]), len(w["faces"])) for w in want]
        torch.cuda.synchronize()
        for o in outs:
            for k, t in o.items():
                assert bool((t == 0x7F7F7F7F).all()), (k_over, k)


def test_rejections_leave_buffers_untouched(three):
    torch = _torch()
    dms, ips, want = three
    h, w = dms[0].shape
    nv, nf = len(want[0]["vertices"]), len(want[0]["faces"])
    outs = _outputs(torch, h, w, nv, nf, 0x5A5A5A5A)
    host = np.full(nv * 3, 5.0, F32)
    pinned = torch.full((nv * 3,), 6.0).pin_memory()
    raw = torch.full((nv * 3 + 4,), 9.0, device="cuda")
    bufs = list(outs.values()) + [pinned, raw] + dms
    before = [_bytes(b) for b in bufs] + [host.tobytes()]
    P = lambda t: t.data_ptr()                                             # noqa: E731
    cases = [
        (dict(vertices=host.ctypes.data), "maps[0].vertices is pageable host memory, not device memory"),
        (dict(normals=P(pinned)), "maps[0].normals is pinned host memory, not device memory"),
        (dict(scales=P(raw) + 2), "maps[0].scales is not 4-byte aligned"),
        (dict(faces=P(outs["vertex_ids"]) + 8), "maps[0].vertex_ids overlaps maps[0].faces"),
        (dict(m1=dict(confidences=P(dms[0]) + 64, cap_vertices=10)), "maps[1].confidences overlaps maps[0].depth_dev"),
        (dict(color_dev=P(dms[0]), color_channels=7), "maps[0].color_channels is 7, must be 1 to 4"),
        (dict(height=1), "maps[0].height is 1, must be at least 2"),
    ]
    for mods, msg in cases:
        arr = _meshes(dms, ips)
        for k, t in outs.items():
            setattr(arr[0], k, P(t))
        arr[0].cap_vertices, arr[0].cap_faces = nv, nf
        for k, v in mods.items():
            if k == "m1":
                for k1, v1 in v.items():
                    setattr(arr[1], k1, v1)
            else:
                setattr(arr[0], k, v)
        assert _run(arr) == (INVALID, "%s: %s" % (FN, msg))
        assert [(m.n_vertices, m.n_faces) for m in arr] == [(0, 0)] * 3
        torch.cuda.synchronize()
        assert [_bytes(b) for b in bufs] + [host.tobytes()] == before, msg
    assert _run(_meshes(dms, ips), iters=-1) == (INVALID, "%s: conf_iterations is -1: Invalid amount of iterations" % FN)
    # the Python layer refuses what is not a contiguous float32 CUDA tensor, or a colour image of another size
    from mve_b200 import depthmap as D
    for bad in (dms[0].double(), dms[0].t(), dms[0].cpu()):
        with pytest.raises(ValueError):
            D.depthmap_pointset_maps([dms[1], bad], ips[:2])
    with pytest.raises(ValueError):
        D.depthmap_triangulate_maps([dms[0]], [ips[0]], [torch.zeros((3, 3, 3), dtype=torch.uint8, device="cuda")])


# ---------------------------------------------------------------- 5. stream order and memory
def test_ordered_after_the_callers_stream(three):
    from mve_b200 import depthmap as D
    torch = _torch()
    srcs, ips, want = three
    dms = [torch.zeros_like(s) for s in srcs]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                                # ~0.1 s of device time before the maps are produced
        for d, s in zip(dms, srcs):
            d.copy_(s)
        got = D.depthmap_pointset_maps(dms, ips, with_normals=True, conf_iterations=4, scale_factor=2.5)
        for d in dms:
            d.fill_(0.0)
    torch.cuda.synchronize()
    for j, (g, w) in enumerate(zip(got, want)):
        _same(g, w, j)


def test_no_device_memory_retained(three):
    from mve_b200 import depthmap as D
    torch = _torch()
    dms, ips, _ = three
    big = [_sparse(2048, 2048, seed=j, keep=0.01) for j in range(3)]
    arrays = list(dms) + big
    ipl = list(ips) + [_ip(2048, 2048)] * 3
    got = D.depthmap_pointset_maps(arrays, ipl, with_normals=True, conf_iterations=4, scale_factor=2.5)
    arr = _meshes(arrays, ipl)
    for m, g in zip(arr, got):
        for k in KEYS:
            if g.get(k) is not None:
                setattr(m, k, g[k].data_ptr())
        m.cap_vertices, m.cap_faces = len(g["vertices"]), len(g["faces"])
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    assert _run(arr)[0] == 0
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] == free0
    # and once more without the caller's vertex ids and vertices: the workspace holds them during the call
    for m in arr:
        m.vertex_ids = m.vertices = None
    assert _run(arr)[0] == 0
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
