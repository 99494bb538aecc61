"""depthmap_confidence_clean and depthmap_cleanup on batches of maps in device memory (-m gpu):
b200mvs_depthmap_confidence_clean_device / b200mvs_depthmap_cleanup_device through depthmap_confidence_clean_maps and
depthmap_cleanup_maps.

Every output is byte for byte the host entry points' (and, where fixtures exist, the reference's, by SHA-256): the edge
maps of test_gpu_depthmap_edges.cleanup_cases in one call per threshold rank with a threshold per map, the golden, ragged
and large maps of depthmap_ops_ref.npz, and the maps of a real reconstruction.  Also covered: batches split into chunks
(more than 2^28 pixels, and one map larger than that), rejected calls leaving every buffer untouched, the order after the
caller's stream, and no device memory kept after a call."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from tests import dm_reference as R
from tests.test_gpu_depthmap_edges import cleanup_cases, sha
from tests.util import golden_ref, golden_scene

pytestmark = pytest.mark.gpu
F32 = np.float32
INVALID = -1
OPS_THRES = (1, 7, 50, 2000)


def _torch():
    import torch
    return torch


def _cuda(a):
    return _torch().from_numpy(np.ascontiguousarray(a)).cuda()


def _sha_t(t):
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()


def ops_case(kind, seed=0):
    """The inputs of tests/test_gpu_depthmap_ops.py (depthmap_ops_ref.npz): golden (T0 view 0), ragged and large maps."""
    rng = np.random.default_rng(seed)
    if kind == "golden":
        ref = golden_ref("T0")
        return np.ascontiguousarray(ref["depth_0"], F32), np.ascontiguousarray(ref["conf_0"], F32)
    h, w = (97, 131) if kind == "ragged" else (270, 480)
    yy, xx = np.mgrid[0:h, 0:w].astype(F32)
    d = (5.0 + 0.4 * np.sin(xx / 17.0) + 0.3 * np.cos(yy / 11.0)).astype(F32)
    d[(xx > w * 0.6) & (yy > h * 0.3)] += 1.5
    hole = rng.random((h, w)) < (0.45 if kind == "ragged" else 0.08)
    d[hole] = 0.0
    d[:, :3] = 0.0
    conf = rng.random((h, w)).astype(F32) - 0.2
    return d, conf


@pytest.fixture(scope="module")
def edges():
    return cleanup_cases(), golden_ref("depthmap_edges")


# ---------------------------------------------------------------- 1. edge cases against the reference
@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
def test_edge_cases_batched(edges, in_place):
    from mve_b200 import depthmap as D
    cases, ref = edges
    names = list(cases)
    src = [_cuda(cases[n][0]) for n in names]
    ranks = max(len(cases[n][2]) for n in names)
    for r in range(ranks):
        thres = [cases[n][2][min(r, len(cases[n][2]) - 1)] for n in names]
        dms = [t.clone() for t in src]
        outs = D.depthmap_cleanup_maps(dms, thres, out=dms if in_place else None)
        for n, t, o, d in zip(names, thres, outs, dms):
            assert _sha_t(o) == str(ref["cleanup_%s_%d" % (n, t)]), (n, t)
            if not in_place:
                assert d.cpu().numpy().tobytes() == cases[n][0].tobytes(), n
    dms = [t.clone() for t in src]
    cms = [_cuda(cases[n][1]) for n in names]
    if in_place:
        D.depthmap_confidence_clean_maps(dms, cms)
        got = dms
    else:
        # the single-map form on CUDA tensors: one call per map, the same bytes
        got = []
        for d, c in zip(dms, cms):
            D.depthmap_confidence_clean(d, c)
            got.append(d)
    for n, g in zip(names, got):
        assert _sha_t(g) == str(ref["confclean_%s" % n]), n
        assert g.cpu().numpy().tobytes() == R.confidence_clean(cases[n][0], cases[n][1]).tobytes(), n


def test_single_map_forms_return_cuda_tensors(edges):
    from mve_b200 import depthmap as D
    cases, ref = edges
    d = _cuda(cases["spiral"][0])
    for t in cases["spiral"][2]:
        o = D.depthmap_cleanup(d, t)
        assert o.is_cuda and o.data_ptr() != d.data_ptr() and o.shape == d.shape
        assert _sha_t(o) == str(ref["cleanup_spiral_%d" % t]), t


# ---------------------------------------------------------------- 2. the depthmap_ops goldens
def test_depthmap_ops_goldens_batched():
    from mve_b200 import depthmap as D
    ref = golden_ref("depthmap_ops")
    kinds = ("golden", "ragged", "large")
    inputs = [ops_case(k) for k in kinds]
    dms = [_cuda(d) for d, _ in inputs]
    for t in OPS_THRES:
        outs = D.depthmap_cleanup_maps(dms, t)
        for k, o in zip(kinds, outs):
            assert _sha_t(o) == str(ref["cleanup_%s_%d" % (k, t)]), (k, t)
    # a threshold per map: each map gets its own
    per_map = [OPS_THRES[j] for j in range(3)]
    for k, t, o in zip(kinds, per_map, D.depthmap_cleanup_maps(dms, per_map)):
        assert _sha_t(o) == str(ref["cleanup_%s_%d" % (k, t)]), (k, t)
    got = [d.clone() for d in dms]
    D.depthmap_confidence_clean_maps(got, [_cuda(c) for _, c in inputs])
    for k, g in zip(kinds, got):
        assert _sha_t(g) == str(ref["confclean_%s" % k]), k


# ---------------------------------------------------------------- 3. a real reconstruction
def test_reconstruction_maps():
    from mve_b200 import depthmap as D, dmrecon
    s = golden_scene("T2")
    sc = dmrecon.Scene.from_synth(s)
    try:
        st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
        maps, _ = sc.reconstruct(st, list(range(s.n_views)), want=("depth", "conf"), on_device=True)
    finally:
        sc.close()
    host_d = [m["depth"].cpu().numpy() for m in maps]
    host_c = [m["conf"].cpu().numpy() for m in maps]
    assert len(maps) >= 8 and sum(int((d != 0).sum()) for d in host_d) > 1000
    for d, c in zip(host_d, host_c):
        D.depthmap_confidence_clean(d, c)                               # the host entry point, in place
    dms = [m["depth"] for m in maps]
    D.depthmap_confidence_clean_maps(dms, [m["conf"] for m in maps])
    for j, (g, h) in enumerate(zip(dms, host_d)):
        assert g.cpu().numpy().tobytes() == h.tobytes(), j
    for t in (0, 1, 100, 10 ** 6):
        outs = D.depthmap_cleanup_maps(dms, t)
        for j, (o, h) in enumerate(zip(outs, host_d)):
            assert o.cpu().numpy().tobytes() == D.depthmap_cleanup(h, t).tobytes(), (j, t)
    # in place, the maps of the reconstruction themselves
    D.depthmap_cleanup_maps(dms, 100, out=dms)
    for j, (g, h) in enumerate(zip(dms, host_d)):
        assert g.cpu().numpy().tobytes() == D.depthmap_cleanup(h, 100).tobytes(), j


# ---------------------------------------------------------------- 4. chunks
def _holey(h, w, seed, holes):
    torch = _torch()
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = 1.0 + torch.rand((h, w), generator=g, device="cuda")
    d[torch.rand((h, w), generator=g, device="cuda") < holes] = 0.0
    return d


def test_chunks_equal_one_call_per_map():
    from mve_b200 import depthmap as D
    torch = _torch()
    # five 8192 x 8192 maps: 5 * 2^26 pixels, chunks of four maps and of one (a 2 GiB workspace)
    dms = [_holey(8192, 8192, seed=j, holes=0.3 + 0.05 * j) for j in range(5)]
    thres = [1, 3, 10, 40, 1000]
    batch = D.depthmap_cleanup_maps(dms, thres)
    for j, (d, t) in enumerate(zip(dms, thres)):
        one = D.depthmap_cleanup_maps([d], t)[0]
        assert torch.equal(batch[j].view(torch.int32), one.view(torch.int32)), j
    del batch, one
    # a single map larger than 2^28 pixels is a chunk of its own, against the host entry point
    big = _holey(16384, 16400, seed=9, holes=0.35)
    del dms
    torch.cuda.empty_cache()
    got = D.depthmap_cleanup_maps([big], 7)[0].cpu().numpy()
    want = D.depthmap_cleanup(big.cpu().numpy(), 7)
    assert got.tobytes() == want.tobytes()


# ---------------------------------------------------------------- 5. rejections leave everything untouched
def _lib():
    from mve_b200 import depthmap as D
    return D._lib()


def _raw_cleanup(depth_ptrs, ws, hs, thres, out_ptrs):
    L = _lib()
    n = len(depth_ptrs)
    dp = (C.c_void_p * n)(*depth_ptrs)
    op = (C.c_void_p * n)(*out_ptrs)
    ws, hs, th = np.array(ws, np.int32), np.array(hs, np.int32), np.array(thres, np.int64)
    stream = _torch().cuda.current_stream().cuda_stream
    rc = L.b200mvs_depthmap_cleanup_device(0, n, dp, ws.ctypes.data_as(C.c_void_p), hs.ctypes.data_as(C.c_void_p),
                                           th.ctypes.data_as(C.c_void_p), op, C.c_void_p(stream))
    return rc, L.b200mvs_last_error(None).decode()


def test_rejections_leave_buffers_untouched():
    torch = _torch()
    fn = "b200mvs_depthmap_cleanup_device"
    h, w = 40, 50
    d0, d1 = _holey(h, w, 1, 0.3), _holey(h, w, 2, 0.3)
    o0, o1 = torch.full((h, w), 7.0, device="cuda"), torch.full((h, w), 7.0, device="cuda")
    host = np.full((h, w), 5.0, F32)
    pinned = torch.full((h, w), 6.0).pin_memory()
    shared = torch.full((2 * h * w,), 8.0, device="cuda")
    raw = torch.full((h * w + 4,), 9.0, device="cuda")
    bufs = [d0, d1, o0, o1, pinned, shared, raw]
    before = [_sha_t(b) for b in bufs] + [sha(host)]
    P = lambda t: t.data_ptr()                                             # noqa: E731
    cases = [
        ((P(d0), host.ctypes.data), (w, w), (h, h), (P(o0), P(o1)), "depth_dev[1] is pageable host memory, not device memory"),
        ((P(d0), P(d1)), (w, w), (h, h), (P(o0), P(pinned)), "out_dev[1] is pinned host memory, not device memory"),
        ((P(d0), P(d1)), (w, w), (h, h), (P(raw) + 2, P(o1)), "out_dev[0] is not 4-byte aligned"),
        ((P(d0), P(d1)), (w, w), (h, h), (P(shared), P(shared[h * w // 2:])), "out_dev[0] overlaps out_dev[1]"),
        ((P(d0), P(d1)), (w, 0), (h, h), (P(o0), P(o1)), "widths[1] is 0, must be at least 1"),
        ((P(d0), None), (w, w), (h, h), (P(o0), P(o1)), "depth_dev[1] is NULL"),
    ]
    for dp, ws, hs, op, msg in cases:
        rc, got = _raw_cleanup(dp, ws, hs, (1, 1), op)
        assert (rc, got) == (INVALID, "%s: %s" % (fn, msg))
        torch.cuda.synchronize()
        assert [_sha_t(b) for b in bufs] + [sha(host)] == before, msg
    # the same rejections through confidence_clean: depth is written there
    L = _lib()
    dp = (C.c_void_p * 2)(P(d0), host.ctypes.data)
    cp = (C.c_void_p * 2)(P(o0), P(o1))
    ws, hs = np.array((w, w), np.int32), np.array((h, h), np.int32)
    rc = L.b200mvs_depthmap_confidence_clean_device(0, 2, dp, cp, ws.ctypes.data_as(C.c_void_p), hs.ctypes.data_as(C.c_void_p), None)
    assert (rc, L.b200mvs_last_error(None).decode()) == (
        INVALID, "b200mvs_depthmap_confidence_clean_device: depth_dev[1] is pageable host memory, not device memory")
    torch.cuda.synchronize()
    assert [_sha_t(b) for b in bufs] + [sha(host)] == before
    # the Python layer refuses what is not a contiguous float32 CUDA tensor
    from mve_b200 import depthmap as D
    for bad in (d0.double(), d0.t(), d0.cpu()):
        with pytest.raises(ValueError):
            D.depthmap_cleanup_maps([d0, bad], 1)


# ---------------------------------------------------------------- 6. stream order
def test_ordered_after_the_callers_stream(edges):
    from mve_b200 import depthmap as D
    torch = _torch()
    cases, ref = edges
    names = ("spiral", "comb", "checker", "special")
    srcs = [_cuda(cases[n][0]) for n in names]
    confs = [_cuda(cases[n][1]) for n in names]
    dms = [torch.ones_like(s) for s in srcs]                         # a map of ones: one island that any threshold <= size keeps
    outs = [torch.full_like(s, 3.0) for s in srcs]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                                # ~0.1 s of device time before the maps are produced
        for d, s in zip(dms, srcs):
            d.copy_(s)
        D.depthmap_cleanup_maps(dms, 2, out=outs)
        got = [o.cpu().numpy() for o in outs]
        for d in dms:
            d.fill_(1.0)
        torch.cuda._sleep(200_000_000)
        for d, s in zip(dms, srcs):
            d.copy_(s)
        D.depthmap_confidence_clean_maps(dms, confs)
        cc = [d.cpu().numpy() for d in dms]
    for n, g, c in zip(names, got, cc):
        assert sha(g) == str(ref["cleanup_%s_2" % n]), n
        assert sha(c) == str(ref["confclean_%s" % n]), n


# ---------------------------------------------------------------- 7. no memory retained
def test_no_device_memory_retained():
    from mve_b200 import depthmap as D
    torch = _torch()
    dms = [_holey(1024, 2048, j, 0.3) for j in range(4)]
    cms = [_holey(1024, 2048, 10 + j, 0.5) - 1.0 for j in range(4)]
    outs = [torch.empty_like(d) for d in dms]
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    D.depthmap_cleanup_maps(dms, 50, out=outs)
    D.depthmap_confidence_clean_maps(dms, cms)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] == free0
