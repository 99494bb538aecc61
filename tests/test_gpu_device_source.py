"""The device image source (-m gpu): b200mvs_set_image_source_device through Scene.set_image_source(on_device=True) and
through ctypes callbacks of its own.

A device source must give what a host source gives for the same bytes: every level of every view for 1-4 channels in
packed HWC, pitched HWC and planar CHW, with and without k2/k4 (the host route pinned to tests/golden/undistort_ref.npz);
and on T0, T5 and T6 under a budget that runs several groups (on T6 out of ref_views order) around reads that evict and
fetch views again, the maps, the counters of stats and b200mvs_memory, through host maps, reconstruct(on_device=True)
and reconstruct_pointset(on_device=True).  Also: the library waits for the fetch's stream, release comes once per
successful fetch after the last read (the image may be overwritten in it), descriptors that do not fit are rejected
before anything reads them and leave the context usable, and one context switches between host, device and no source."""
import functools
import os
import re

import numpy as np
import pytest

from tests import undistort_reference as UR
from tests.test_gpu_pset_on_device import host as pset_host
from tests.test_gpu_reconstruct_pointset import F_SET, same
from tests.util import ROOT, golden_scene

pytestmark = pytest.mark.gpu
CAM = dict(paspect=1.0, ppoint=(0.5, 0.5), rot=np.eye(3, dtype=np.float32), trans=np.zeros(3, np.float32))
MAPS = ("depth", "conf", "dz", "normal", "view_ids")
LAYOUTS = ("packed", "pitched", "chw")
COUNTS = ("n_opt", "n_sample_sets", "n_rounds", "n_filled", "n_seeds_processed", "n_seeds_success", "n_entries_peak",
          "n_patch_launches", "n_kernel_launches", "n_grid_barriers")
MEMORY = ("budget", "fixed", "n_groups", "n_loads", "bytes_loaded", "n_evictions", "peak")


def _settings(s):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)


def _as_layout(img, layout, device, seed=0):
    """A uint8 CUDA tensor holding `img` (H x W x C) in `layout`; pitched and planar ones are views into a larger buffer
    whose padding is noise."""
    import torch
    h, w, c = img.shape
    src = torch.from_numpy(np.ascontiguousarray(img)).to(device)
    g = torch.Generator(device="cpu").manual_seed(seed)
    if layout == "packed":
        return src if c > 1 or seed % 2 else src[:, :, 0]          # grey also as H x W
    if layout == "pitched":
        row = w * c + 13
        buf = torch.randint(0, 256, (9 + h * row,), dtype=torch.uint8, generator=g).to(device)
        t = buf.as_strided((h, w, c), (row, c, 1), 9)
    else:
        row, plane = w + 3, (h + 2) * (w + 3) + 5
        buf = torch.randint(0, 256, (7 + c * plane,), dtype=torch.uint8, generator=g).to(device)
        t = buf.as_strided((c, h, w), (plane, row, 1), 7)
        src = src.permute(2, 0, 1)
    t.copy_(src)
    return t


def _levels(sc, v):
    return [sc.level(v, k).tobytes() for k in range(sc.num_levels(v))]


def _rgb(img):
    return np.ascontiguousarray(img[:, :, :3] if img.shape[2] >= 3 else np.repeat(img[:, :, :1], 3, axis=2))


@pytest.mark.parametrize("distorted", [False, True], ids=["plain", "k2k4"])
def test_levels_equal_host_source_in_every_layout(distorted):
    import torch
    from mve_b200 import dmrecon
    golden = np.load(os.path.join(ROOT, "tests", "golden", "undistort_ref.npz"))
    if distorted:
        cases = [c for c in UR.cases() if c[1] * c[2] >= 900 and (c[5], c[6]) != (0.0, 0.0)]
    else:
        cases = [("plain%d" % c, 97 + c, 75, c, 1.0, 0.0, 0.0, 100 + c) for c in (1, 2, 3, 4)]
    assert {c[3] for c in cases} == {1, 2, 3, 4}
    images = [UR.make_image(w, h, c, seed) for _, w, h, c, _, _, _, seed in cases]

    def scene():
        sc = dmrecon.Scene(len(cases))
        for v, (name, w, h, c, flen, k2, k4, seed) in enumerate(cases):
            sc.set_view_camera(v, w, h, flen, **CAM)
            sc.set_view_distortion(v, k2, k4)
        return sc
    ref = scene()
    ref.set_image_source(lambda v: images[v])
    expected = [_levels(ref, v) for v in range(len(cases))]
    for v, case in enumerate(cases):                                    # the host route is the reference's
        want = images[v]
        if distorted:
            want = UR.undistort_k2k4(images[v], case[4], case[5], case[6])
            UR.check(golden, case, want)
        assert expected[v][0] == _rgb(want).tobytes(), case[0]
    ref.close()
    dev = "cuda:0"
    for layout in LAYOUTS:
        tensors = [_as_layout(img, layout, dev, v) for v, img in enumerate(images)]
        sc = scene()
        sc.set_image_source(lambda v: tensors[v], on_device=True, layout="chw" if layout == "chw" else "hwc")
        for v, case in enumerate(cases):
            assert _levels(sc, v) == expected[v], (layout, case[0])
        m = sc.memory_stats()
        assert m.n_loads == len(cases) and m.bytes_loaded == sum(i.size for i in images), m.as_dict()
        sc.close()
    torch.cuda.synchronize()


def _level_sizes(w, h, scale_or_all):
    """(w, h) of every pyramid level, as the library halves them: (w + 1) / 2 while both sides stay >= 1."""
    out = [(w, h)]
    while len(out) <= scale_or_all and min(out[-1]) > 1:
        w, h = (w + 1) // 2, (h + 1) // 2
        out.append((w, h))
    return out


@functools.lru_cache(maxsize=None)
def _budget_scene(name):
    """A golden scene, its reference views, a budget under which they run in several groups, on T6 out of ref_views order
    (in T0 and T5 every view selects all others, so their groups stay in order), with room to spare for the point-set
    workspace of reconstruct_pointset, and a budget that holds two pyramids (reading every view's level 0 evicts)."""
    from mve_b200 import dmrecon
    s = golden_scene(name)
    st = _settings(s)
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    fixed = sc.memory_stats().fixed
    px = max(w * h for w, h in (_level_sizes(*s.size(v), st.scale)[st.scale] for v in range(s.n_views)))
    pyr = max(sum(20 * ((w + 3) & ~3) * h for w, h in _level_sizes(*s.size(v), 64)) for v in range(s.n_views))
    slack = 256 * px + (1 << 20)
    for seed in range(8):
        refs = np.random.default_rng(seed).permutation(s.n_views).tolist()
        single = max(sc.working_set(st, [r]) for r in refs)
        total = sc.working_set(st, refs)
        for avail in np.linspace(single + slack, total, 40).astype(np.int64).tolist():
            plans = [sc.plan_batches(st, refs, int(a)) for a in np.linspace(avail - slack, avail, 9).astype(np.int64)]
            if plans[0][0] >= 2 and all(p[0] == plans[0][0] and (name != "T6" or (np.diff(p[1]) < 0).any()) for p in plans):
                sc.close()
                return s, st, refs, fixed + int(avail), fixed + 2 * pyr + 4096
    sc.close()
    raise AssertionError("no budget gives several groups")


def _run(s, st, refs, budgets, source, mode):
    """On one fresh context with the given source: a reconstruction, every view's level 0 read under the small budget
    (evicting and fetching again), and a second reconstruction, which fetches again what the reads evicted.  Returns (the
    results of both reconstructions, their counters, b200mvs_memory at the end)."""
    import torch
    from mve_b200 import dmrecon
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    dev = "cuda:%d" % sc.device
    if source == "host":
        def install(budget):
            sc.set_image_source(lambda v: s.images[v], budget)
    else:
        held = {v: _as_layout(s.images[v], "chw" if source == "chw" else "pitched", dev, v) for v in range(s.n_views)}

        def install(budget):
            sc.set_image_source(lambda v: held[v], budget, on_device=True, layout="chw" if source == "chw" else "hwc")
    results, counts = [], []
    for step in range(2):
        install(budgets[0])
        if mode == "maps":
            res, stats = sc.reconstruct(st, refs)
        elif mode == "maps_on_device":
            res, stats = sc.reconstruct(st, refs, on_device=True)
            res = [{k: t.cpu().numpy() for k, t in d.items()} for d in res]
        else:
            res, stats = sc.reconstruct_pointset(st, refs, options=F_SET, on_device=True)
            res = pset_host(res)
        results.append(res)
        counts.append({k: getattr(stats, k) for k in COUNTS})
        if step == 0:
            install(budgets[1])
            for v in range(s.n_views):
                sc.level(v, 0)
    torch.cuda.synchronize()
    mem = sc.memory_stats().as_dict()
    sc.close()
    return results, counts, {k: mem[k] for k in MEMORY}


def _same_maps(got, want):
    for d, h in zip(got, want):
        for k in MAPS:
            assert d[k].dtype == h[k].dtype and d[k].tobytes() == h[k].tobytes(), k


@pytest.mark.parametrize("name", ["T0", "T5", "T6"])
@pytest.mark.parametrize("mode", ["maps", "maps_on_device", "pointset_on_device"])
def test_reconstruction_under_budget_equals_host_source(name, mode):
    s, st, refs, *budgets = _budget_scene(name)
    want, counts, mem = _run(s, st, refs, budgets, "host", mode)
    assert mem["n_groups"] >= 2 and mem["peak"] <= budgets[0] and mem["n_loads"] > s.n_views and mem["n_evictions"], mem
    for source in ("hwc", "chw"):
        got, c2, m2 = _run(s, st, refs, budgets, source, mode)
        assert c2 == counts and m2 == mem, (source, c2, counts, m2, mem)
        for g, w in zip(got, want):
            if mode == "pointset_on_device":
                same(g, w)
            else:
                _same_maps(g, w)


def test_waits_for_the_fetch_stream():
    """Each fetch fills its tensor with a sentinel, then, behind a long sleep on the same side stream, copies the image in,
    and returns without synchronising; the pyramid must be built from the image."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T5")
    st = _settings(s)
    refs = list(range(s.n_views))
    want, _ = dmrecon.Scene.from_synth(s).reconstruct(st, refs)
    dev = torch.device("cuda:0")
    images = [torch.from_numpy(s.images[v]).to(dev) for v in range(s.n_views)]
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    fetched = []

    def fetch(v):
        assert torch.cuda.current_stream(dev) == side
        t = torch.full(images[v].shape, 7, dtype=torch.uint8, device=dev)
        torch.cuda._sleep(50_000_000)
        t.copy_(images[v])
        fetched.append(v)
        return t
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    sc.set_image_source(fetch, on_device=True)
    with torch.cuda.stream(side):
        got, _ = sc.reconstruct(st, refs)
    assert sorted(fetched) == refs
    for d, h in zip(got, want):
        for k in MAPS:
            assert d[k].tobytes() == h[k].tobytes(), k
    sc.close()


class RawSource:
    """A device source installed through the C ABI: describe(view) gives the descriptor fields of each fetch; counts
    fetches and releases, and runs on_release(view) in the release callback."""

    def __init__(self, sc, describe, budget=0, on_release=None, counts_of=None):
        from mve_b200 import dmrecon
        self.fetches, self.releases = (counts_of.fetches, counts_of.releases) if counts_of else ([], [])

        def _fetch(_user, view_id, out):
            d = describe(int(view_id))
            if d is None:
                return 1
            o = out.contents
            o.data, o.w, o.h, o.channels, o.row_pitch, o.plane_pitch, o.cuda_stream = d
            self.fetches.append(int(view_id))
            return 0

        def _release(_user, view_id):
            self.releases.append(int(view_id))
            if on_release:
                on_release(int(view_id))
        self.cbs = (dmrecon._DEVICE_FETCH_FN(_fetch), dmrecon._RELEASE_FN(_release))
        assert sc._lib.b200mvs_set_image_source_device(sc._h, self.cbs[0], self.cbs[1], None, int(budget)) == 0


def test_release_once_per_fetch_after_the_last_read():
    """release overwrites the image; the maps must not change, and every successful fetch is released exactly once."""
    import torch
    from mve_b200 import dmrecon
    s, st, refs, budget, small = _budget_scene("T6")
    want, _, mem = _run(s, st, refs, (budget, small), "host", "maps")
    dev = torch.device("cuda:0")
    held = {}

    def describe(v):
        t = torch.from_numpy(s.images[v]).to(dev)
        held[v] = t
        h, w, c = t.shape
        return t.data_ptr(), w, h, c, w * c, 0, None

    def overwrite(v):
        held.pop(v).fill_(0)
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    for step, w in enumerate(want):
        src = RawSource(sc, describe, budget, overwrite, src if step else None)
        _same_maps(sc.reconstruct(st, refs)[0], w)
        if step == 0:
            src = RawSource(sc, describe, small, overwrite, src)
            for v in range(s.n_views):
                sc.level(v, 0)
    assert len(src.fetches) == mem["n_loads"] > s.n_views and sorted(src.releases) == sorted(src.fetches) and not held
    assert sc.memory_stats().n_loads == mem["n_loads"] and sc.memory_stats().n_evictions == mem["n_evictions"]
    # one release per fetch also for levels read one at a time
    n = len(src.fetches)
    src = RawSource(sc, describe, small, overwrite, src)
    for v in range(s.n_views):
        sc.level(v, 0)
    assert len(src.releases) == len(src.fetches) > n and not held
    sc.close()


def test_rejected_descriptors_leave_the_context_usable():
    """Host memory (numpy and pinned), row and plane pitches that are too small, and 0 or 5 channels: each fails the call
    with B200MVS_ERR_INVALID_ARG naming the view, before anything reads the image; the fetch is released, and the same
    context then reconstructs correctly."""
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    st = _settings(s)
    ref = 0
    want, _ = dmrecon.Scene.from_synth(s).reconstruct(st, [ref])
    dev = torch.device("cuda:0")
    h, w, c = s.images[0].shape
    good = {v: torch.from_numpy(s.images[v]).to(dev) for v in range(s.n_views)}
    host_np = np.ascontiguousarray(s.images[0])
    pinned = torch.from_numpy(s.images[0]).pin_memory()
    planar = torch.zeros(c * h * w, dtype=torch.uint8, device=dev)
    bad = {
        "numpy": ((host_np.ctypes.data, w, h, c, w * c, 0), r"data is pageable host memory"),
        "pinned": ((pinned.data_ptr(), w, h, c, w * c, 0), r"data is pinned host memory"),
        "row": ((good[0].data_ptr(), w, h, c, w * c - 1, 0), r"row_pitch must be at least %d" % (w * c)),
        "row_planar": ((planar.data_ptr(), w, h, c, w - 1, h * w), r"row_pitch must be at least %d" % w),
        "plane": ((planar.data_ptr(), w, h, c, w, h * w - 1), r"planes overlap"),
        "negative": ((good[0].data_ptr(), w, h, c, w * c, -1), r"plane_pitch not negative"),
        "ch0": ((good[0].data_ptr(), w, h, 0, w * c, 0), r"is %dx%dx0, registered as %dx%d" % (w, h, w, h)),
        "ch5": ((good[0].data_ptr(), w, h, 5, w * 5, 0), r"is %dx%dx5, registered as %dx%d" % (w, h, w, h)),
        "size": ((good[0].data_ptr(), w - 1, h, c, w * c, 0), r"registered as %dx%d" % (w, h)),
    }
    if torch.cuda.device_count() > 1:
        other = torch.from_numpy(s.images[0]).to("cuda:1")
        bad["other_device"] = ((other.data_ptr(), w, h, c, w * c, 0), r"data is memory of device 1, not of device 0")
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    for what, (desc, msg) in bad.items():
        src = RawSource(sc, lambda v: desc + (None,))
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.reconstruct(st, [ref])
        assert e.value.code == dmrecon.ERR_INVALID_ARG and e.value.failed_view == ref, (what, str(e.value))
        m = re.search(r"device image of view (\d+) ", str(e.value))
        assert m and re.search(msg, str(e.value)), (what, str(e.value))
        assert src.fetches == src.releases == [int(m.group(1))], what
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.level(3, 0)
        assert e.value.code == dmrecon.ERR_INVALID_ARG and "device image of view 3 " in str(e.value), what
        assert sc.memory_stats().n_loads == 0
    sc.set_image_source(lambda v: good[v], on_device=True)
    got, _ = sc.reconstruct(st, [ref])
    for k in MAPS:
        assert got[0][k].tobytes() == want[0][k].tobytes(), k
    sc.close()


def test_python_wrapper_rejects_unfit_tensors():
    import torch
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    dev = torch.device("cuda:0")
    for fetch, layout, msg in ((lambda v: s.images[v], "hwc", "torch.uint8 tensor"),
                               (lambda v: torch.from_numpy(s.images[v]), "hwc", "torch.uint8 tensor"),
                               (lambda v: torch.from_numpy(s.images[v]).to(dev).float(), "hwc", "torch.uint8 tensor"),
                               (lambda v: torch.from_numpy(s.images[v]).to(dev).permute(2, 0, 1).contiguous().permute(1, 2, 0),
                                "hwc", "channel stride"),
                               (lambda v: torch.from_numpy(s.images[v]).to(dev).permute(2, 0, 1), "chw", "pixel stride")):
        sc.set_image_source(fetch, on_device=True, layout=layout)
        with pytest.raises(ValueError, match=msg):
            sc.level(0, 0)
    with pytest.raises(ValueError, match="layout"):
        sc.set_image_source(lambda v: None, on_device=True, layout="cwh")
    sc.close()


def test_switching_sources_on_one_context():
    """host -> device -> none (images uploaded) -> host on one context under one budget: the maps never change, and each
    source's fetches are counted."""
    import torch
    from mve_b200 import dmrecon
    s, st, refs, budget, small = _budget_scene("T6")
    dev = torch.device("cuda:0")
    planar = {v: torch.from_numpy(s.images[v]).to(dev).permute(2, 0, 1).contiguous() for v in range(s.n_views)}
    device_fetches = []

    def fetch(v):
        device_fetches.append(v)
        return planar[v]
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    sc.set_image_source(lambda v: s.images[v], budget)
    want, _ = sc.reconstruct(st, refs)
    sc.set_image_source(lambda v: s.images[v], small)
    for v in range(s.n_views):                  # leaves only the last views read resident
        sc.level(v, 0)
    n0 = sc.memory_stats().n_loads
    sc.set_image_source(fetch, budget, on_device=True, layout="chw")
    got, _ = sc.reconstruct(st, refs)
    assert device_fetches and sc.memory_stats().n_loads == n0 + len(device_fetches)
    results = [got]
    sc.set_image_source(None)
    assert sc.memory_stats().budget == 0
    for v in range(s.n_views):
        sc.set_view(v, s.images[v], s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    results.append(sc.reconstruct(st, refs)[0])
    n1 = len(device_fetches)
    sc.set_image_source(lambda v: s.images[v], budget)
    results.append(sc.reconstruct(st, refs)[0])
    assert len(device_fetches) == n1
    for got in results:
        for d, h in zip(got, want):
            for k in MAPS:
                assert d[k].tobytes() == h[k].tobytes(), k
    sc.close()
