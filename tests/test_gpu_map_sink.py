"""Host and device maps of one batch (-m gpu): Scene.reconstruct and Scene.reconstruct(on_device=True) of T6 under the
same small image-source budget, which splits the batch into groups out of ref_views order.  Each run has a fresh Scene,
so the two routes must agree byte for byte in their maps and exactly in memory_stats, frontier_info and plan_info (its
times aside), and must write the same width and height into every view's b200mvs_maps.  Views cancelled before the call
(one of a group that still runs, and every view of another group) leave their buffers untouched on both routes; the
first still gets its width and height, the others none.  Without maps (download=False) the batch fails: its results
would have to stay on the device, and they do not fit one launch."""
import numpy as np
import pytest

from tests.util import golden_scene

pytestmark = pytest.mark.gpu

MAPS = ("depth", "conf", "dz", "normal", "view_ids")
SENTINEL = -7


class _Recording:
    """The library, keeping the b200mvs_maps array of the last reconstruct call: the widths and heights it wrote."""

    def __init__(self, lib):
        self._lib, self.maps = lib, None

    def __getattr__(self, name):
        f = getattr(self._lib, name)
        if name not in ("b200mvs_reconstruct", "b200mvs_reconstruct_device"):
            return f

        def call(h, settings, n, refs, maps, *rest):
            self.maps = maps
            return f(h, settings, n, refs, maps, *rest)
        return call


@pytest.fixture(scope="module")
def batch():
    """T6 in a permuted order and a budget whose plan makes several groups, out of ref_views order, one of them of
    several views: (scene, settings, refs, budget, group of each ref)."""
    from mve_b200 import dmrecon
    s = golden_scene("T6")
    st = dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    refs = np.random.default_rng(3).permutation(s.n_views).tolist()
    sc = dmrecon.Scene.from_synth(s, lazy=True)
    try:
        fixed = sc.memory_stats().fixed
        single = max(sc.working_set(st, [r]) for r in refs)
        total = sc.working_set(st, refs)
        for avail in np.linspace(single, total, 40).astype(np.int64).tolist():
            n, groups = sc.plan_batches(st, refs, int(avail))
            if n >= 2 and (np.diff(groups) < 0).any() and np.bincount(groups).max() >= 2:
                return s, st, refs, fixed + int(avail), np.asarray(groups)
    finally:
        sc.close()
    raise AssertionError("no budget splits T6 into groups out of order")


def _run(batch, on_device, out=None, progress=None):
    """One reconstruction of the batch on a fresh Scene: host maps, the (width, height) of every view's b200mvs_maps,
    and the memory, frontier and plan figures."""
    from mve_b200 import dmrecon
    s, st, refs, budget, _ = batch
    sc = dmrecon.Scene.from_synth(s, lazy=True, budget_bytes=budget)
    try:
        sc._lib = rec = _Recording(sc._lib)
        maps, _ = sc.reconstruct(st, refs, out=out, progress=progress, on_device=on_device)
        if on_device:
            maps = [{k: t.cpu().numpy() for k, t in d.items()} for d in maps]
        sizes = [(rec.maps[j].width, rec.maps[j].height) for j in range(len(refs))]
        plan = {k: v for k, v in sc.plan_info().items() if not k.startswith("ms_")}
        return maps, sizes, (sc.memory_stats().as_dict(), sc.frontier_info(), plan)
    finally:
        sc.close()


def test_host_and_device_maps_agree(batch):
    import torch
    from mve_b200 import dmrecon
    _, _, refs, budget, groups = batch
    host, h_sizes, h_info = _run(batch, False)
    dev, d_sizes, d_info = _run(batch, True)
    for a, b in zip(host, dev):
        assert sorted(a) == sorted(b) == sorted(MAPS)
        for k in MAPS:
            assert a[k].dtype == b[k].dtype and a[k].tobytes() == b[k].tobytes(), k
    assert h_sizes == d_sizes == [m["depth"].shape[::-1] for m in host]
    assert h_info == d_info
    mem = h_info[0]
    assert mem["n_groups"] == groups.max() + 1 and mem["n_loads"] > 0 and mem["peak"] <= mem["budget"] == budget, mem

    # cancelled before the call: one view of the largest group, and every view of another group
    big = np.bincount(groups).argmax()
    skipped = (big + 1) % (groups.max() + 1)
    cancel = [int(np.flatnonzero(groups == big)[0])] + np.flatnonzero(groups == skipped).tolist()
    infos = []
    for on_device in (False, True):
        progress = (dmrecon.Progress * len(refs))()
        for j in cancel:
            progress[j].cancelled = 1
        out = [{k: np.full(m[k].shape, SENTINEL, m[k].dtype) for k in MAPS} for m in host]
        if on_device:
            out = [{k: torch.from_numpy(a).to("cuda:0") for k, a in d.items()} for d in out]
        got, sizes, info = _run(batch, on_device, out, progress)
        infos.append(info)
        for j in range(len(refs)):
            if j in cancel:
                assert progress[j].status == 5, (on_device, j)
                assert all((got[j][k] == SENTINEL).all() for k in MAPS), (on_device, j)
            else:
                assert progress[j].status == 0, (on_device, j)
                assert all(got[j][k].tobytes() == host[j][k].tobytes() for k in MAPS), (on_device, j)
        want = [(0, 0) if groups[j] == skipped else host[j]["depth"].shape[::-1] for j in range(len(refs))]
        assert sizes == want, on_device
    assert infos[0] == infos[1]


def test_download_false_needs_one_group(batch):
    from mve_b200 import dmrecon
    s, st, refs, budget, groups = batch
    sc = dmrecon.Scene.from_synth(s, lazy=True, budget_bytes=budget)
    try:
        with pytest.raises(dmrecon.B200MVSError) as e:
            sc.reconstruct(st, refs, download=False)
        assert e.value.code == dmrecon.ERR_INVALID_ARG
        assert ("maps == NULL keeps the results on the device, but the budget splits the batch into %d launches"
                % (groups.max() + 1)) in str(e.value)
    finally:
        sc.close()
