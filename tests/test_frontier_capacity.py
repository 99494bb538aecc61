"""The frontier capacity setting on the CPU (planning contexts): b200mvs_working_set and b200mvs_plan_batches size the
frontier with max(ceil(entries_per_px * pixels), seeds, min_entries) entries, the default reproduces the fixed capacity
of earlier releases, and bad arguments are rejected."""
import math

import pytest

from tests.test_device_budget import _formula, _levels, _scene, _settings

FRONTIER_BYTES = 4 * 32 + 40 + 1                         # two queues, run list, grouped run list, result, written flag


def _px(s, refs):
    lw, lh = _levels(s.width, s.height)[s.scale]
    return len(refs) * lw * lh


def _seeds(sc, st, refs):
    """Seeds of a batch: with no per-pixel term and a floor of one entry the capacity is the seed count."""
    sc.set_frontier_capacity(0.0, 1)
    small = sc.working_set(st, refs)
    sc.set_frontier_capacity(0.0, 1 << 30)
    big = sc.working_set(st, refs)
    sc.set_frontier_capacity()
    assert (big - small) % FRONTIER_BYTES == 0
    return (1 << 30) - (big - small) // FRONTIER_BYTES


@pytest.mark.parametrize("name", ["T0", "T3", "C2", "C5"])
def test_working_set_matches_formula(name):
    s, sc = _scene(name)
    st = _settings(s)
    sel = {v: sc.global_view_selection(st, v) for v in range(s.n_views)}
    nf = len(s.feat_refs)
    default_cap = lambda refs: max(2 * _px(s, refs), 1 << 16)
    for refs in ([0], [s.n_views - 1], list(range(min(s.n_views, 8))), list(range(s.n_views))):
        seeds = _seeds(sc, st, refs)
        assert 0 < seeds <= nf * len(refs)
        base = _formula(s, refs, sel, nf) - default_cap(refs) * FRONTIER_BYTES
        for f, floor in ((2.0, 1 << 16), (1.0, 1 << 16), (0.5, 4096), (0.25, 1), (0.1, 1 << 12), (0.013, 1), (0.0, 7), (3.0, 0)):
            sc.set_frontier_capacity(f, floor)
            cap = max(math.ceil(f * _px(s, refs)), seeds, floor)
            assert sc.working_set(st, refs) == base + cap * FRONTIER_BYTES, (refs, f, floor)
        sc.set_frontier_capacity()


@pytest.mark.parametrize("name", ["T0", "T4", "C2"])
def test_default_is_the_fixed_capacity(name):
    """A fresh context, the default arguments and (2.0, 65536) all give the byte formula of the fixed capacity."""
    s, sc = _scene(name)
    st = _settings(s)
    sel = {v: sc.global_view_selection(st, v) for v in range(s.n_views)}
    refs = list(range(s.n_views))
    want = _formula(s, refs, sel, len(s.feat_refs))
    assert sc.working_set(st, refs) == want
    sc.set_frontier_capacity(0.5, 1)
    assert sc.working_set(st, refs) < want
    sc.set_frontier_capacity(2.0, 65536)
    assert sc.working_set(st, refs) == want
    avail = max(want // 2, max(sc.working_set(st, [r]) for r in refs))
    n_default = sc.plan_batches(st, refs, avail)
    sc.set_frontier_capacity(0.5, 1)
    sc.set_frontier_capacity()
    n_again = sc.plan_batches(st, refs, avail)
    assert n_again[0] == n_default[0] and (n_again[1] == n_default[1]).all()


def test_c4_fewer_groups_with_a_smaller_capacity():
    """C4 (32 views of 4096 x 3072) within 16 GiB: half an entry per pixel plans fewer launches than the default."""
    s, sc = _scene("C4")
    st = _settings(s)
    refs = list(range(s.n_views))
    avail = (16 << 30) - sc.memory_stats().fixed
    n_default, _ = sc.plan_batches(st, refs, avail)
    sc.set_frontier_capacity(0.5, 1 << 16)
    n_half, groups = sc.plan_batches(st, refs, avail)
    for g in range(n_half):
        assert sc.working_set(st, [r for r, gg in zip(refs, groups) if gg == g]) <= avail
    sc.set_frontier_capacity()
    assert n_half < n_default, (n_half, n_default)


@pytest.mark.parametrize("args", [(-0.5, 65536), (float("nan"), 65536), (float("inf"), 65536), (65.0, 65536),
                                  (0.0, 0), (2.0, (1 << 40) + 1), (2.0, -1)])
def test_bad_arguments_rejected(args):
    from mve_b200 import dmrecon
    s, sc = _scene("T0")
    st = _settings(s)
    before = sc.working_set(st, [0])
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.set_frontier_capacity(*args)
    assert e.value.code == dmrecon.ERR_INVALID_ARG
    assert sc.working_set(st, [0]) == before                       # a rejected setting changes nothing


def test_frontier_info_before_any_call():
    s, sc = _scene("T0")
    assert sc.frontier_info() == dict(initial=0, final=0, resumes=0)
