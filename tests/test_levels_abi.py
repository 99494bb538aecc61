"""Per-entry pyramid levels on the CPU: b200mvs_working_set_levels against a restatement of the byte formula with one level
per entry, b200mvs_plan_batches_levels against a restatement of its greedy rule, equality with the single-level calls at
uniform levels, and the argument errors of the *_levels entry points.  Planning contexts (B200MVS_DEVICE_NONE) only."""
import ctypes as C
import math

import numpy as np
import pytest

from tests.util import golden_scene

ENTRY, PATCH_OUT, JOB_PARAMS = 32, 40, 232          # sizeof(Entry), sizeof(PatchOut), sizeof(JobParams)
C_NUM, MAP_PER_PX = 8, 40


def _levels(w, h):
    out = [(w, h)]
    while min(w, h) >= 30:                               # buildPyramid (image_pyramid.cc:22-53)
        w, h = (w + 1) // 2, (h + 1) // 2
        out.append((w, h))
    return out


def _pyramid_bytes(w, h):
    return sum(((lw + 3) & ~3) * lh for lw, lh in _levels(w, h)) * 20      # RGBX8 + 2x2 quad per texel, pitch of 4


def _max_pixels_level(w, h, max_pixels):
    """apps/dmrecon get_scale_from_max_pixels (dmrecon.cc:89-111)."""
    if w * h <= max_pixels:
        return 0
    ratio = np.float32(w * h) / np.float32(max_pixels)
    return max(0, int(math.ceil(math.log(ratio) / math.log(4.0))))


def _formula(s, entries, sel, n_features):
    """Device bytes of one launch of `entries` ((view, level) pairs): each view's pyramid once, then per entry its maps,
    tiles and per-view arrays at its level, and the frontier arrays for all of them."""
    views = set()
    for r, l in entries:
        views |= {r} | set(sel[(r, l)])
    px = tiles = 0
    for r, l in entries:
        lw, lh = _levels(*s.size(r))[l]
        px += lw * lh
        tiles += ((lw + 15) // 16) * ((lh + 15) // 16)
    assert n_features <= max(2 * px, 1 << 16)           # at most one seed per feature: the seed term cannot decide the capacity
    cap = max(2 * px, 1 << 16)
    per_job = 8 + JOB_PARAMS + 4 + 4 + 8
    return (sum(_pyramid_bytes(*s.size(v)) for v in views) + px * MAP_PER_PX + 2048 + cap * (4 * ENTRY + PATCH_OUT + 1)
            + tiles * 12 + C_NUM * 8 + len(entries) * per_job)


def _planning(s):
    from mve_b200 import dmrecon
    sc = dmrecon.Scene(s.n_views, device=-1)
    for v in range(s.n_views):
        sc.set_view_camera(v, *s.size(v), s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
    sc.set_features(s.feat_pos, s.feat_refs)
    return sc


_SCENES = {}


def _scene(name):
    if name not in _SCENES:
        if name.startswith("T"):
            s = golden_scene(name)
        else:
            from mve_b200 import synth
            s = synth.make_scene(name, only_views=[])
        _SCENES[name] = (s, _planning(s))
    return _SCENES[name]


def _settings(s, scale=None):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale if scale is None else scale, nr_recon_neighbors=s.nr_recon_neighbors)


def _entries(name, s):
    """The (views, levels) of a mixed call on each scene: T6 at the levels --max-pixels=10000 gives (1 for the 179x180
    views, 0 for the 118x58 and 58x118 ones), T0 and C2 with every view at two levels, interleaved."""
    if name == "T6":
        views = list(range(s.n_views))
        return views, [_max_pixels_level(*s.size(v), 10000) for v in views]
    lo = {"T0": 0, "C2": 1}[name]
    views = [v for v in range(s.n_views) for _ in (0, 1)]
    return views, [lo + (k % 2) for k in range(len(views))]


def _selections(s, sc, views, levels):
    return {(v, l): sc.global_view_selection(_settings(s, l), v) for v, l in set(zip(views, levels))}


@pytest.mark.parametrize("name", ["T6", "T0", "C2"])
def test_working_set_levels_matches_formula(name):
    s, sc = _scene(name)
    views, levels = _entries(name, s)
    if name == "T6":
        assert sorted(set(zip((s.size(v) for v in views), levels))) == [((58, 118), 0), ((118, 58), 0), ((179, 180), 1)]
    sel = _selections(s, sc, views, levels)
    nf = len(s.feat_refs)
    st = _settings(s, scale=-7)                         # s->scale is not read by the *_levels calls
    for k in (1, 2, 5, len(views)):
        ent = list(zip(views[:k], levels[:k]))
        assert sc.working_set(st, views[:k], scales=levels[:k]) == _formula(s, ent, sel, nf), ent
    # a view at two levels counts its pyramid once
    v = views[0]
    two = sc.working_set(st, [v, v], scales=[0, 1])
    assert two == _formula(s, [(v, 0), (v, 1)], sel | _selections(s, sc, [v, v], [0, 1]), nf)
    one_each = sc.working_set(st, [v], scales=[0]) + sc.working_set(st, [v], scales=[1])
    assert two < one_each


@pytest.mark.parametrize("name", ["T0", "T2", "T6", "C2"])
def test_uniform_levels_are_the_single_level_calls(name):
    s, sc = _scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    uniform = [s.scale] * len(refs)
    assert sc.working_set(st, refs, scales=uniform) == sc.working_set(st, refs)
    assert sc.working_set(st, refs[:3], scales=uniform[:3]) == sc.working_set(st, refs[:3])
    single = max(sc.working_set(st, [r]) for r in refs)
    total = sc.working_set(st, refs)
    for avail in (total, single, max(single, total // 2), max(single, int(total * 0.7))):
        n1, g1 = sc.plan_batches(st, refs, avail)
        n2, g2 = sc.plan_batches(st, refs, avail, scales=uniform)
        assert n1 == n2 and (g1 == g2).all(), avail


def _greedy(s, entries, sel, available, nf):
    """b200mvs_plan_batches' rule (include/b200mvs.h) over entries: a group opens with the first unassigned entry, then
    repeatedly takes the unassigned entry that fits and adds the fewest new pyramid bytes (ties: lowest index)."""
    group = [-1] * len(entries)
    n = 0

    def need(e):
        return {e[0]} | set(sel[e])

    for first in range(len(entries)):
        if group[first] >= 0:
            continue
        members = [entries[first]]
        assert _formula(s, members, sel, nf) <= available
        group[first] = n
        while True:
            have = set().union(*(need(e) for e in members))
            best, best_add = -1, 0
            for j in range(first + 1, len(entries)):
                if group[j] >= 0:
                    continue
                add = sum(_pyramid_bytes(*s.size(v)) for v in need(entries[j]) - have)
                if best >= 0 and add >= best_add:
                    continue
                if _formula(s, members + [entries[j]], sel, nf) <= available:
                    best, best_add = j, add
            if best < 0:
                break
            group[best] = n
            members.append(entries[best])
        n += 1
    return n, group


@pytest.mark.parametrize("name", ["T6", "T0", "C2"])
def test_plan_batches_levels_follows_the_greedy_rule(name):
    s, sc = _scene(name)
    views, levels = _entries(name, s)
    sel = _selections(s, sc, views, levels)
    nf = len(s.feat_refs)
    entries = list(zip(views, levels))
    st = _settings(s)
    single = [sc.working_set(st, [v], scales=[l]) for v, l in entries]
    total = sc.working_set(st, views, scales=levels)
    for avail in (total, max(single), max(max(single), total // 2), max(max(single), int(total * 0.3))):
        n, groups = sc.plan_batches(st, views, avail, scales=levels)
        assert (n, groups.tolist()) == _greedy(s, entries, sel, avail, nf), avail
        for g in range(n):
            idx = [j for j in range(len(entries)) if groups[j] == g]
            assert sc.working_set(st, [views[j] for j in idx], scales=[levels[j] for j in idx]) <= avail
    from mve_b200 import dmrecon
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.plan_batches(st, views, max(single) - 1, scales=levels)
    assert e.value.code == dmrecon.ERR_NO_MEMORY
    assert e.value.failed_view == views[int(np.argmax(single))]


def _lib():
    from mve_b200 import dmrecon
    return dmrecon.lib()


def _message():
    return _lib().b200mvs_last_error(None).decode()


def _raw_plan(sc, st, refs, levels):
    """b200mvs_plan_batches_levels with the level array as given (None = NULL): (rc, message, failed view)."""
    r = np.asarray(refs, np.int32)
    lv = None if levels is None else np.asarray(levels, np.int32)
    groups = np.zeros(len(r), np.int32)
    failed = C.c_int32(-99)
    rc = _lib().b200mvs_plan_batches_levels(sc._h, C.byref(st), len(r), r.ctypes.data_as(C.c_void_p),
                                            None if lv is None else lv.ctypes.data_as(C.c_void_p), 1 << 40,
                                            groups.ctypes.data_as(C.c_void_p), C.byref(failed))
    return rc, _message() if rc < 0 else "", failed.value


def test_level_errors():
    from mve_b200 import dmrecon
    s, sc = _scene("T6")
    st = _settings(s)
    refs = list(range(s.n_views))
    ok = sc.working_set(st, refs)
    n_levels = sc.num_levels(3)
    bad = [
        ([0, 3, 5], [0, -1, 0], dmrecon.ERR_INVALID_ARG, "Invalid scale factor", 3),
        ([0, 3, 5], [0, n_levels, 0], dmrecon.ERR_INVALID_ARG, "Invalid scale factor", 3),
        ([0, 3, 5, 3], [0, 1, 0, 1], dmrecon.ERR_INVALID_ARG, "view 3 appears more than once at level 1", 3),
        ([0, 3], None, dmrecon.ERR_INVALID_ARG, "b200mvs_plan_batches_levels: levels is NULL", -1),
    ]
    for refs_b, levels_b, code, msg, failed in bad:
        rc, m, f = _raw_plan(sc, st, refs_b, levels_b)
        assert (rc, m, f) == (code, msg, failed), (refs_b, levels_b)
        assert sc.working_set(st, refs) == ok                        # the context stays usable
    # the other entry points report the same checks with the same codes and messages
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.working_set(st, [0, 3], scales=[0, -1])
    assert (e.value.code, str(e.value).split(": ", 1)[1]) == (dmrecon.ERR_INVALID_ARG, "Invalid scale factor")
    r = np.asarray([0], np.int32)
    out = C.c_uint64()
    assert _lib().b200mvs_working_set_levels(sc._h, C.byref(st), 1, r.ctypes.data_as(C.c_void_p), None, C.byref(out)) == dmrecon.ERR_INVALID_ARG
    assert _message() == "b200mvs_working_set_levels: levels is NULL"
    failed = C.c_int32(-99)
    assert _lib().b200mvs_reconstruct_levels(sc._h, C.byref(st), 1, r.ctypes.data_as(C.c_void_p), None, None, None, None,
                                             C.byref(failed)) == dmrecon.ERR_INVALID_ARG
    assert (_message(), failed.value) == ("b200mvs_reconstruct_levels: levels is NULL", -1)
    # a view may appear at several levels
    assert sc.working_set(st, [3, 3, 0], scales=[0, 1, 0]) > 0
    # the Python forms check the length of scales
    with pytest.raises(ValueError):
        sc.working_set(st, [0, 3], scales=[0])
    with pytest.raises(ValueError):
        sc.plan_batches(st, [0, 3], 1 << 40, scales=[0, 0, 0])
    assert sc.working_set(st, refs) == ok


def test_side_limit_applies_per_entry():
    """The 65535-pixels-per-side limit is checked at each entry's level: level 0 of a 140000 x 60 view is rejected, its
    level 2 (35000 x 15) passes the checks and fails only in planning (the view sees no feature)."""
    from mve_b200 import dmrecon
    sc = dmrecon.Scene(2, device=-1)
    rot = np.eye(3, dtype=np.float32)
    sc.set_view_camera(0, 140000, 60, 1.0, 1.0, (0.5, 0.5), rot, (0, 0, 0))
    sc.set_view_camera(1, 140000, 60, 1.0, 1.0, (0.5, 0.5), rot, (0, 0, 1))
    sc.set_features(np.zeros((1, 3), np.float32), [np.asarray([0, 1], np.int32)])
    st = dmrecon.Settings(scale=0)
    assert sc.num_levels(0) == 3
    rc, m, f = _raw_plan(sc, st, [1, 0], [2, 0])
    assert (rc, m, f) == (-6, "reference level larger than 65535 pixels per side", 0)
    rc, m, f = _raw_plan(sc, st, [1, 0], [2, 2])
    assert (rc, m) == (dmrecon.ERR_GLOBAL_VS, "Global View Selection failed")
