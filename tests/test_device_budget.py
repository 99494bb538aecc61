"""Device budget planning on the CPU: b200mvs_working_set against a restatement of the byte formula, b200mvs_plan_batches'
grouping rule, and the single accounted allocator.  Planning contexts (B200MVS_DEVICE_NONE) only: cameras and features."""
import os
import re

import numpy as np
import pytest

from tests.util import ROOT, golden_scene

ENTRY, PATCH_OUT, JOB_PARAMS = 32, 40, 232          # sizeof(Entry), sizeof(PatchOut), sizeof(JobParams)
C_NUM, HIST_PER_JOB, MAP_PER_PX = 8, 8192 + 64, 40


def _levels(w, h):
    out = [(w, h)]
    while min(w, h) >= 30:                               # buildPyramid (image_pyramid.cc:22-53)
        w, h = (w + 1) // 2, (h + 1) // 2
        out.append((w, h))
    return out


def _pyramid_bytes(w, h):
    return sum(((lw + 3) & ~3) * lh for lw, lh in _levels(w, h)) * 20      # RGBX8 + 2x2 quad per texel, pitch of 4


def _formula(s, refs, sel, n_features, thresholded=False):
    views = set(refs)
    for r in refs:
        views |= set(sel[r])
    lw, lh = _levels(s.width, s.height)[s.scale]
    px = len(refs) * lw * lh
    tiles = len(refs) * ((lw + 15) // 16) * ((lh + 15) // 16)
    assert n_features <= max(2 * px, 1 << 16)           # at most one seed per feature: the seed term cannot decide the capacity
    cap = max(2 * px, 1 << 16)
    per_job = 8 + JOB_PARAMS + 4 + 4 + 8 + (HIST_PER_JOB * 4 if thresholded else 0)
    return (len(views) * _pyramid_bytes(s.width, s.height) + px * MAP_PER_PX + 2048 + cap * (4 * ENTRY + PATCH_OUT + 1)
            + tiles * 12 + C_NUM * 8 + len(refs) * per_job)


def _planning(s):
    from mve_b200 import dmrecon
    sc = dmrecon.Scene(s.n_views, device=-1)
    for v in range(s.n_views):
        sc.set_view_camera(v, s.width, s.height, s.flen[v], s.paspect[v], s.ppoint[v], s.rot[v], s.trans[v])
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


def _settings(s, **kw):
    from mve_b200 import dmrecon
    return dmrecon.Settings(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors, **kw)


@pytest.mark.parametrize("name", ["T0", "T3", "T4", "C2", "C5"])
def test_working_set_matches_formula(name):
    s, sc = _scene(name)
    st = _settings(s)
    sel = {v: sc.global_view_selection(st, v) for v in range(s.n_views)}
    if name == "T3":
        assert all(len(sel[v]) == 20 for v in range(s.n_views))
    nf = len(s.feat_refs)
    for refs in ([0], [s.n_views - 1], list(range(min(s.n_views, 8))), list(range(s.n_views))):
        assert sc.working_set(st, refs) == _formula(s, refs, sel, nf), refs
    if name == "T0":
        lw, lh = _levels(s.width, s.height)[s.scale]
        assert 2 * lw * lh < 1 << 16                    # one view: the frontier floor of 64 Ki entries
        st_t = _settings(s, frontier_topk=64)
        assert sc.working_set(st_t, [0, 1]) == _formula(s, [0, 1], sel, nf, thresholded=True)


def _check_plan(sc, st, refs, available):
    n, groups = sc.plan_batches(st, refs, available)
    assert n >= 1 and sorted(set(groups.tolist())) == list(range(n))          # every view in exactly one group
    for g in range(n):
        assert sc.working_set(st, [r for r, gg in zip(refs, groups) if gg == g]) <= available
    n2, groups2 = sc.plan_batches(st, refs, available)
    assert n2 == n and (groups2 == groups).all()                                  # deterministic
    return n, groups


@pytest.mark.parametrize("name", ["T0", "T1", "T2", "T4", "C2"])
def test_plan_batches(name):
    from mve_b200 import dmrecon
    s, sc = _scene(name)
    st = _settings(s)
    refs = list(range(s.n_views))
    total = sc.working_set(st, refs)
    single = [sc.working_set(st, [r]) for r in refs]
    assert _check_plan(sc, st, refs, total)[0] == 1
    assert _check_plan(sc, st, refs, total * 10)[0] == 1
    n, groups = _check_plan(sc, st, refs, max(single))
    assert n == len(refs)
    for frac in (0.8, 0.6, 0.4):
        _check_plan(sc, st, refs, max(max(single), int(total * frac)))
    with pytest.raises(dmrecon.B200MVSError) as e:
        sc.plan_batches(st, refs, max(single) - 1)
    assert e.value.code == dmrecon.ERR_NO_MEMORY
    assert e.value.failed_view == refs[int(np.argmax(single))]      # the first view, in order, that does not fit alone


def test_plan_batches_prefers_shared_pyramids():
    """A group takes next the view that adds the fewest new pyramid bytes; the caller's order only opens groups."""
    s, sc = _scene("T2")
    st = _settings(s)
    refs = list(range(s.n_views))
    sel = {v: set(sc.global_view_selection(st, v)) | {v} for v in refs}
    avail = max(sc.working_set(st, [r]) for r in refs) + 1
    while True:
        n, groups = sc.plan_batches(st, refs, avail)
        if n < len(refs):
            break
        avail = int(avail * 1.05)
    members = [r for r, g in zip(refs, groups) if g == 0]
    assert members[0] == 0
    second = min((r for r in refs if r != 0 and sc.working_set(st, [0, r]) <= avail),
                 key=lambda r: (len(sel[r] - sel[0]), r))
    assert second in members


def _source():
    src = open(os.path.join(ROOT, "mve_b200", "csrc", "b200mvs.cu")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _span(src, head):
    """Where the definition that starts with `head` (a pattern ending at its opening brace) begins and ends."""
    m = re.search(head, src)
    assert m, head
    depth, i = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(src[i], 0)
        i += 1
    return m.start(), i


def _only_in(src, call, heads):
    """The positions of `call`, after checking that there is one and that each lies in one of the definitions `heads`."""
    spans = [_span(src, h) for h in heads]
    calls = [m.start() for m in re.finditer(call, src)]
    assert calls, call
    assert all(any(a <= c < b for a, b in spans) for c in calls), call
    return calls


def test_cuda_malloc_only_in_the_accounted_allocator():
    src = _source()
    calls = _only_in(src, r"\bcuda(Malloc|Free)\s*\(", (r"cudaError_t dev_alloc\([^)]*\)\s*\{", r"void dev_free\([^)]*\)\s*\{"))
    assert len(calls) == 2


def test_context_resources_have_one_owner():
    """Pinned blocks, events and the stream are made only where their owner is (the context, a staging slot) and freed
    only by the owners' deleters; b200mvs_destroy frees nothing by hand, and only the accounted allocator changes the
    resident bytes."""
    src = _source()
    create, destroy = r"int b200mvs_create\([^)]*\)\s*\{", r"void b200mvs_destroy\([^)]*\)\s*\{"
    stage = (r"int next_stage\([^)]*\)\s*\{", r"int upload_host\([^)]*\)\s*\{")
    _only_in(src, r"\bcuda(MallocHost|HostAlloc|FreeHost)\s*\(", (create, *stage, r"struct FreeHost\s*\{"))
    _only_in(src, r"\bcudaEvent(Create\w*|Destroy)\s*\(", (create, *stage, r"struct DestroyEvent\s*\{"))
    _only_in(src, r"\bcudaStream(Create\w*|Destroy)\s*\(", (create, r"struct DestroyStream\s*\{"))
    a, b = _span(src, destroy)
    assert not re.search(r"\b(cuda\w*(Free\w*|Destroy)|dev_free|release\w*)\s*\(", src[a:b]), src[a:b]
    _only_in(src, r"\bmem\.resident\s*[-+]?=(?!=)", [r"%s\([^)]*\)\s*\{" % f for f in
                                                      ("cudaError_t dev_alloc", "cudaError_t dev_charge", "void dev_uncharge", "void dev_free")])
    for gone in ("ev_pool", "get_event", "PlanAllocs", "pinned.clear()"):
        assert gone not in src, gone
