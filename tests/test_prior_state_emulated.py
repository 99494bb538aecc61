"""The state rule of a prior seed (mve_b200/csrc/prior_seed.cuh prior_seed_state, the function k_prior_seeds calls)
compiled by g++ and run on the CPU: the dz and local views it gives equal tests/prior_state_reference.py bit for bit, on
random maps and on the edge cases of the rule."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests.prior_state_reference import prior_state_seeds, seed_state

EMU = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = str(tmp_path_factory.mktemp("prior_emu") / "libprior_emu.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-pthread", "-I" + EMU,
                           os.path.join(EMU, "prior_emu.cc"), "-o", lib])
    L = C.CDLL(lib)
    L.emu_prior_seed_state.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                       C.c_int, C.c_uint, C.c_void_p, C.c_void_p]
    return L


def _run(L, dz, ids, w, h, W, H, gview, N):
    """The device rule for n candidates: dz n x 2 float32 or None, ids n x 4 int32 or None -> (n x 2 dz, n slot words)."""
    n = len(dz) if dz is not None else len(ids)
    g = np.ascontiguousarray(gview, np.int32)
    out_dz = np.empty((n, 2), np.float32)
    out_slots = np.empty(n, np.uint32)
    dz = None if dz is None else np.ascontiguousarray(dz, np.float32)
    ids = None if ids is None else np.ascontiguousarray(ids, np.int32)
    L.emu_prior_seed_state(n, None if dz is None else dz.ctypes.data, None if ids is None else ids.ctypes.data, w, h, W,
                           H, g.ctypes.data, len(g), N, out_dz.ctypes.data, out_slots.ctypes.data)
    return out_dz, out_slots


def _slot_ids(word, gview):
    """The local view ids of a slot word, None for no local views."""
    if word == 0xFFFFFFFF:
        return None
    out = []
    for k in range(4):
        s = (int(word) >> (8 * k)) & 0xFF
        if s != 0xFF:
            out.append(int(gview[s]))
    return out


def _check(L, dz, ids, w, h, W, H, gview, N):
    got_dz, got_slots = _run(L, dz, ids, w, h, W, H, gview, N)
    n = len(got_slots)
    for i in range(n):
        di, dj, local = seed_state(None if dz is None else dz[i], None if ids is None else ids[i], w, h, W, H, gview, N)
        assert got_dz[i].tobytes() == np.array([di, dj], np.float32).tobytes(), (i, dz[i] if dz is not None else None)
        assert _slot_ids(got_slots[i], gview) == local, (i, ids[i] if ids is not None else None, gview, N)
    return got_slots


@pytest.mark.parametrize("seed", range(6))
def test_random_maps(emu, seed):
    rng = np.random.default_rng(seed)
    n = 4000
    n_views = int(rng.integers(6, 60))
    n_global = int(rng.integers(1, min(n_views, 32) + 1))
    gview = np.sort(rng.choice(n_views, n_global, replace=False)).astype(np.int32)
    dz = rng.normal(0, 0.05, (n, 2)).astype(np.float32)
    ids = rng.integers(-1, n_views, (n, 4)).astype(np.int32)
    w, h = (int(v) for v in rng.integers(1, 2000, 2))
    W, H = (int(v) for v in rng.integers(5, 2000, 2))
    for N in (1, 2, 3, 4):
        _check(emu, dz, ids, w, h, W, H, gview, N)
        _check(emu, dz, None, w, h, W, H, gview, N)
        _check(emu, None, ids, w, h, W, H, gview, N)


def test_non_finite_dz(emu):
    big = np.float32(3e38)
    dz = np.array([[np.nan, 0.1], [0.1, np.nan], [np.inf, 0.0], [0.0, -np.inf], [big, 0.0], [0.0, -big], [big, big],
                   [1e-3, -2e-3], [-0.0, 0.0]], np.float32)
    # ratio 2: 3e38 overflows to inf, so the seed gets (0, 0); ratio 1/3: it stays finite
    for w, h, W, H in ((200, 100, 100, 50), (100, 50, 300, 150), (640, 480, 640, 480)):
        _check(emu, dz, None, w, h, W, H, np.arange(8, dtype=np.int32), 4)
    got, _ = _run(emu, dz, None, 200, 100, 100, 50, np.arange(8, dtype=np.int32), 4)
    assert (got[:7] == 0).all() and got[7].tolist() == [np.float32(2e-3), np.float32(-4e-3)]


def test_id_rule_branches(emu):
    gview = np.array([1, 3, 4, 7, 9, 12], np.int32)
    ids = np.array([
        [3, 4, 7, 9],          # exactly 4 in the selection
        [9, 7, 4, 3],          # unsorted: slots come out ascending
        [3, 3, 4, 7],          # a duplicate: 3 distinct
        [3, 4, 7, 2],          # one outside the selection
        [-1, 3, 4, 7],         # -1 mixed with valid ids
        [-1, -1, -1, -1],      # none
        [3, 4, -1, -1],        # fewer than N
        [1, 3, 4, 12],
        [0, 2, 5, 6],          # none in the selection
        [12, 12, 12, 12],      # one id four times
        [-5, 1, 1, 9],         # a negative id other than -1
    ], np.int32)
    dz = np.zeros((len(ids), 2), np.float32)
    for N in (1, 2, 3, 4):
        slots = _check(emu, dz, ids, 10, 10, 10, 10, gview, N)
        n_valid = [len({i for i in row if i >= 0 and i in set(gview.tolist())}) for row in ids.tolist()]
        assert [s != 0xFFFFFFFF for s in slots] == [v == N for v in n_valid]
    # N = 3 with the maps of an N = 4 run: four valid ids are more than N, so that seed runs the full selection
    _, slots = _run(emu, None, ids[:1], 10, 10, 10, 10, gview, 3)
    assert slots[0] == 0xFFFFFFFF
    _, slots = _run(emu, None, ids[2:3], 10, 10, 10, 10, gview, 3)
    assert _slot_ids(slots[0], gview) == [3, 4, 7]


def test_full_selection_and_reference_seeds(emu):
    """32 global views (every slot bit) and the seeds of a whole entry, as prior_state_seeds states them."""
    rng = np.random.default_rng(11)
    gview = np.sort(rng.choice(100, 32, replace=False)).astype(np.int32)
    ids = rng.choice(np.concatenate([gview, [-1, 100, 101]]), (40, 4)).astype(np.int32)
    ids[:4] = gview[[0, 31, 15, 16]]
    _check(emu, None, ids, 7, 5, 21, 15, gview, 4)
    h, w, W, H, stride = 17, 23, 61, 45, 3
    depth = rng.uniform(1, 2, (h, w)).astype(np.float32)
    dz = rng.normal(0, 0.1, (h, w, 2)).astype(np.float32)
    pid = rng.choice(np.concatenate([gview[:6], [-1]]), (h, w, 4)).astype(np.int32)
    seeds = prior_state_seeds(W, H, depth, stride, gview, 2, dz, pid)
    assert seeds
    py = np.array([(2 * y + 1) * h // (2 * H) for _, y, *_ in seeds])
    px = np.array([(2 * x + 1) * w // (2 * W) for x, _, *_ in seeds])
    got_dz, got_slots = _run(emu, dz[py, px], pid[py, px], w, h, W, H, gview, 2)
    for q, gd, gs in zip(seeds, got_dz, got_slots):
        assert gd.tolist() == [q[3], q[4]] and _slot_ids(gs, gview) == q[5]
