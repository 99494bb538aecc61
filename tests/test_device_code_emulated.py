"""The product's DEVICE code on the CPU.  The two patch-optimisation implementations - mve_b200/csrc/patch_warp.cuh (one
warp per patch, mode 1) and patch_thread.cuh (one thread per patch, mode 2), with the state machine they share in
patch_opt.cuh - are compiled by g++ against a small SIMT emulation (tests/emu/simt_emu.h: 32 host threads per warp,
collectives through a barrier) and run on the oracle's execution trace.  This checks the kernels' LOGIC - pass state
machine, lane-distributed arrays, batched reductions, local view selection and view replacement - without a GPU;
last-bit numerics differ from the GPU (exact reciprocals, libm).  Inputs (pyramid bytes, calibrations) come from the
oracle, which is bit-exact with the product's pyramid kernels (tests/test_gpu_parity.py::test_pyramid_bit_exact)."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle_py as O
from tests.emu import build as emu_build
from tests.util import golden_ref, golden_scene, patch_compare

MAX_LEVELS = 12
EMU_VIEW = np.dtype([("campos", "<f4", (3,)), ("inv_ax0", "<f4"), ("w2c", "<f4", (12,)), ("rot", "<f4", (9,)),
                     ("nlevels", "<i4"), ("ax", "<f4", (MAX_LEVELS,)), ("ay", "<f4", (MAX_LEVELS,)),
                     ("cx", "<f4", (MAX_LEVELS,)), ("cy", "<f4", (MAX_LEVELS,)), ("w", "<i4", (MAX_LEVELS,)),
                     ("h", "<i4", (MAX_LEVELS,)), ("pitch", "<i4", (MAX_LEVELS,)), ("img", "<u8", (MAX_LEVELS,)),
                     ("quad", "<u8", (MAX_LEVELS,))], align=True)
EMU_IN = np.dtype([("x", "<i4"), ("y", "<i4"), ("depth", "<f4"), ("dzI", "<f4"), ("dzJ", "<f4"), ("slots", "<u4")])
EMU_OUT = np.dtype([("conf", "<f4"), ("depth", "<f4"), ("dzI", "<f4"), ("dzJ", "<f4"), ("nx", "<f4"), ("ny", "<f4"),
                    ("nz", "<f4"), ("slots", "<u4"), ("iterations", "<i4"), ("flags", "<i4"), ("sets", "<u4")])


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(emu_build.build())
    v, i, o = C.c_int(), C.c_int(), C.c_int()
    assert lib.emu_struct_sizes(C.byref(v), C.byref(i), C.byref(o)) == MAX_LEVELS
    assert (v.value, i.value, o.value) == (EMU_VIEW.itemsize, EMU_IN.itemsize, EMU_OUT.itemsize)
    return lib


def _lut():
    i = np.arange(256)
    x = i / 255.0
    return np.where(i <= 0.04045 * 255.0, x / 12.92, ((x + 0.055) / 1.055) ** 2.4).astype(np.float32)


def _run(lib, s, osc, ref, gsel, settings, pin, mode=1):
    keep = []          # keeps the RGBX arrays alive
    views = np.zeros(s.n_views, EMU_VIEW)
    for v in range(s.n_views):
        R = s.rot[v].astype(np.float32)
        t = s.trans[v].astype(np.float32)
        views[v]["campos"] = [-R[0] * t[0] - R[3] * t[1] - R[6] * t[2], -R[1] * t[0] - R[4] * t[1] - R[7] * t[2],
                              -R[2] * t[0] - R[5] * t[1] - R[8] * t[2]]
        views[v]["w2c"] = [R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]]
        views[v]["rot"] = R
        nl = osc.num_levels(v)
        views[v]["nlevels"] = nl
        for l in range(nl):
            K, Ki = osc.level_calib(v, l)
            img = osc.level(v, l)
            h, w = img.shape[:2]
            pitch = (w + 3) & ~3
            rgbx = np.zeros((h, pitch, 4), np.uint8)
            rgbx[:, :w, :3] = img
            rgbx[:, :w, 3] = 255
            keep.append(rgbx)
            # quad image (mve_b200/csrc/b200mvs.cu k_make_quads): the 2x2 neighbourhood of every texel, clamped at the border
            t = rgbx.view(np.uint32)[:, :, 0]
            x1 = np.minimum(np.arange(pitch) + 1, w - 1)
            y1 = np.minimum(np.arange(h) + 1, h - 1)
            quad = np.ascontiguousarray(np.stack([t, t[:, x1], t[y1, :], t[y1][:, x1]], -1))
            keep.append(quad)
            views[v]["quad"][l] = quad.ctypes.data
            views[v]["ax"][l], views[v]["ay"][l], views[v]["cx"][l], views[v]["cy"][l] = K[0], K[4], K[2], K[5]
            views[v]["w"][l], views[v]["h"][l], views[v]["pitch"][l] = w, h, pitch
            views[v]["img"][l] = rgbx.ctypes.data
            if l == 0:
                views[v]["inv_ax0"] = Ki[0]
    _, Ki = osc.level_calib(ref, settings.scale)
    ki = np.array([Ki[0], Ki[2], Ki[4], Ki[5]], np.float32)
    Hs, Ws = osc.level(ref, settings.scale).shape[:2]
    gv = np.asarray(gsel, np.int32)
    fs = np.array([settings.min_ncc, settings.min_parallax, settings.accept_ncc, settings.min_refine_diff], np.float32)
    isv = np.array([settings.max_iterations, settings.nr_recon_neighbors, settings.scale, settings.use_color_scale], np.int32)
    ein = np.zeros(len(pin), EMU_IN)
    ein["x"], ein["y"], ein["depth"], ein["dzI"], ein["dzJ"] = pin["x"], pin["y"], pin["depth"], pin["dz_i"], pin["dz_j"]
    slot_of = {v: k for k, v in enumerate(gsel)}
    for i in range(len(pin)):
        sl = sorted(slot_of[int(v)] for v in pin["local_ids"][i][:pin["n_local"][i]])
        word = 0xFFFFFFFF
        for k, q in enumerate(sl):
            word = (word & ~(0xFF << (8 * k))) | (q << (8 * k))
        ein["slots"][i] = word
    eout = np.zeros(len(pin), EMU_OUT)
    lut = _lut()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.emu_optimize_patches(p(views), s.n_views, ref, Ws, Hs, p(ki), p(gv), len(gv), p(fs), p(isv), p(lut), p(ein), len(ein), p(eout), mode)
    assert rc == 0
    out = np.zeros(len(pin), O.PATCH_OUT)
    out["conf"], out["depth"], out["dz_i"], out["dz_j"] = eout["conf"], eout["depth"], eout["dzI"], eout["dzJ"]
    out["normal"] = np.stack([eout["nx"], eout["ny"], eout["nz"]], 1)
    out["iterations"], out["converged"], out["opti_success"] = eout["iterations"], eout["flags"] & 1, (eout["flags"] >> 1) & 1
    for i in range(len(pin)):
        ids = [gsel[(int(eout["slots"][i]) >> (8 * k)) & 0xFF] if ((int(eout["slots"][i]) >> (8 * k)) & 0xFF) < len(gsel) else -1 for k in range(4)]
        out["local_ids"][i] = ids
        out["n_local"][i] = sum(1 for q in ids if q >= 0)
    return out, eout


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("name,view,kw", [("T0", 0, {}), ("T2", 0, {}), ("T4", 1, {}), ("T0", 2, dict(use_color_scale=0)),
                                          ("T2", 5, dict(nr_recon_neighbors=3)), ("T5", 1, {}), ("T6", 2, {})])
def test_kernel_body_on_oracle_trace(emu, name, view, kw, mode):
    """Seeds (full local view selection), propagated patches and - on the orbit scene - view replacements."""
    s = golden_scene(name)
    osc = O.OracleScene(s)
    base = dict(scale=s.scale, nr_recon_neighbors=s.nr_recon_neighbors)
    base.update(kw)
    st = O.default_settings(**base)
    gsel = osc.global_view_selection(st, view)
    r = osc.reconstruct(st, view, trace_cap=100000)
    tin, tout = r["trace_in"], r["trace_out"]
    seeds = np.nonzero(tin["n_local"] == 0)[0][:60]
    rest = np.nonzero(tin["n_local"] != 0)[0]
    # patches whose view set changed = a view was replaced on the way (rare path)
    changed = [i for i in rest if tout["conf"][i] > 0 and (tout["local_ids"][i] != tin["local_ids"][i]).any()][:40]
    pick = np.unique(np.concatenate([seeds, rest[:: max(1, len(rest) // 160)][:160], np.asarray(changed, dtype=np.int64)])).astype(np.int64)
    got, raw = _run(emu, s, osc, view, gsel, st, tin[pick], mode)
    c = patch_compare(got, tout[pick])
    n = c["n"]
    assert n >= 150
    assert c["ok_mismatch"] <= max(1, 0.01 * n), (c["ok_mismatch"], n)
    assert c["ids_mismatch"] <= max(1, 0.01 * n), (c["ids_mismatch"], n)
    assert (got["iterations"] != tout[pick]["iterations"])[c["both"]].mean() < 0.02
    assert np.percentile(c["rel"], 99) < 5e-5
    assert np.percentile(c["conf_abs"], 99) < 2e-4
    assert np.percentile(c["nrm_abs"], 99) < 1e-3
    # the fused sample sets per optimisation stay below the reference's separate ones (SURVEY 8d)
    assert raw["sets"][c["both"]].mean() < 40


@pytest.mark.parametrize("mode", [1, 2])
def test_kernel_body_vs_reference_golden(emu, mode):
    """Same device code against mvs::PatchOptimization results of the compiled reference (golden T0 subset)."""
    s = golden_scene("T0")
    ref = golden_ref("T0")
    osc = O.OracleScene(s)
    st = O.default_settings(scale=s.scale)
    pin, pout = ref["patch_in"], ref["patch_out"]
    pick = np.concatenate([np.arange(0, len(pin) - 6, 9), np.arange(len(pin) - 6, len(pin))])     # incl. the hostile inputs
    got, _ = _run(emu, s, osc, int(ref["patch_ref_view"]), ref["patch_gvs"].tolist(), st, pin[pick], mode)
    c = patch_compare(got, pout[pick])
    assert c["ok_mismatch"] <= 1 and c["ids_mismatch"] <= 1
    assert np.percentile(c["rel"], 99) < 5e-5
