"""The drop-in itself (-m gpu): the reference's UNMODIFIED CLI driver (apps/dmrecon/dmrecon.cc, compiled from the
reference tree) linked against our mvs::DMRecon shim + libb200mvs.so instead of libmve_dmrecon.a, run on an MVE scene
directory, must leave the same embeddings on disk as the reference binary did (golden maps minted by
tests/golden/make_golden.py from the reference CLI).  Skipped when oracle/_ref/shim/dmrecon_b200 was not built."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests.test_gpu_parity import CLI_CONF_P99
from tests.util import ROOT, golden_ref, golden_scene, map_stats

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "oracle", "_ref", "shim", "dmrecon_b200")


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built (needs the reference sources at build time)")
@pytest.mark.parametrize("name,views", [("T0", [0, 3]), ("T1", [4]), ("T5", [1]), ("T6", [2])])
def test_cli_writes_reference_layout(name, views):
    from mve_b200 import synth
    s = golden_scene(name)
    ref = golden_ref(name)
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        cmd = [CLI, "-s%d" % s.scale, "--local-neighbors=%d" % s.nr_recon_neighbors, "--keep-conf", "--keep-dz",
               "--progress=silent", "--force", "-l" + ",".join(str(v) for v in views), tmp]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stdout + out.stderr
        for v in views:
            vd = os.path.join(tmp, "views", "view_%04d.mve" % v)
            depth = synth.read_mvei(os.path.join(vd, "depth-L%d.mvei" % s.scale))
            conf = synth.read_mvei(os.path.join(vd, "conf-L%d.mvei" % s.scale))
            dz = synth.read_mvei(os.path.join(vd, "dz-L%d.mvei" % s.scale))
            assert depth.shape[2] == 1 and conf.shape[2] == 1 and dz.shape[2] == 2 and depth.dtype == np.float32
            iou, rel, both = map_stats(ref["depth_%d" % v], depth[:, :, 0])
            assert iou > 0.99
            assert np.percentile(rel, 50) < 5e-4 and np.percentile(rel, 99) < 5e-3
            assert np.percentile(np.abs(ref["conf_%d" % v] - conf[:, :, 0])[both], 99) < CLI_CONF_P99.get(name, 2e-2)
            if s.scale:
                und = [f for f in os.listdir(vd) if f.startswith("undist-L%d" % s.scale)]
                assert und, "undist-L<s> must be saved for scale != 0 (dmrecon.cc:138-143)"
                assert (synth.read_mvei(os.path.join(vd, und[0])) == ref["undist_%d" % v]).all()
        # resume semantics live in the unchanged driver: a second run without --force skips finished views
        out2 = subprocess.run([c for c in cmd if c != "--force"], capture_output=True, text=True, timeout=600)
        assert out2.returncode == 0


PLY_VIEWS = (0, 3)


def ply_cmd(exe, s, scene_dir):
    return [exe, "-s%d" % s.scale, "--progress=silent", "--force", "-p", "--plydest=plyout",
            "-l" + ",".join(str(v) for v in PLY_VIEWS), scene_dir]


def read_ply_header(path):
    """Binary little-endian PLY of mve::geom::save_ply_view: returns (n_vertices, n_faces, header text)."""
    raw = open(path, "rb").read()
    end = raw.index(b"end_header\n") + len(b"end_header\n")
    head = raw[:end].decode("ascii", "replace")
    nv = int([l for l in head.splitlines() if l.startswith("element vertex")][0].split()[-1])
    nf = int(([l for l in head.splitlines() if l.startswith("element face")] or ["element face 0"])[0].split()[-1])
    return nv, nf, head


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_writes_ply_like_the_reference():
    """-p / --writeply (settings.writePlyFile, plyPath; dmrecon.cc:109-117, single_view.cc:123-138): the drop-in writes
    mvs-<id>-L<s>.ply / .xf through the same libmve writers; vertex and face counts follow the depth map, so they agree with
    the reference's file (golden T0_ply_ref.npz) up to the pixels on which the maps differ, the .xf files are identical."""
    from mve_b200 import synth
    s = golden_scene("T0")
    ref = golden_ref("T0_ply")
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        out = subprocess.run(ply_cmd(CLI, s, tmp), capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="2"))
        assert out.returncode == 0, out.stdout + out.stderr
        for v in PLY_VIEWS:
            name = "mvs-%04d-L%d" % (v, s.scale)
            a = os.path.join(tmp, "plyout", name + ".ply")
            assert os.path.exists(a)
            assert open(os.path.join(tmp, "plyout", name + ".xf")).read() == str(ref["xf_%d" % v])
            nva, nfa, ha = read_ply_header(a)
            nvb, nfb = (int(x) for x in ref["ply_%d" % v])
            assert [l for l in ha.splitlines() if l.startswith("property")] == ref["ply_props_%d" % v].tolist()
            assert abs(nva - nvb) <= 0.01 * nvb + 5 and abs(nfa - nfb) <= 0.03 * nfb + 20, (nva, nvb, nfa, nfb)


@pytest.mark.skipif(not os.path.exists(CLI), reason="oracle/_ref/shim/dmrecon_b200 not built")
def test_cli_batches_the_views_in_flight():
    """The OpenMP threads of the unmodified driver (apps/dmrecon/dmrecon.cc:285) are combined into ONE b200mvs_reconstruct per
    GPU: with 6 views on 6 threads every 'Reconstructed view' line reports the features of the whole batch."""
    import re
    from mve_b200 import synth
    s = golden_scene("T0")
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_mve_scene(s, tmp)
        cmd = [CLI, "-s%d" % s.scale, "--progress=simple", "--force", tmp]
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=dict(os.environ, OMP_NUM_THREADS="6"))
        assert out.returncode == 0, out.stdout + out.stderr
        feats = [int(m) for m in re.findall(r"batch of all views in flight: (\d+) features processed", out.stdout)]
        assert len(feats) == s.n_views
        single = subprocess.run([CLI, "-s%d" % s.scale, "--progress=simple", "--force", "-l0", tmp], capture_output=True, text=True, timeout=600)
        one = int(re.findall(r"batch of all views in flight: (\d+) features processed", single.stdout)[0])
        assert max(feats) >= 3 * one, (feats, one)       # at least half of the team ended up in one batch
