"""Per-view counters of one frontier launch with thousands of reference views (-m gpu).  The host copy of a launch's
counters holds the `filled` count of every view of a full group apart from the launch's control block, so a large batch
reports the same progress[].filled and stats.n_filled as the views run one at a time."""
import pytest

from tests.util import golden_scene

pytestmark = pytest.mark.gpu


def test_filled_of_every_view_of_a_large_launch():
    from mve_b200 import dmrecon
    s = golden_scene("T0")
    st = dmrecon.Settings(scale=1, nr_recon_neighbors=s.nr_recon_neighbors)
    g = dmrecon.Scene.from_synth(s)
    single = []
    for v in range(s.n_views):
        prog = (dmrecon.Progress * 1)()
        _, stats = g.reconstruct(st, [v], want=("depth",), progress=prog)
        assert prog[0].filled == stats.n_filled > 0
        single.append(prog[0].filled)
    refs = [j % s.n_views for j in range(2112)]          # more than 2048 counters: past the first 16 KiB of the host copy
    prog = (dmrecon.Progress * len(refs))()
    _, stats = g.reconstruct(st, refs, want=("depth",), progress=prog)
    assert stats.n_patch_launches == 1
    assert [prog[j].filled for j in range(len(refs))] == [single[r] for r in refs]
    assert stats.n_filled == sum(single[r] for r in refs)
    g.close()
