"""Argument checks of the b200mvs_pset_* C ABI that come before any device work, so they hold without a GPU: option
combinations that cannot give the reference's output are rejected with B200MVS_ERR_INVALID_ARG and a message."""
import pytest


@pytest.mark.parametrize("opts,msg", [
    (dict(with_normals=True, with_conf=True, poisson_normals=True, conf_iterations=0), "Invalid amount of iterations"),
    (dict(with_conf=True, conf_iterations=0), "Invalid amount of iterations"),
    (dict(with_conf=True, conf_iterations=-3), "Invalid amount of iterations"),
    (dict(poisson_normals=True, with_normals=True), "poisson_normals needs with_normals and with_conf"),
    (dict(correspondence=True, aabb=((0, 0, 0), (1, 1, 1))), "correspondence needs every vertex"),
])
def test_pset_create_rejects(opts, msg):
    from mve_b200 import depthmap as D
    from mve_b200 import dmrecon
    with pytest.raises(dmrecon.B200MVSError) as e:
        D.scene_pointset([], opts)
    assert e.value.code == dmrecon.ERR_INVALID_ARG and msg in str(e.value), str(e.value)
