"""NumPy statement of the state rule of b200mvs_set_view_prior_state (include/b200mvs.h): next to the depth of
tests/prior_reference.py, the dz and local views each prior seed of an entry carries."""
import numpy as np

from tests.prior_reference import prior_seeds


def seed_state(dz, ids, w: int, h: int, W: int, H: int, gview, N: int):
    """The state of one candidate: (dz_i, dz_j, local ids or None).  dz: the prior pixel's two float32 values or None;
    ids: its four int32 view ids or None; w x h the prior's size, W x H the entry's map, gview the entry's global
    selection, N nr_recon_neighbors."""
    di = dj = np.float32(0)
    if dz is not None:
        with np.errstate(over="ignore", invalid="ignore"):        # an overflow is the case the rule tests for
            a = np.float32(dz[0]) * (np.float32(w) / np.float32(W))
            b = np.float32(dz[1]) * (np.float32(h) / np.float32(H))
        if np.isfinite(a) and np.isfinite(b):
            di, dj = a, b
    local = None
    if ids is not None:
        valid = sorted({int(i) for i in ids if i >= 0 and int(i) in set(int(g) for g in gview)})
        if len(valid) == N:
            local = valid
    return float(di), float(dj), local


def prior_state_seeds(W: int, H: int, depth: np.ndarray, stride: int, gview, N: int, dz=None, ids=None, mask=None):
    """The seeds of one entry with a W x H map: [(x, y, depth, dz_i, dz_j, local ids or None)] in row-major order.
    depth: h x w float32; dz: h x w x 2 float32 or None; ids: h x w x 4 int32 or None."""
    depth = np.asarray(depth, np.float32)
    h, w = depth.shape
    out = []
    for x, y, d in prior_seeds(W, H, depth, stride, mask):
        py, px = (2 * y + 1) * h // (2 * H), (2 * x + 1) * w // (2 * W)
        st = seed_state(None if dz is None else dz[py, px], None if ids is None else ids[py, px], w, h, W, H, gview, N)
        out.append((x, y, d) + st)
    return out
