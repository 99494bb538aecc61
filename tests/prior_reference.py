"""NumPy statement of the prior seed rule of b200mvs_set_view_prior (include/b200mvs.h): which pixels of a W x H map a
prior seeds, and at which depth."""
import numpy as np


def prior_cells(n: int, stride: int) -> int:
    """Candidate columns (rows) of a map n pixels wide (high): x = 2 + stride i <= n - 3."""
    return (n - 5) // stride + 1 if n >= 5 else 0


def prior_seeds(W: int, H: int, prior: np.ndarray, stride: int, mask=None):
    """The seeds of one entry with a W x H map: [(x, y, depth)] in row-major order.  prior: h x w float32; mask: the
    view's reconstruction mask (any size, 0 = background) or None.  Candidate (x, y) reads prior pixel
    ((2x+1) w // 2W, (2y+1) h // 2H) and seeds when that value is finite and > 0 and the mask pixel under it by the same
    rule is not 0."""
    prior = np.asarray(prior, np.float32)
    h, w = prior.shape
    out = []
    for k in range(prior_cells(H, stride)):
        y = 2 + stride * k
        for i in range(prior_cells(W, stride)):
            x = 2 + stride * i
            d = prior[(2 * y + 1) * h // (2 * H), (2 * x + 1) * w // (2 * W)]
            if not (np.isfinite(d) and d > 0):
                continue
            if mask is not None:
                mh, mw = mask.shape
                if mask[(2 * y + 1) * mh // (2 * H), (2 * x + 1) * mw // (2 * W)] == 0:
                    continue
            out.append((x, y, float(d)))
    return out
