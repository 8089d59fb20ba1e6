"""CPU oracle of the directed Chamfer distances (utils.training.chamfer_distances): for masks a, b of one map,
d(A -> B) = mean over A's cells of the Euclidean distance, in cells, to the nearest cell of B, and d(B -> A); NaN in
both when either set is empty.  `chamfer` uses scipy.ndimage.distance_transform_edt; `chamfer_brute` compares every
pair of cells, for small masks."""
import numpy as np
from scipy import ndimage


def chamfer(a, b) -> np.ndarray:
    """fp64 [B,2] of masks [B,H,W] (or [B,1,H,W]); a cell is in a set iff its value != 0."""
    a, b = np.asarray(a), np.asarray(b)
    if a.ndim == 4:
        a, b = a[:, 0], b[:, 0]
    out = np.full((a.shape[0], 2), np.nan)
    for k, (x, y) in enumerate(zip(a != 0, b != 0)):
        if x.any() and y.any():
            # distance_transform_edt gives each non-zero cell its distance to the nearest zero cell
            out[k, 0] = ndimage.distance_transform_edt(~y)[x].mean()
            out[k, 1] = ndimage.distance_transform_edt(~x)[y].mean()
    return out


def chamfer_brute(a, b) -> np.ndarray:
    a, b = np.asarray(a), np.asarray(b)
    if a.ndim == 4:
        a, b = a[:, 0], b[:, 0]
    out = np.full((a.shape[0], 2), np.nan)
    for k, (x, y) in enumerate(zip(a != 0, b != 0)):
        pa, pb = np.argwhere(x).astype(np.float64), np.argwhere(y).astype(np.float64)
        if len(pa) and len(pb):
            d = np.sqrt(((pa[:, None, :] - pb[None, :, :]) ** 2).sum(-1))
            out[k] = d.min(1).mean(), d.min(0).mean()
    return out
