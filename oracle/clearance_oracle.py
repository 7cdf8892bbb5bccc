"""Dense CPU restatement of svsdf_map_clearance (include/svsdf.h): every occupied map column, its centre, the swept-volume SDF there
(the oracle's getTrueSDFofSweptVolume<true>, oracle_py.Oracle.query), the cells with value <= d_max in map order, and the summary.

No band, no GPU: every occupied column is evaluated.  The GPU tests hold the library's band result to the same list computed from
svsdf_query over all occupied centres, and the strict build to this module bit for bit."""
from __future__ import annotations

import math

import numpy as np


def occupied_columns(occ) -> np.ndarray:
    """occ [X, Y] or [X, Y, Z] bool -> [n, 2] int64 (i, j) of the columns with any occupied layer, in ascending i * Y + j order."""
    occ = np.asarray(occ, dtype=bool)
    if occ.ndim == 3:
        occ = occ.any(axis=2)
    return np.argwhere(occ).astype(np.int64)


def centres(ij, origin, res) -> np.ndarray:
    """getGridCubeCenter: ((i + 0.5) res + ox, (j + 0.5) res + oy), one rounding per operation (as the extraction kernel computes it)."""
    ij = np.asarray(ij, dtype=np.int64).reshape(-1, 2)
    xy = np.empty((ij.shape[0], 2))
    for a in range(2):
        xy[:, a] = (ij[:, a].astype(np.float64) + 0.5) * float(res) + float(origin[a])
    return xy


def check_d_max(d_max) -> float:
    d = float(d_max)
    if not d >= 0.0:
        raise ValueError("d_max must be >= 0 or +inf")
    return d


def summarise(ij, xy, sdf, tstar, d_max, n_occupied, n_evaluated=None) -> dict:
    """The listed cells (value <= d_max, in the given order) and the summary computed from them: n_within, n_colliding (value <= 0),
    min_sdf (+inf when the list is empty) and argmin (first in list order among ties; -1 when empty)."""
    d = check_d_max(d_max)
    sdf = np.asarray(sdf, dtype=np.float64).reshape(-1)
    keep = sdf <= d
    out = dict(ij=np.asarray(ij).reshape(-1, 2)[keep], xy=np.asarray(xy, dtype=np.float64).reshape(-1, 2)[keep], sdf=sdf[keep],
               tstar=np.asarray(tstar, dtype=np.float64).reshape(-1)[keep], n_occupied=int(n_occupied),
               n_evaluated=int(len(sdf) if n_evaluated is None else n_evaluated))
    s = out["sdf"]
    out["n_within"] = int(s.size)
    out["n_colliding"] = int(np.count_nonzero(s <= 0.0))
    out["argmin"] = int(np.argmin(s)) if s.size else -1  # np.argmin: the first occurrence of the minimum
    out["min_sdf"] = float(s[out["argmin"]]) if s.size else math.inf
    return out


def clearance(orc, occ, origin, res, d_max=math.inf) -> dict:
    """svsdf_map_clearance evaluated densely: `orc` is an oracle_py.Oracle whose trajectory is set; occ [X, Y(, Z)] the occupancy,
    origin the map's (x, y) minimum corner, res its resolution."""
    check_d_max(d_max)
    ij = occupied_columns(occ)
    xy = centres(ij, origin, res)
    if len(ij):
        sdf, ts, _, _ = orc.query(np.c_[xy, np.zeros(len(xy))])
    else:
        sdf, ts = np.empty(0), np.empty(0)
    return summarise(ij, xy, sdf, ts, d_max, len(ij))
