"""The case matrix of the A* front end's reference pin (tests/test_oracle_front_ref_pin.py, tests/test_gpu_front_edges.py,
tests/golden/make_front_golden.py), and the records each implementation produces on it.

Expand cases: every analytic shape + Circle, without and with a body-frame pre-transform, each on one of the map geometries
GEOMS (resolutions 0.1 / 0.25 / 1 / 2.5, an origin not exact in binary, half boxes from under one cell to 160 cells per side,
X or Y = 1, Y = 0, 1, 31 mod 32, Y + 2h = 0, 1, 7 mod 8, no inflation (kernel size 1), densities 0 / 0.01 / 0.3 / 1, safe margins below, at and above res / 2).
Nodes: the map's corners and edge cells (so that projInMap clamps the box on every side) and random ones; father yaws: the
edges of `father_i = int(K (fy + pi) / (2 pi))` (pi = 3.1415926536) — -pi and its neighbouring doubles, pi - eps, 0, the
kernel yaws 2 pi i / K - pi and their neighbours, and values outside [-pi, pi) where the index must be clamped.
Search cases: a scene per shape and pre-transform at res 0.25 and 2.5 with 1 and 64 yaw kernels.

The reference's own code is undefined in three places the matrix reaches, so the reference pin leaves them out and the GPU test
holds the device to the oracle there: father yaws whose index falls outside [0, K) (checkKernelValue indexes its arrays with
it unclamped), yaw counts whose initShape loop runs K + 1 times (3, 36, 63 here; DESIGN.md §4), and the Circle: Circle(conf), the
constructor the reference's registry calls (Shape.hpp:444-458), never runs initShape, so it has no kernels to search with.
"""
from __future__ import annotations

import hashlib
import math

import numpy as np

SHAPES = ["star", "sdHorseshoe", "sdPie", "sdPie2", "sdArc", "sdTunnel", "sdCutDisk", "sdTrapezoid", "sdRhombus", "sdHeart", "sdRoundedX",
          "bigX", "sdRoundedCross", "sdOrientedVesica", "sdMoon", "sdUnevenCapsule", "Circle"]
PRE = [(0.0, 0.0, 0.0), (0.3, -0.2, 20.0)]
PI_CODE = 3.1415926536  # sw_manager.hpp:20
REF_KERNEL_SHAPES = SHAPES[:16]  # Circle(conf) never runs initShape (Shape.hpp:444-458)
ORIGIN = (-12.37, 3.1)

# res, X, Y, kernel_size, yaw kernels, front_end_safeh, density.  The yaw counts whose initShape loop overruns (3, 36, 63) are
# outside the reference pin, so each geometry that carries one also appears with a count that does not.
GEOMS = [
    dict(res=0.1, X=250, Y=223, ks=17, K=18, safeh=0.0, density=0.01),    # box 90 cells per side; Y = 31 mod 32, Y + 2h = 7 mod 8
    dict(res=2.5, X=40, Y=33, ks=1, K=1, safeh=0.0, density=0.3),         # box 0.4 cell; Y = 1 mod 32 and mod 8
    dict(res=0.25, X=1, Y=64, ks=3, K=2, safeh=0.0, density=0.3),         # X = 1; Y = 0 mod 32
    dict(res=1.0, X=37, Y=1, ks=31, K=63, safeh=0.0, density=0.3),        # Y = 1, Y + 2h = 7 mod 8; K = 63 overruns initShape
    dict(res=0.25, X=60, Y=32, ks=17, K=64, safeh=0.125, density=0.3),    # safeh = res / 2; Y + 2h = 0 mod 8
    dict(res=2.5, X=30, Y=31, ks=3, K=3, safeh=2.0, density=1.0),         # full map; safeh > res / 2; K = 3 overruns
    dict(res=1.0, X=40, Y=40, ks=17, K=36, safeh=0.0, density=0.0),       # empty map; K = 36 overruns
    dict(res=0.1, X=180, Y=97, ks=31, K=18, safeh=0.03, density=0.01),    # box 160 cells per side; safeh < res / 2
    dict(res=1.0, X=37, Y=1, ks=31, K=64, safeh=0.0, density=0.3),        # the three above with counts the reference pin reaches
    dict(res=2.5, X=30, Y=31, ks=3, K=2, safeh=2.0, density=1.0),
    dict(res=1.0, X=40, Y=40, ks=17, K=18, safeh=0.0, density=0.0),
    dict(res=0.25, X=45, Y=39, ks=1, K=18, safeh=0.0, density=0.3),       # no inflation (h = 0) and a 4-cell box: clamped at hi itself
]


def init_shape_overruns(K: int) -> bool:
    """Shape.hpp:401: `for (yaw = -PI; yaw < PI; yaw += yaw_res, ind++)` runs more than K times."""
    PI = 3.14159265358979323846
    yr, y, n = 2 * PI / K, -PI, 0
    while y < PI:
        n += 1
        y += yr
    return n > K


def father_index(K: int, fy: np.ndarray) -> np.ndarray:
    return np.trunc(K * ((np.asarray(fy, dtype=np.float64) + PI_CODE) / (2 * PI_CODE))).astype(np.int64)


def father_yaws(K: int) -> np.ndarray:
    up, dn = math.inf, -math.inf
    v = [-PI_CODE, math.nextafter(-PI_CODE, up), math.nextafter(-PI_CODE, dn), math.pi - 1e-12, PI_CODE - 1e-12,
         math.nextafter(PI_CODE, dn), 0.0, -0.0, 3.2, -3.2, -3.5, 10.0, -10.0, math.pi, -math.pi]
    for i in sorted({0, 1, K // 2, K - 1}):
        y = 2 * PI_CODE * i / K - PI_CODE  # the child yaw checkKernelValue hands back for kernel i
        v += [y, math.nextafter(y, up), math.nextafter(y, dn)]
    return np.array(v)


def expand_cases():
    out = []
    for i in range(2 * len(SHAPES)):
        g = dict(GEOMS[i % len(GEOMS)])
        g.update(shape=SHAPES[i % len(SHAPES)], pp=PRE[i // len(SHAPES)], seed=1000 + i)
        out.append(g)
    return out


def expand_inputs(c):
    """occ [X, Y] bool, node_ij [n, 2], node_yaw [n]."""
    X, Y = c["X"], c["Y"]
    rng = np.random.default_rng(c["seed"])
    occ = rng.random((X, Y)) < c["density"] if 0 < c["density"] < 1 else np.full((X, Y), c["density"] >= 1)
    edge = [(0, 0), (0, Y - 1), (X - 1, 0), (X - 1, Y - 1), (X // 2, 0), (X // 2, Y - 1), (0, Y // 2), (X - 1, Y // 2), (1, 1), (X - 2, Y - 2),
            (1, Y - 1), (X - 1, 1)]
    ij = [(min(max(a, 0), X - 1), min(max(b, 0), Y - 1)) for a, b in edge]
    ij += list(zip(rng.integers(0, X, 12), rng.integers(0, Y, 12)))
    fys = father_yaws(c["K"])
    ij = np.array(ij, dtype=np.int32)
    n = max(len(ij), len(fys))
    ij = ij[np.arange(n) % len(ij)]
    fy = fys[np.arange(n) % len(fys)]
    return occ, ij, fy


def ref_defined(c, fy):
    """Nodes on which the reference's own code is defined (see the module docstring)."""
    if init_shape_overruns(c["K"]) or c["shape"] not in REF_KERNEL_SHAPES:
        return np.zeros(len(fy), dtype=bool)
    fi = father_index(c["K"], fy)
    return (fi >= 0) & (fi < c["K"])


def search_cases():
    """Every shape with and without the pre-transform; res 0.25 (17-cell kernels) and 2.5 (3-cell kernels), K = 1 and 64."""
    out = []
    for s in range(2 * len(SHAPES)):
        res = (0.25, 2.5)[s % 2]
        fine = res == 0.25
        out.append(dict(shape=SHAPES[s % len(SHAPES)], pp=PRE[s // len(SHAPES)], res=res, ks=17 if fine else 3, K=(1, 64)[(s // 2) % 2],
                        safeh=0.0, X=56 if fine else 20, Y=52 if fine else 19, density=0.0015 if fine else 0.04, seed=2000 + s))
    return out


def search_inputs(c):
    """occ [X, Y], start [m, 2], goal [m, 2] in world coordinates: the map's two corners (getGridIndex clamps the upper one),
    three pairs at least a kernel's half width from the border, and a start just outside the map (the search does not run)."""
    X, Y, res = c["X"], c["Y"], c["res"]
    rng = np.random.default_rng(c["seed"])
    occ = rng.random((X, Y)) < c["density"]
    lo = np.array(ORIGIN)
    hi = lo + res * np.array([X, Y])
    m = res * min(c["ks"] // 2 + 2, min(X, Y) // 4)
    st = rng.uniform(lo + m, hi - m, (5, 2))
    go = rng.uniform(lo + m, hi - m, (5, 2))
    st[0], go[0] = lo, hi
    st[4] = [lo[0] - 0.5 * res, lo[1]]
    return occ, st, go


def digest(a) -> str:
    a = np.ascontiguousarray(a)
    if a.dtype == bool:
        a = a.astype(np.uint8)
    return hashlib.sha256(a.tobytes()).hexdigest()


def aabb_digest(points_fn, c, ij):
    """getPointsInAABB2D around the centre of every valid neighbour cell of the nodes, half box kernel_size/2 + 1."""
    hb = c["ks"] // 2 + 1
    h = hashlib.sha256()
    for ix, iy in ij:
        for m in range(9):
            vx, vy = ix + m // 3 - 1, iy + m % 3 - 1
            if not (0 <= vx < c["X"] and 0 <= vy < c["Y"]):
                continue
            centre = ((vx + 0.5) * c["res"] + ORIGIN[0], (vy + 0.5) * c["res"] + ORIGIN[1])
            pts = np.ascontiguousarray(points_fn(centre, hb), dtype=np.float64)
            h.update(np.int64(len(pts)).tobytes())
            h.update(pts.tobytes())
    return h.hexdigest()


def pack_paths(paths):
    lens = np.array([0 if p is None else len(p) for p in paths], dtype=np.int32)
    cat = np.concatenate([p for p in paths if p is not None], axis=0) if lens.any() else np.zeros((0, 3))
    return lens, cat


def _expand_record(i, c, impl, defined):
    """impl: an object with kernels(), cspace(), expand(ij, fy), check_kernel_value(fy, ij), points_in_aabb(centre, half)."""
    occ, ij, fy = expand_inputs(c)
    rec = {}
    _, _, byt = impl.kernels()
    rec[f"e{i}_kern"] = np.array(digest(byt))
    rec[f"e{i}_cspace"] = np.array(digest(impl.cspace()))
    rec[f"e{i}_aabb"] = np.array(aabb_digest(impl.points_in_aabb, c, ij))
    d = np.asarray(defined)
    ok, cy, parts = impl.expand(ij[d], fy[d])
    rec[f"e{i}_ok"], rec[f"e{i}_cy"], rec[f"e{i}_parts"] = ok.astype(np.uint8), cy, parts
    ok1, cy1 = impl.check_kernel_value(fy[d], ij[d])
    rec[f"e{i}_ckv_ok"], rec[f"e{i}_ckv_cy"] = ok1.astype(np.uint8), cy1
    return rec


def _search_record(i, paths, ex, found):
    lens, cat = pack_paths(paths)
    return {f"s{i}_len": lens, f"s{i}_path": cat, f"s{i}_ex": np.asarray(ex, dtype=np.int32), f"s{i}_found": np.asarray(found, dtype=np.uint8)}


def reference_records(variant="portable"):
    """Every record of the reference's own code (oracle/_ref/libref_front_<variant>.so) on the matrix, where it is defined."""
    from oracle import ref_front_py as RF

    rec = {}
    for i, c in enumerate(expand_cases()):
        occ, ij, fy = expand_inputs(c)
        d = ref_defined(c, fy)
        if not d.any():
            continue
        R = RF.RefFront(c["shape"], occ, ORIGIN, c["res"], c["ks"], c["K"], c["safeh"], c["pp"], variant=variant)
        rec[f"e{i}_mk"] = np.array(digest(R.map_kernel()))
        rec.update(_expand_record(i, c, R, d))
        assert np.array_equal(R.cspace(True), R.cspace(False)), ("kernelConv<true> != kernelConv<false>", i)
        R.close()
    for i, c in enumerate(search_cases()):
        if c["shape"] not in REF_KERNEL_SHAPES:
            continue
        occ, st, go = search_inputs(c)
        R = RF.RefFront(c["shape"], occ, ORIGIN, c["res"], c["ks"], c["K"], c["safeh"], c["pp"], variant=variant)
        paths, ex, found = R.astar(st, go)
        rec.update(_search_record(i, paths, ex, found))
        R.close()
    return rec


class OracleFront:
    """oracle/frontend_oracle.hpp through oracle_py, with RefFront's calls."""

    def __init__(self, oracle_mod, c, occ):
        self.o, self.c, self.occ = oracle_mod, c, occ
        self.kw = dict(kernel_size=c["ks"], kernel_count=c["K"], safeh=c["safeh"], poly_params=c["pp"])

    def kernels(self):
        c = self.c
        return self.o.shape_kernels(c["shape"], c["ks"], c["K"], c["res"], c["safeh"], poly_params=c["pp"])

    def cspace(self):
        c = self.c
        return self.o.cspace(c["shape"], self.occ, c["ks"], c["K"], c["res"], c["safeh"], variant="byte", poly_params=c["pp"])

    def expand(self, ij, fy):
        return self.o.expand_nodes(self.c["shape"], self.occ, ij, fy, origin=ORIGIN, map_res=self.c["res"], **self.kw)

    def check_kernel_value(self, fy, ij):
        c = self.c
        return self.o.check_kernel_value(c["shape"], self.occ, fy, ij, c["ks"], c["K"], c["res"], c["safeh"], poly_params=c["pp"])

    def points_in_aabb(self, centre, half):
        return self.o.points_in_aabb(self.occ, centre, half, origin=ORIGIN, map_res=self.c["res"])


def oracle_records(oracle_mod, all_nodes=False):
    """The oracle's records on the matrix: on the reference's defined nodes, or (all_nodes) on every node of every case."""
    rec = {}
    for i, c in enumerate(expand_cases()):
        occ, ij, fy = expand_inputs(c)
        d = np.ones(len(fy), dtype=bool) if all_nodes else ref_defined(c, fy)
        if not d.any():
            continue
        rec.update(_expand_record(i, c, OracleFront(oracle_mod, c, occ), d))
    for i, c in enumerate(search_cases()):
        occ, st, go = search_inputs(c)
        paths, ex = oracle_mod.astar(c["shape"], occ, st, go, origin=ORIGIN, map_res=c["res"], kernel_size=c["ks"], kernel_count=c["K"],
                                     safeh=c["safeh"], max_path=4096, poly_params=c["pp"])
        rec.update(_search_record(i, paths, ex, [p is not None for p in paths]))
    return rec


def save_npz(path, rec):
    """np.savez_compressed with fixed zip timestamps and key order, so that the same records give the same bytes."""
    import io
    import zipfile

    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(rec):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(rec[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), compress_type=zipfile.ZIP_DEFLATED)
