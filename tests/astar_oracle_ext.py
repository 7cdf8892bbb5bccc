"""Test helper: the CPU oracle's A* with an expansion budget and per-search branch counters (tests/cpp/astar_oracle_ext.cpp).

The shared library is compiled on first use into a temporary directory (the tree is left as it is), with the oracle's own flags
(portable sin/cos, no FMA contraction), so its searches are bit for bit those of oracle_py.astar."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def _load():
    global _lib
    if _lib is None:
        d = tempfile.mkdtemp(prefix="astar_oracle_ext_")
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, "libastar_oracle_ext.so")
        subprocess.check_call(["/usr/bin/g++", "-O3", "-fopenmp", "-std=c++17", "-fPIC", "-mfma", "-ffp-contract=off", "-shared",
                               os.path.join(_HERE, "cpp", "astar_oracle_ext.cpp"), "-o", so])
        L = C.CDLL(so)
        dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.ext_astar.restype = C.c_int
        L.ext_astar.argtypes = [C.c_char_p, dp, C.c_int, C.c_int, C.c_double, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_double, C.c_double,
                                C.c_double, C.c_int, dp, dp, C.c_int, C.c_int, dp, ip, ip, ip]
        _lib = L
    return _lib


def astar(name, occ, start_xy, goal_xy, origin=(0.0, 0.0), map_res=1.0, kernel_size=17, kernel_count=18, safeh=0.0, max_path=1024,
          poly_params=(0.0, 0.0, 0.0), max_expansions=None, counts=False):
    """oracle_py.astar with max_expansions (None: the reference's unbounded loop) passed to the oracle's astar_search.  counts=True
    appends counts [n, 3] per search: closed nodes re-opened, open nodes improved without re-keying, pops decided by insertion order
    among equal keys (from an instrumented copy of the loop that must reproduce the oracle's paths and expansion counts)."""
    occ = np.ascontiguousarray(occ, dtype=np.uint8)
    X, Y = occ.shape
    pp = np.ascontiguousarray(poly_params, dtype=np.float64)
    st = np.ascontiguousarray(start_xy, dtype=np.float64).reshape(-1, 2)
    go = np.ascontiguousarray(goal_xy, dtype=np.float64).reshape(-1, 2)
    n = st.shape[0]
    path = np.zeros((n, max_path, 3))
    ln = np.zeros(n, dtype=np.int32)
    ex = np.zeros(n, dtype=np.int32)
    cnt = np.zeros((n, 3), dtype=np.int32) if counts else None
    dp, ip = C.POINTER(C.c_double), C.POINTER(C.c_int)
    differ = _load().ext_astar(name.encode(), pp.ctypes.data_as(dp), kernel_size, kernel_count, safeh, occ.ctypes.data_as(C.POINTER(C.c_uint8)),
                               X, Y, float(origin[0]), float(origin[1]), float(map_res), n, st.ctypes.data_as(dp), go.ctypes.data_as(dp),
                               max_path, (1 << 30) if max_expansions is None else int(max_expansions), path.ctypes.data_as(dp),
                               ln.ctypes.data_as(ip), ex.ctypes.data_as(ip), cnt.ctypes.data_as(ip) if counts else None)
    assert differ == 0, f"the instrumented search differs from the oracle's in {differ} searches"
    paths = [path[q, : ln[q]].copy() if ln[q] else None for q in range(n)]
    return (paths, ex, cnt) if counts else (paths, ex)
