"""Host-only check of the LMBM plug-in (svsdf_lmbm_*), run by tests/test_capi_host.py in a subprocess.  Prints one JSON line.

    python tests/tools/lmbm_plugin_check.py [--lib PATH]

PATH is any library exporting lmbm::lmbm_optimize: tests/cpp/lmbm_standin.cpp built by the test, or by default oracle/_ref/lmbm.so
(the reference's prebuilt binary, which needs a libgfortran.so.5 on the loader path; scipy bundles a copy).

1. svsdf_lmbm_minimize on a non-smooth test function == calling lmbm::lmbm_optimize of the same file directly (ctypes), bit for bit.
2. Two handles opened as PRIVATE COPIES minimise two different functions concurrently from two threads and each returns what it returns
   when run alone; two handles on the SAME instance (private_copy = 0) share the library's static callback slot (lmbm.cpp:4-6), which is
   what makes the private copies necessary — shown by the handles' distinct load addresses of the optimise symbol."""
import ctypes as C
import glob
import json
import os
import sys
import threading

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REFDIR = os.path.join(ROOT, "oracle", "_ref")
LMBM = os.path.join(REFDIR, "lmbm.so")
SYM = "_ZN4lmbm13lmbm_optimizeEiPdS0_PFdPvPKdS0_iES1_PFiS1_S3_iEPNS_16lmbm_parameter_tE"


def ensure_loader_path():
    if os.environ.get("SVSDF_LMBM_REEXEC") == "1":
        return
    link = os.path.join(REFDIR, "libgfortran.so.5")
    extra = [REFDIR]
    if not os.path.exists(link):
        import scipy

        cand = sorted(glob.glob(os.path.join(os.path.dirname(scipy.__file__), "..", "scipy.libs", "libgfortran-*.so.5*")))
        if cand:
            if os.path.lexists(link):
                os.remove(link)
            os.symlink(os.path.abspath(cand[0]), link)
    if os.path.exists(link):
        extra.append(os.path.dirname(os.path.realpath(link)))
    env = dict(os.environ, SVSDF_LMBM_REEXEC="1", LD_LIBRARY_PATH=":".join(extra + [os.environ.get("LD_LIBRARY_PATH", "")]))
    os.execve(sys.executable, [sys.executable] + sys.argv, env)


def main():
    global LMBM
    if "--lib" in sys.argv:  # a self-contained library: no Fortran runtime to find
        LMBM = os.path.abspath(sys.argv[sys.argv.index("--lib") + 1])
    elif not os.path.exists(LMBM):
        print(json.dumps({"unavailable": "oracle/_ref/lmbm.so not present"}))
        return
    else:
        ensure_loader_path()
    import numpy as np

    sys.path.insert(0, ROOT)
    from implicit_svsdf_planner_b200 import api

    def make(seed, n):
        rng = np.random.default_rng(seed)
        A = rng.normal(size=(n, n))
        A = A @ A.T / n + np.eye(n)
        c = rng.normal(size=n)

        def fun(x):  # smooth bowl + l1 kink + max term: non-smooth, convex
            r = x - c
            k = int(np.argmax(np.abs(x)))
            g = A @ r + 0.3 * np.sign(x)
            g[k] += 0.5 * np.sign(x[k])
            return 0.5 * r @ A @ r + 0.3 * np.abs(x).sum() + 0.5 * np.abs(x[k]), g

        return fun, rng.normal(size=n) * 3

    out = {}
    # 1. plug-in vs the library called directly
    fun, x0 = make(1, 12)
    h = api.Lmbm(LMBM, private_copy=True)
    rc, x, f, ne = h.minimize(fun, x0)
    L = C.CDLL(LMBM)
    opt = getattr(L, SYM)
    opt.restype = C.c_int
    dp = C.POINTER(C.c_double)

    def _eval(_i, xp, gp, n):
        xv = np.ctypeslib.as_array(xp, shape=(n,))
        fv, g = fun(xv.copy())
        np.ctypeslib.as_array(gp, shape=(n,))[:] = g
        return float(fv)

    cb = api.EVAL_T(_eval)
    noprog = C.CFUNCTYPE(C.c_int, C.c_void_p, dp, C.c_int)(lambda _i, _x, _k: 0)  # lmbm.cpp calls it unconditionally
    xd = x0.copy()
    fd = C.c_double()
    p = api.lmbm_default_params()
    rcd = opt(C.c_int(xd.size), xd.ctypes.data_as(dp), C.byref(fd), cb, None, noprog, C.byref(p))
    out["direct_equal"] = bool(rc == rcd and np.array_equal(x, xd) and f == fd.value)
    out["status"], out["f"], out["evals"], out["f_start"] = int(rc), float(f), int(ne), float(fun(x0)[0])
    # 2. concurrency with private copies
    funs = [make(10 + k, 8 + 4 * k) for k in range(2)]
    alone = []
    for fn, xs in funs:
        hh = api.Lmbm(LMBM, private_copy=True)
        alone.append(hh.minimize(fn, xs))
        hh.close()
    handles = [api.Lmbm(LMBM, private_copy=True) for _ in funs]
    res = [None, None]

    def work(k):
        for _ in range(5):  # several runs each, interleaved by the GIL hand-over inside the callbacks
            res[k] = handles[k].minimize(funs[k][0], funs[k][1])

    th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    [t.start() for t in th]
    [t.join() for t in th]
    out["concurrent_equal_alone"] = bool(all(res[k][0] == alone[k][0] and np.array_equal(res[k][1], alone[k][1]) and res[k][2] == alone[k][2] for k in range(2)))
    out["concurrent_status"] = [int(r[0]) for r in res]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
