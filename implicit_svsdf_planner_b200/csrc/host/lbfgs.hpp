// host/lbfgs.hpp — outer optimiser of the drop-in: limited-memory BFGS with the Lewis–Overton weak-Wolfe line search (suitable for
// the piecewise-smooth SVSDF cost).  Algorithm and return codes follow the clean LBFGS-Lite the reference vendors
// (src/utils/include/utils/lbfgs_ref.hpp:276-395 line search, :434-716 driver); re-implemented without Eigen on plain arrays and
// re-entrant (no static state, unlike the reference's LMBM wrapper src/utils/include/utils/lmbm.cpp:4-6).
//
// The solver is a machine that stops whenever it needs its caller (lbfgs_begin / lbfgs_step): to evaluate f and g at x, or to run
// the progress hook.  Its state is one LbfgsMachine and caller-provided flat storage (LbfgsArrays), so the same code runs in a host
// loop (Lbfgs::minimize) and, on one lane of each problem's warp, on the device (svsdf_backend.cu, svsdf_optimize_device).  Both builds keep
// the operations in this order without contraction (host: -ffp-contract=off, device: -fmad=false); division and sqrt are
// correctly rounded on both sides, so both give the same bits.
#pragma once
#include <cmath>
#include <cstddef>
#include <vector>

#include "../svsdf_types.h"

namespace svsdf {
namespace host {

struct LbfgsParams {
    int mem_size = 8;
    int past = 3;
    double delta = 1.0e-6;
    double g_epsilon = 1.0e-5;
    int max_iterations = 0;
    int max_linesearch = 64;
    double min_step = 1.0e-20;
    double max_step = 1.0e+20;
    double f_dec_coeff = 1.0e-4;
    double s_curv_coeff = 0.9;
    double cautious_factor = 1.0e-6;
    double machine_prec = 1.0e-16;
    int nonsmooth_restarts = 0;   // see svsdf_lbfgs_params
    // 1: behave like the reference's patched utils/lbfgs.hpp (the solver of its mid end): the line search accepts on the Armijo
    // condition alone (the weak-Wolfe branch is `if (0)`, lbfgs.hpp:375) and a quasi-Newton direction with |d| >= 0.04 or d.g > 0 —
    // or a skipped cautious update — is replaced by -g scaled to the previous direction's length after one more evaluation at the
    // same point (lbfgs.hpp:759-779).
    int reference_patch = 0;
};

enum LbfgsCode {
    LBFGS_CONVERGENCE = 0,
    LBFGS_STOP = 1,
    LBFGS_CANCELED = 2,
    LBFGS_NOMOREPROGRESS = 3,  // line search failed along -g: no decrease to line-search precision (kink of a non-smooth cost)
    LBFGSERR_UNKNOWNERROR = -1024,
    LBFGSERR_INVALID_N,
    LBFGSERR_INVALID_MEMSIZE,
    LBFGSERR_INVALID_GEPSILON,
    LBFGSERR_INVALID_TESTPERIOD,
    LBFGSERR_INVALID_DELTA,
    LBFGSERR_INVALID_MINSTEP,
    LBFGSERR_INVALID_MAXSTEP,
    LBFGSERR_INVALID_FDECCOEFF,
    LBFGSERR_INVALID_SCURVCOEFF,
    LBFGSERR_INVALID_MACHINEPREC,
    LBFGSERR_INVALID_MAXLINESEARCH,
    LBFGSERR_INVALID_FUNCVAL,
    LBFGSERR_MINIMUMSTEP,
    LBFGSERR_MAXIMUMSTEP,
    LBFGSERR_MAXIMUMLINESEARCH,
    LBFGSERR_MAXIMUMITERATION,
    LBFGSERR_WIDTHTOOSMALL,
    LBFGSERR_INVALIDPARAMETERS,
    LBFGSERR_INCREASEGRADIENT,
};

typedef double (*lbfgs_eval_fn)(void *instance, const double *x, double *g, const int n);
typedef int (*lbfgs_progress_fn)(void *instance, const double *x, const int k);

struct LbfgsResult {
    double f = 0.0;
    int iterations = 0;
    int evaluations = 0;
    int status = 0;
};

// What the machine asks of its caller after lbfgs_begin / lbfgs_step.
enum LbfgsAsk {
    LBFGS_DONE = 0,      // finished: LbfgsMachine::R holds the result, x the returned iterate
    LBFGS_EVAL = 1,      // evaluate f and g at x; g goes to lbfgs_eval_grad(M, A); then lbfgs_step(.., f, 0)
    LBFGS_PROGRESS = 2,  // after an accepted line search: the progress hook at (x, M.k); then lbfgs_step(.., 0, cancel)
};

// Caller-provided storage of one run on n variables (lbfgs_doubles(P, n) doubles besides x; lbfgs_arrays carves it).
struct LbfgsArrays {
    double *x, *xp, *g, *gp, *d, *gs, *pf, *S, *Y, *ys_hist, *alpha;
};

struct LbfgsMachine {
    int n, next, k, head, stored, restarts, count, ls, bracketed, touched, into_gs;
    double fx, step, fx_before, olddnorm, lo, hi, finit, dgtest, dstest;
    LbfgsResult R;
};

// the comparisons of std::max / std::min (not fmax / fmin, whose NaN rule differs)
SVSDF_HD inline double lbfgs_max(double a, double b) { return a < b ? b : a; }
SVSDF_HD inline int lbfgs_imax(int a, int b) { return a < b ? b : a; }
SVSDF_HD inline int lbfgs_imin(int a, int b) { return b < a ? b : a; }

SVSDF_HD inline size_t lbfgs_doubles(const LbfgsParams &P, int n) {
    // xp, g, gp, d, gs | pf | S, Y | ys_hist, alpha  (P must pass lbfgs_check)
    return (size_t)5 * n + (size_t)lbfgs_imax(1, P.past) + (size_t)2 * P.mem_size * n + (size_t)2 * P.mem_size;
}
SVSDF_HD inline LbfgsArrays lbfgs_arrays(double *x, double *base, const LbfgsParams &P, int n) {
    LbfgsArrays A;
    A.x = x;
    A.xp = base;
    A.g = A.xp + n;
    A.gp = A.g + n;
    A.d = A.gp + n;
    A.gs = A.d + n;
    A.pf = A.gs + n;
    A.S = A.pf + lbfgs_imax(1, P.past);
    A.Y = A.S + (size_t)P.mem_size * n;
    A.ys_hist = A.Y + (size_t)P.mem_size * n;
    A.alpha = A.ys_hist + P.mem_size;
    return A;
}
// where the gradient of the evaluation the machine asks for goes
SVSDF_HD inline double *lbfgs_eval_grad(const LbfgsMachine &M, const LbfgsArrays &A) { return M.into_gs ? A.gs : A.g; }

SVSDF_HD inline int lbfgs_check(const LbfgsParams &P, int n) {
    if (n <= 0) return LBFGSERR_INVALID_N;
    if (P.mem_size <= 0) return LBFGSERR_INVALID_MEMSIZE;
    if (P.g_epsilon < 0.0) return LBFGSERR_INVALID_GEPSILON;
    if (P.past < 0) return LBFGSERR_INVALID_TESTPERIOD;
    if (P.delta < 0.0) return LBFGSERR_INVALID_DELTA;
    if (P.min_step < 0.0) return LBFGSERR_INVALID_MINSTEP;
    if (P.max_step < P.min_step) return LBFGSERR_INVALID_MAXSTEP;
    if (!(P.f_dec_coeff > 0.0 && P.f_dec_coeff < 1.0)) return LBFGSERR_INVALID_FDECCOEFF;
    if (!(P.s_curv_coeff < 1.0 && P.s_curv_coeff > P.f_dec_coeff)) return LBFGSERR_INVALID_SCURVCOEFF;
    if (!(P.machine_prec > 0.0)) return LBFGSERR_INVALID_MACHINEPREC;
    if (P.max_linesearch <= 0) return LBFGSERR_INVALID_MAXLINESEARCH;
    return 0;
}
SVSDF_HD inline double lbfgs_dot(const double *a, const double *b, int n) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += a[i] * b[i];
    return s;
}
SVSDF_HD inline void lbfgs_axpy(double a, const double *x, double *y, int n) {
    for (int i = 0; i < n; ++i) y[i] += a * x[i];
}
SVSDF_HD inline double lbfgs_amax(const double *a, int n) {
    double r = 0.0;
    for (int i = 0; i < n; ++i) r = lbfgs_max(r, std::fabs(a[i]));
    return r;
}

// Starts a run at A.x: checks the parameters, zeroes the storage and asks for the first evaluation (or ends at once with the check's
// code).  The storage must hold lbfgs_doubles(P, n) doubles once the check has passed.
SVSDF_HD inline int lbfgs_begin(const LbfgsParams &P, LbfgsMachine &M, const LbfgsArrays &A, int n) {
    M = LbfgsMachine();
    M.n = n;
    if ((M.R.status = lbfgs_check(P, n)) != 0) return LBFGS_DONE;
    for (double *p = A.xp; p != A.alpha + P.mem_size; ++p) *p = 0.0;
    M.next = 0;
    M.into_gs = 0;
    return LBFGS_EVAL;
}

// Resumes the machine with the value the caller was asked for (f after LBFGS_EVAL, cancel after LBFGS_PROGRESS).
SVSDF_HD inline int lbfgs_step(const LbfgsParams &P, LbfgsMachine &M, const LbfgsArrays &A, double f, int cancel) {
    // resume points (M.next) and internal continuations
    enum { FIRST, LS_EVAL, PROGRESS, STEEPEST_QN, STEEPEST_SKIP, ITERATE, LS_TRY, LS_DONE, DIRECTION, FINISH };
    const int n = M.n, m = P.mem_size;
    double *x = A.x, *xp = A.xp, *g = A.g, *gp = A.gp, *d = A.d;
    int at = M.next;
    for (;;) {
        switch (at) {
            case FIRST:
                M.fx = f;
                M.R.evaluations = 1;
                if (!std::isfinite(M.fx)) {  // a failed first evaluation (NaN cost, g left at zero) must not read as convergence
                    M.R.status = LBFGSERR_INVALID_FUNCVAL;
                    M.R.f = M.fx;
                    return LBFGS_DONE;
                }
                A.pf[0] = M.fx;
                for (int i = 0; i < n; ++i) d[i] = -g[i];
                M.k = 0;
                if (lbfgs_amax(g, n) / lbfgs_max(1.0, lbfgs_amax(x, n)) <= P.g_epsilon) {
                    M.R.status = LBFGS_CONVERGENCE;
                    at = FINISH;
                    break;
                }
                M.step = 1.0 / std::sqrt(lbfgs_dot(d, d, n));
                M.head = M.stored = M.restarts = 0;
                M.olddnorm = 1.0;
                M.k = 1;
                at = ITERATE;
                break;
            case ITERATE: {  // top of the iteration: save the point, then the line search's set-up
                for (int i = 0; i < n; ++i) xp[i] = x[i];
                for (int i = 0; i < n; ++i) gp[i] = g[i];
                M.step = M.step < P.max_step ? M.step : 0.5 * P.max_step;
                M.fx_before = M.fx;
                if (!(M.step > 0.0)) {
                    M.ls = LBFGSERR_INVALIDPARAMETERS;
                    at = LS_DONE;
                    break;
                }
                const double dginit = lbfgs_dot(gp, d, n);
                if (0.0 < dginit) {
                    M.ls = LBFGSERR_INCREASEGRADIENT;
                    at = LS_DONE;
                    break;
                }
                M.finit = M.fx;
                M.dgtest = P.f_dec_coeff * dginit;
                M.dstest = P.s_curv_coeff * dginit;
                M.lo = 0.0;
                M.hi = P.max_step;
                M.bracketed = M.touched = 0;
                M.count = 1;
                at = LS_TRY;
                break;
            }
            case LS_TRY:
                for (int i = 0; i < n; ++i) x[i] = xp[i] + M.step * d[i];
                M.next = LS_EVAL;
                M.into_gs = 0;
                return LBFGS_EVAL;
            case LS_EVAL:  // Lewis–Overton: Armijo + weak Wolfe by bisection / doubling
                M.fx = f;
                ++M.R.evaluations;
                at = LS_DONE;
                if (std::isinf(M.fx) || std::isnan(M.fx)) {
                    M.ls = LBFGSERR_INVALID_FUNCVAL;
                    break;
                }
                if (M.fx > M.finit + M.step * M.dgtest) {
                    M.hi = M.step;
                    M.bracketed = 1;
                } else if (!P.reference_patch && lbfgs_dot(g, d, n) < M.dstest) {
                    M.lo = M.step;
                } else {
                    M.ls = M.count;
                    break;
                }
                if (P.max_linesearch <= M.count) {
                    M.ls = LBFGSERR_MAXIMUMLINESEARCH;
                    break;
                }
                if (M.bracketed && (M.hi - M.lo) < P.machine_prec * M.hi) {
                    M.ls = LBFGSERR_WIDTHTOOSMALL;
                    break;
                }
                M.step = M.bracketed ? 0.5 * (M.lo + M.hi) : M.step * 2.0;
                if (M.step < P.min_step) {
                    M.ls = LBFGSERR_MINIMUMSTEP;
                    break;
                }
                if (M.step > P.max_step) {
                    if (M.touched) {
                        M.ls = LBFGSERR_MAXIMUMSTEP;
                        break;
                    }
                    M.touched = 1;
                    M.step = P.max_step;
                }
                ++M.count;
                at = LS_TRY;
                break;
            case LS_DONE:
                if (M.ls < 0) {
                    for (int i = 0; i < n; ++i) x[i] = xp[i];
                    for (int i = 0; i < n; ++i) g[i] = gp[i];
                    M.fx = M.fx_before;
                    const int ls = M.ls;
                    const bool recoverable = ls == LBFGSERR_MAXIMUMLINESEARCH || ls == LBFGSERR_MINIMUMSTEP || ls == LBFGSERR_WIDTHTOOSMALL ||
                                             ls == LBFGSERR_INCREASEGRADIENT || ls == LBFGSERR_MAXIMUMSTEP;
                    at = FINISH;
                    if (P.nonsmooth_restarts > 0 && recoverable) {
                        if (M.stored > 0 && M.restarts < P.nonsmooth_restarts) {
                            // the quasi-Newton model is wrong across a kink: forget it and search along -g from here
                            ++M.restarts;
                            M.stored = 0;
                            M.head = 0;
                            for (int i = 0; i < n; ++i) d[i] = -g[i];
                            M.step = 1.0 / std::sqrt(lbfgs_dot(d, d, n));
                            at = ITERATE;
                            break;
                        }
                        M.R.status = LBFGS_NOMOREPROGRESS;
                        break;
                    }
                    M.R.status = ls;
                    break;
                }
                M.restarts = 0;
                M.next = PROGRESS;
                return LBFGS_PROGRESS;
            case PROGRESS: {
                at = FINISH;
                if (cancel) { M.R.status = LBFGS_CANCELED; break; }
                if (lbfgs_amax(g, n) / lbfgs_max(1.0, lbfgs_amax(x, n)) < P.g_epsilon) { M.R.status = LBFGS_CONVERGENCE; break; }
                if (P.past > 0) {
                    if (P.past <= M.k) {
                        const double rate = std::fabs(A.pf[M.k % P.past] - M.fx) / lbfgs_max(1.0, std::fabs(M.fx));
                        if (rate < P.delta) { M.R.status = LBFGS_STOP; break; }
                    }
                    A.pf[M.k % P.past] = M.fx;
                }
                if (P.max_iterations != 0 && P.max_iterations <= M.k) { M.R.status = LBFGSERR_MAXIMUMITERATION; break; }
                ++M.k;
                double *s = A.S + (size_t)M.head * n, *y = A.Y + (size_t)M.head * n;
                for (int i = 0; i < n; ++i) { s[i] = x[i] - xp[i]; y[i] = g[i] - gp[i]; }
                const double ys = lbfgs_dot(y, s, n), yy = lbfgs_dot(y, y, n);
                A.ys_hist[M.head] = ys;
                for (int i = 0; i < n; ++i) d[i] = -g[i];
                // cautious update (Li & Fukushima): skip the pair when curvature is too small
                const double cau = lbfgs_dot(s, s, n) * std::sqrt(lbfgs_dot(gp, gp, n)) * P.cautious_factor;
                at = DIRECTION;
                if (ys > cau) {
                    M.stored = lbfgs_imin(m, M.stored + 1);
                    M.head = (M.head + 1) % m;
                    int j = M.head;
                    for (int i = 0; i < M.stored; ++i) {  // two-loop recursion, newest to oldest
                        j = (j + m - 1) % m;
                        A.alpha[j] = lbfgs_dot(A.S + (size_t)j * n, d, n) / A.ys_hist[j];
                        lbfgs_axpy(-A.alpha[j], A.Y + (size_t)j * n, d, n);
                    }
                    const double scale = ys / yy;
                    for (int i = 0; i < n; ++i) d[i] *= scale;
                    for (int i = 0; i < M.stored; ++i) {  // oldest to newest
                        const double beta = lbfgs_dot(A.Y + (size_t)j * n, d, n) / A.ys_hist[j];
                        lbfgs_axpy(A.alpha[j] - beta, A.S + (size_t)j * n, d, n);
                        j = (j + 1) % m;
                    }
                    // (`!(|d| < 0.04)` rather than the reference's `|d| >= 0.04`: a non-finite direction — a stored pair with y.s == 0
                    // once the iterates stop moving — also takes the fallback instead of ending the run with a NaN cost)
                    if (P.reference_patch && (!(std::sqrt(lbfgs_dot(d, d, n)) < 0.04) || lbfgs_dot(d, g, n) > 0)) M.next = STEEPEST_QN;
                    else break;
                } else if (P.reference_patch) {
                    M.next = STEEPEST_SKIP;
                } else {
                    break;
                }
                // the reference's fallback direction: re-evaluate at x (its own callback returns the same gradient again),
                // d = -g / |g| * |d_prev|
                for (int i = 0; i < n; ++i) A.gs[i] = 0.0;
                M.into_gs = 1;
                return LBFGS_EVAL;
            }
            case STEEPEST_QN:
            case STEEPEST_SKIP: {
                ++M.R.evaluations;
                for (int i = 0; i < n; ++i) g[i] = A.gs[i];
                for (int i = 0; i < n; ++i) d[i] = -g[i];
                const double z = lbfgs_dot(d, d, n);
                if (z > 0) {
                    const double nn = std::sqrt(z);
                    for (int i = 0; i < n; ++i) d[i] /= nn;
                }
                for (int i = 0; i < n; ++i) d[i] *= M.olddnorm;
                if (at == STEEPEST_SKIP) M.head = (M.head + 1) % m;  // the slot just written is skipped without counting as stored (lbfgs.hpp:776)
                at = DIRECTION;
                break;
            }
            case DIRECTION:
                if (P.reference_patch) M.olddnorm = std::sqrt(lbfgs_dot(d, d, n));
                M.step = 1.0;
                at = ITERATE;
                break;
            default:  // FINISH
                M.R.f = M.fx;
                M.R.iterations = M.k;
                return LBFGS_DONE;
        }
    }
}

// The host loop around the machine: the caller's callbacks evaluate, and the progress hook runs after every accepted line search.
class Lbfgs {
   public:
    explicit Lbfgs(const LbfgsParams &p) : P(p) {}

    LbfgsResult minimize(double *x, int n, lbfgs_eval_fn eval, void *inst, lbfgs_progress_fn progress, void *puser) {
        LbfgsMachine M;
        LbfgsArrays A{};
        A.x = x;
        if (lbfgs_check(P, n) == 0) {
            store.assign(lbfgs_doubles(P, n), 0.0);
            A = lbfgs_arrays(x, store.data(), P, n);
        }
        for (int ask = lbfgs_begin(P, M, A, n); ask != LBFGS_DONE;) {
            if (ask == LBFGS_EVAL) {
                const double f = eval(inst, x, lbfgs_eval_grad(M, A), n);
                ask = lbfgs_step(P, M, A, f, 0);
            } else {
                ask = lbfgs_step(P, M, A, 0.0, progress && progress(puser, x, M.k) ? 1 : 0);
            }
        }
        return M.R;
    }

   private:
    LbfgsParams P;
    std::vector<double> store;
};

}  // namespace host
}  // namespace svsdf
