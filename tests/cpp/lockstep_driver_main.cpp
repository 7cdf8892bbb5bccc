// Test driver of host/lockstep.hpp (tests/test_lockstep_driver.py): n seeded L-BFGS minimisations, run either one after the other with a
// direct callback ("alone") or in lock-step through lockstep_run with a CPU batched evaluator in place of svsdf_optimize_lockstep's
// device round.  Prints one line per problem (the bits of the result) and a summary line.
//
//   lockstep_driver_main alone <n> <seed>
//   lockstep_driver_main lockstep <n> <seed> <max_in_flight>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "lbfgs.hpp"
#include "lockstep.hpp"

using namespace svsdf::host;

struct Fn {  // f(x) = sum_i a_i (x_i - c_i)^2 + s sin(x_0 x_1) [+ k sum_i |x_i - c_i|]  (kinked when k > 0)
    int d;
    std::vector<double> a, c;
    double s, k;
    int max_it;
    std::vector<double> x0;
};

static Fn make_fn(int idx, unsigned seed) {
    std::mt19937_64 r(seed * 1000003u + idx);
    std::uniform_real_distribution<double> u(0.0, 1.0);
    Fn f;
    f.d = 2 + (int)(r() % 7);
    for (int i = 0; i < f.d; ++i) {
        f.a.push_back(0.5 + 4.0 * u(r));
        f.c.push_back(4.0 * u(r) - 2.0);
        f.x0.push_back(6.0 * u(r) - 3.0);
    }
    f.s = 0.3 * u(r);
    f.k = (idx % 3 == 2) ? 0.2 + u(r) : 0.0;
    f.max_it = (idx % 4 == 1) ? 3 + (int)(r() % 5) : 0;  // some stop at max_iterations, the others converge
    return f;
}

static double eval_fn(const Fn &f, const double *x, double *g) {
    double v = 0.0;
    for (int i = 0; i < f.d; ++i) {
        const double e = x[i] - f.c[i];
        v += f.a[i] * e * e + f.k * std::fabs(e);
        g[i] = 2.0 * f.a[i] * e + f.k * (e > 0 ? 1.0 : (e < 0 ? -1.0 : 0.0));
    }
    v += f.s * std::sin(x[0] * x[1]);
    g[0] += f.s * std::cos(x[0] * x[1]) * x[1];
    g[1] += f.s * std::cos(x[0] * x[1]) * x[0];
    return v;
}

static LbfgsParams params_of(const Fn &f) {
    LbfgsParams p;
    p.mem_size = 6;
    p.g_epsilon = 1e-10;
    p.max_iterations = f.max_it;
    p.nonsmooth_restarts = 8;
    return p;
}

static void print_result(int k, const Fn &f, const std::vector<double> &x, const LbfgsResult &R) {
    std::printf("P %d %d %d %d", k, R.status, R.iterations, R.evaluations);
    uint64_t b;
    std::memcpy(&b, &R.f, 8);
    std::printf(" %016llx", (unsigned long long)b);
    for (int i = 0; i < f.d; ++i) {
        std::memcpy(&b, &x[i], 8);
        std::printf(" %016llx", (unsigned long long)b);
    }
    std::printf("\n");
}

int main(int argc, char **argv) {
    if (argc < 4) return 2;
    const bool lock = std::strcmp(argv[1], "lockstep") == 0;
    const int n = std::atoi(argv[2]);
    const unsigned seed = (unsigned)std::atoi(argv[3]);
    std::vector<Fn> fns;
    for (int k = 0; k < n; ++k) fns.push_back(make_fn(k, seed));
    std::vector<std::vector<double>> xs(n);
    std::vector<LbfgsResult> res(n);
    int64_t rounds = 0, violations = 0;
    if (!lock) {
        for (int k = 0; k < n; ++k) {
            xs[k] = fns[k].x0;
            Lbfgs L(params_of(fns[k]));
            res[k] = L.minimize(xs[k].data(), fns[k].d, [](void *inst, const double *x, double *g, const int) { return eval_fn(*(const Fn *)inst, x, g); },
                                (void *)&fns[k], nullptr, nullptr);
        }
    } else {
        const int M = std::min(n, std::max(1, std::atoi(argv[4])));
        std::vector<const Fn *> in_slot(M);
        int finished = 0;
        auto enter = [&](int s, int k) {
            xs[k] = fns[k].x0;
            in_slot[s] = &fns[k];
            return LockstepEntry{xs[k].data(), fns[k].d, params_of(fns[k])};
        };
        // The batched evaluator checks that a round holds every live problem: with every slot taking the next problem as soon as it is
        // done, the live problems are min(M, n - finished) (finished counts problems that have left).
        auto round = [&](std::vector<LockstepEval> &evals) {
            if ((int)evals.size() != std::min(M, n - finished)) ++violations;
            for (LockstepEval &e : evals) e.f = eval_fn(*in_slot[e.slot], e.x, e.g);
        };
        auto leave = [&](int, int k, const LbfgsResult &R) {
            res[k] = R;
            ++finished;
        };
        rounds = lockstep_run(n, M, enter, round, leave);
    }
    for (int k = 0; k < n; ++k) print_result(k, fns[k], xs[k], res[k]);
    std::printf("S %lld %lld\n", (long long)rounds, (long long)violations);
    return 0;
}
