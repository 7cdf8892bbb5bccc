// host/lockstep.hpp — the round driver of the lock-step back end (svsdf_optimize_lockstep).  CUDA-free, so it is tested on the CPU
// with a batched evaluator of its own (tests/cpp/lockstep_driver_main.cpp).
//
// Up to M problems are in flight, each an L-BFGS machine (host/lbfgs.hpp) in a slot, and the calling thread advances them round by
// round.  Before each round, in ascending slot order, a problem whose machine is done leaves and a free slot takes the next problem in
// index order, whose first evaluation joins the round being formed.  The ROUND is every slot whose machine asks for an evaluation, in
// ascending slot order, handed to the caller's round function in one call; then every machine in it resumes with its cost.  So every
// round holds every live problem.  There is no progress hook: a machine goes on at once after each accepted line search.
//
// Each problem's evaluations are the same whichever problems share its rounds, so what a problem computes depends neither on M nor on
// the problems beside it.
#pragma once
#include <cstdint>
#include <vector>

#include "lbfgs.hpp"

namespace svsdf {
namespace host {

// How problem k enters: the n variables it starts from (minimised in place) and its solver parameters.
struct LockstepEntry {
    double *x;
    int n;
    LbfgsParams P;
};

// One evaluation of a round: the round function evaluates at x, writes the gradient to g and the cost to f.
struct LockstepEval {
    int slot;
    const double *x;
    double *g;
    double f;
};

// Runs problems 0 .. n-1, at most M at a time; returns the number of rounds.
//   enter(slot, k) -> LockstepEntry       problem k takes the slot
//   round(std::vector<LockstepEval> &)    evaluates the round
//   leave(slot, k, const LbfgsResult &)   problem k's machine is done; its iterate is at its entry's x
// enter and leave run on the calling thread in slot order.  The machines resume across OpenMP threads, one slot per iteration.
template <class Enter, class Round, class Leave>
int64_t lockstep_run(int n, int M, Enter &&enter, Round &&round, Leave &&leave) {
    struct Slot {
        int k = -1;  // the problem in the slot; -1: none
        int ask = LBFGS_DONE;
        LbfgsParams P;
        LbfgsMachine m;
        LbfgsArrays A{};
        std::vector<double> store;
    };
    std::vector<Slot> slots(M);
    std::vector<LockstepEval> evals;
    int next = 0;
    int64_t rounds = 0;
    for (;;) {
        evals.clear();
        for (int s = 0; s < M; ++s) {
            Slot &sl = slots[s];
            while (sl.ask == LBFGS_DONE) {
                if (sl.k >= 0) leave(s, sl.k, sl.m.R);
                sl.k = -1;
                if (next == n) break;
                sl.k = next++;
                const LockstepEntry e = enter(s, sl.k);
                sl.P = e.P;
                sl.A = LbfgsArrays{};
                sl.A.x = e.x;
                if (lbfgs_check(e.P, e.n) == 0) {  // otherwise lbfgs_begin ends at once without touching the storage
                    sl.store.assign(lbfgs_doubles(e.P, e.n), 0.0);
                    sl.A = lbfgs_arrays(e.x, sl.store.data(), e.P, e.n);
                }
                sl.ask = lbfgs_begin(sl.P, sl.m, sl.A, e.n);
            }
            if (sl.ask == LBFGS_EVAL) evals.push_back(LockstepEval{s, sl.A.x, lbfgs_eval_grad(sl.m, sl.A), 0.0});
        }
        if (evals.empty()) return rounds;
        round(evals);
        ++rounds;
        const int count = (int)evals.size();
#pragma omp parallel for schedule(dynamic)
        for (int j = 0; j < count; ++j) {
            Slot &sl = slots[evals[j].slot];
            int ask = lbfgs_step(sl.P, sl.m, sl.A, evals[j].f, 0);
            while (ask == LBFGS_PROGRESS) ask = lbfgs_step(sl.P, sl.m, sl.A, 0.0, 0);
            sl.ask = ask;
        }
    }
}

}  // namespace host
}  // namespace svsdf
