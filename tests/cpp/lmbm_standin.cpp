// A stand-in for the reference's prebuilt LMBM library (not redistributed): the same entry point, lmbm::lmbm_optimize with the
// signature of lmbm.h:214-221, and the same property that makes svsdf_lmbm_open load PRIVATE COPIES — the callback, its
// instance and the iterate live in file-scope statics (lmbm.cpp:4-6 keeps its callback that way), so two runs sharing one loaded
// instance would overwrite each other.  The method is a plain descent along -g with a halving step (deterministic, no threads);
// tests/test_capi_host.py and tests/test_gpu_lmbm.py build it to exercise the plug-in without the reference's binary.
//
//     g++ -O2 -std=c++17 -shared -fPIC tests/cpp/lmbm_standin.cpp -o liblmbm_standin.so
#include <cmath>
#include <vector>

namespace lmbm {
struct lmbm_parameter_t {  // lmbm.h:15-174, member order and types (svsdf_lmbm_params mirrors it)
    float timeout;
    int bundle_size, ini_corrections, max_corrections, exponent_distmeasure, max_iterations, max_evaluations, past, verbose,
        update_method, scaling_strategy;
    double delta_past, f_rel_eps, f_lower_bound, terminate_param1, terminate_param2, distance_measure, sufficient_dec, max_stepsize;
};
typedef double (*lmbm_evaluate_t)(void *instance, const double *x, double *g, const int n);
typedef int (*lmbm_progress_t)(void *instance, const double *x, const int k);

static lmbm_evaluate_t s_eval = nullptr;
static void *s_instance = nullptr;
static int s_n = 0;
static std::vector<double> s_x, s_g, s_trial, s_gtrial;

static double evaluate(const std::vector<double> &x, std::vector<double> &g) { return s_eval(s_instance, x.data(), g.data(), s_n); }

// 0: iteration or evaluation budget used up, 2: the step fell below terminate_param1 without a decrease, -1: cancelled by progress
int lmbm_optimize(int n, double *x, double *fx, lmbm_evaluate_t eval, void *instance, lmbm_progress_t progress, lmbm_parameter_t *param) {
    if (n <= 0 || !x || !fx || !eval || !param) return -3;
    s_eval = eval;
    s_instance = instance;
    s_n = n;
    s_x.assign(x, x + n);
    s_g.assign(n, 0.0);
    s_trial.assign(n, 0.0);
    s_gtrial.assign(n, 0.0);
    double f = evaluate(s_x, s_g);
    int evals = 1, ret = 0;
    double step = param->max_stepsize;
    for (int k = 1; k <= param->max_iterations && evals < param->max_evaluations; ++k) {
        if (progress && progress(s_instance, s_x.data(), k) != 0) { ret = -1; break; }
        double gn = 0.0;
        for (int i = 0; i < n; ++i) gn += s_g[i] * s_g[i];
        gn = std::sqrt(gn);
        if (!(gn > 0.0)) break;
        bool moved = false;
        while (evals < param->max_evaluations && step > param->terminate_param1) {
            for (int i = 0; i < n; ++i) s_trial[i] = s_x[i] - step * s_g[i] / gn;
            const double ft = evaluate(s_trial, s_gtrial);
            ++evals;
            if (ft < f) {
                f = ft;
                s_x.swap(s_trial);
                s_g.swap(s_gtrial);
                step *= 2.0;
                moved = true;
                break;
            }
            step *= 0.5;
        }
        if (!moved) {
            if (!(step > param->terminate_param1)) ret = 2;
            break;
        }
    }
    for (int i = 0; i < n; ++i) x[i] = s_x[i];
    *fx = f;
    return ret;
}
}  // namespace lmbm
