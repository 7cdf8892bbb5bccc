// svsdf_backend.h — the device back end of svsdf_optimize_device (svsdf_backend.cu): the L-BFGS machine (host/lbfgs.hpp) and the MINCO
// evaluation halves (host/minco.hpp) of every problem in flight, one warp per problem, on device-resident state.
#pragma once
#include <cuda_runtime.h>

#include "host/lbfgs.hpp"
#include "host/minco.hpp"
#include "svsdf_types.h"

namespace svsdf {

// A problem of the call (uploaded once at the start): where its outputs live in the result block and its boundary conditions.
struct BackendProblem {
    int N;
    int pad_;
    int64_t res_off;             // doubles into BackendArgs::res: x (4N - 3, x0 on entry, the iterate in flight), T (N), coeffs (18N)
    double initS[9], finalS[9];  // 3x3 column-major
};
// A problem's scalar results (written when its machine finishes; f0 at its first successful evaluation)
struct BackendResult {
    double f0, f;
    int iterations, evaluations, solver_status, status;  // status: svsdf_optimize's return (solver status, or the last evaluation's error)
    int f0_set, pad_;
};
// One slot: the machine of the problem in it and the state between its evaluations
struct BackendSlot {
    host::LbfgsMachine M;
    int problem;      // the problem in the slot
    int last_status;  // error of its last evaluation (0: none)
    int good_evals;   // successful evaluations so far
    int pad_;
    double energy;    // MINCO energy of the trajectory in flight
};
// What the host reads of every slot each round
struct BackendStatus {
    int ask;          // LBFGS_EVAL: the slot takes part in the next round; LBFGS_DONE: its problem has finished
    int valid;        // the trajectory passes traj_layout's checks (every T > 0 and finite, D < 300 s)
    int K1, N;
    double D;
    int64_t n_inside; // interior points of its last evaluation
};
// A slot's part in a round (uploaded with the round's problem table): its record at out_off, or rc != 0 (the evaluation failed)
struct BackendRoundItem {
    int slot, rc;
    int64_t out_off;  // doubles into the round's records
    int64_t blob_off; // doubles into the round's blobs
    int64_t pose_off; // records into BackendArgs::pose_rec (the pose penalty's, when it is on)
};
struct BackendArgs {
    host::LbfgsParams P;
    double rho;
    host::DynamicsParams dyn;     // the context's speed and yaw-rate limits (svsdf_set_dynamics), used when dyn_on
    int dyn_on;
    int pose_on;                  // the context's pose penalty (svsdf_set_pose_penalty): its parameters and the round's sample records
    host::PoseParams pose;
    const double *pose_rec;
    int Nmax;
    int64_t slot_doubles;
    BackendSlot *slots;
    double *mem;                  // [slots][slot_doubles]: lbfgs storage, boundary, MINCO and the evaluation halves' arrays
    BackendStatus *status;        // [slots]
    const BackendProblem *prob;   // [problems]
    BackendResult *result;        // [problems]
    double *res;                  // the result block
};

// Doubles of one slot's storage for trajectories of up to Nmax pieces.
inline int64_t backend_slot_doubles(const host::LbfgsParams &P, int Nmax) {
    const int nv = 4 * Nmax - 3;
    // lbfgs | head, tail | band | b | t | times, gradByTimes, partialGradByTimes | partialGradByCoeffs | gradByPoints | adj | dynPartial
    return (int64_t)host::lbfgs_doubles(P, nv) + 18 + (int64_t)host::minco_band_doubles(Nmax) + 18 * Nmax + 5 * Nmax + 3 * Nmax +
           18 * Nmax + 3 * (Nmax - 1) + 18 * Nmax + Nmax;
}

// launchers (svsdf_backend.cu).  init: problems enter slots (pairs [slot, problem]); blob: the round's blobs; backward: the round's
// records into the machines.  Each leaves every slot it touched asking for an evaluation (status filled) or finished.
cudaError_t launch_backend_init(const BackendArgs &B, const int *slot_problem, int count, cudaStream_t st);
cudaError_t launch_backend_blob(const BackendArgs &B, const BackendRoundItem *items, int count, double *blobs, cudaStream_t st);
cudaError_t launch_backend_backward(const BackendArgs &B, const BackendRoundItem *items, int count, const double *records, cudaStream_t st);

}  // namespace svsdf
