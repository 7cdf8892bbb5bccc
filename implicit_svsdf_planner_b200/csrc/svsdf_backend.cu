// svsdf_backend.cu — the device back end of svsdf_optimize_device: every problem in flight keeps its L-BFGS machine, MINCO and the
// halves of its evaluation in device memory, and one warp per problem runs the host's own code on them (host/lbfgs.hpp on
// lane 0, host/minco.hpp's BackendEvalView with the warp's lanes sharing independent rows, right-hand sides and pieces), in the host's order.  Built with -fmad=false, as the host unit is built with -ffp-contract=off:
// no contraction on either side, correctly rounded division and sqrt on both, so every problem gets svsdf_optimize's bits.
//   k_backend_init:     problems enter slots; the machine starts and asks for its first evaluation
//   k_backend_blob:     the round's trajectory blobs, byte for byte fill_blob's (the layer-1 lattice accumulated on one thread)
//   k_backend_backward: the round's records (and the pose and dynamics penalties, when they are on) through MINCO's adjoint into the
//                       machines, which ask for the next evaluation or finish
// Asking for an evaluation runs its forward half (tau -> T, MINCO, energy, partial gradients) and traj_layout's checks at once.
#include <cmath>

#include "svsdf_backend.h"

namespace svsdf {
namespace {

struct SlotView {
    host::LbfgsArrays L;
    host::BackendEvalView E;
    int N;
};

__device__ SlotView carve(const BackendArgs &B, int s) {
    const BackendProblem &pr = B.prob[B.slots[s].problem];
    const int N = pr.N, nv = 4 * N - 3;
    double *p = B.mem + (int64_t)s * B.slot_doubles;
    SlotView V;
    V.N = N;
    V.L = host::lbfgs_arrays(B.res + pr.res_off, p, B.P, nv);
    p += host::lbfgs_doubles(B.P, nv);
    double *head = p, *tail = p + 9;
    p += 18;
    V.E.m.N = N;
    V.E.m.head = head;
    V.E.m.tail = tail;
    V.E.m.A = p;
    p += host::minco_band_doubles(N);
    V.E.m.b = p;
    p += 18 * N;
    V.E.m.t = p;
    p += 5 * N;
    V.E.times = p;
    V.E.gradByTimes = p + N;
    V.E.partialGradByTimes = p + 2 * N;
    p += 3 * N;
    V.E.partialGradByCoeffs = p;
    p += 18 * N;
    V.E.gradByPoints = p;
    p += 3 * (N - 1);
    V.E.adj = p;
    p += 18 * N;
    V.E.dynPartial = p;
    return V;
}

// a problem's warp: its lanes share the independent work of MINCO and the evaluation halves (host/minco.hpp's Team)
struct WarpTeam {
    int l;
    __device__ int lane() const { return l; }
    __device__ int size() const { return 32; }
    __device__ void sync() const { __syncwarp(); }
};

// the forward half of the evaluation the machine asks for, and traj_layout's checks and lattice count (svsdf_runtime_eval.cpp)
__device__ void ask_evaluation(const BackendArgs &B, int s, const SlotView &V, const WarpTeam &team) {
    const double energy = host::backend_forward(V.E, V.L.x, team);
    if (team.lane() != 0) return;
    B.slots[s].energy = energy;
    BackendStatus &st = B.status[s];
    int valid = 1;
    double D = 0.0;
    for (int i = 0; i < V.N; ++i) {
        const double T = V.E.times[i];
        if (!(T > 0.0) || !isfinite(T)) {
            valid = 0;
            break;
        }
        D += T;
    }
    if (valid && !(D < kMaxDuration)) valid = 0;
    int K1 = 0;
    if (valid)
        for (double t = 0.0; t <= D; t += 0.15) K1++;
    st.ask = host::LBFGS_EVAL;
    st.valid = valid;
    st.K1 = K1;
    st.N = V.N;
    st.D = D;
}

// HostEval::finish and svsdf_optimize_lockstep's status rule
__device__ void finish(const BackendArgs &B, int s, const SlotView &V, const WarpTeam &team) {
    const BackendSlot &sl = B.slots[s];
    const BackendProblem &pr = B.prob[sl.problem];
    const int N = V.N;
    for (int i = team.lane(); i < N; i += team.size()) V.E.times[i] = host::forwardT(V.L.x[i]);
    team.sync();
    host::minco_set_parameters(V.E.m, V.L.x + N, V.E.times, team);
    double *T_out = B.res + pr.res_off + 4 * N - 3, *c_out = T_out + N;
    for (int i = team.lane(); i < N; i += team.size()) T_out[i] = V.E.times[i];
    for (int e = team.lane(); e < 18 * N; e += team.size()) c_out[e] = V.E.m.b[e];
    if (team.lane() != 0) return;
    BackendResult &r = B.result[sl.problem];
    r.f = sl.M.R.f;
    r.iterations = sl.M.R.iterations;
    r.evaluations = sl.M.R.evaluations;
    r.solver_status = sl.M.R.status;
    r.status = sl.last_status != 0 ? sl.last_status : (sl.M.R.status == 0 ? 1 : sl.M.R.status);
    B.status[s].ask = host::LBFGS_DONE;
}

// ask: lane 0's machine request.  The machine runs on lane 0 (its dot products are sequential sums); the others wait for its x.
__device__ void advance(const BackendArgs &B, int s, const SlotView &V, int ask, const WarpTeam &team) {
    if (team.lane() == 0)
        while (ask == host::LBFGS_PROGRESS) ask = host::lbfgs_step(B.P, B.slots[s].M, V.L, 0.0, 0);  // no progress hook on the device
    ask = __shfl_sync(0xffffffffu, ask, 0);
    team.sync();
    if (ask == host::LBFGS_EVAL) ask_evaluation(B, s, V, team);
    else finish(B, s, V, team);
}

// one warp per problem, kBackendWarps problems per CTA
constexpr int kBackendWarps = 4;

__global__ void __launch_bounds__(kBackendWarps * 32) k_backend_init(const BackendArgs B, const int *slot_problem, int count) {
    const int j = blockIdx.x * kBackendWarps + threadIdx.x / 32;
    if (j >= count) return;
    const WarpTeam team{(int)(threadIdx.x & 31)};
    const int s = slot_problem[2 * j];
    BackendSlot &sl = B.slots[s];
    if (team.lane() == 0) {
        sl.problem = slot_problem[2 * j + 1];
        sl.last_status = 0;
        sl.good_evals = 0;
        B.status[s].n_inside = 0;
    }
    team.sync();
    const SlotView V = carve(B, s);
    const BackendProblem &pr = B.prob[sl.problem];
    int ask = 0;
    if (team.lane() == 0) {
        for (int e = 0; e < 9; ++e) {
            const_cast<double *>(V.E.m.head)[e] = pr.initS[e];
            const_cast<double *>(V.E.m.tail)[e] = pr.finalS[e];
        }
        B.result[sl.problem].f0_set = 0;
        ask = host::lbfgs_begin(B.P, sl.M, V.L, 4 * V.N - 3);
    }
    advance(B, s, V, ask, team);
}

// one CTA per round item: header, T, coefficients [piece][dim][power], zeros; thread 0 the lattice `for (t = 0; t <= D; t += 0.15)`
__global__ void k_backend_blob(const BackendArgs B, const BackendRoundItem *items, double *blobs) {
    const BackendRoundItem it = items[blockIdx.x];
    if (it.rc != 0) return;
    const SlotView V = carve(B, it.slot);
    const BackendStatus st = B.status[it.slot];
    const int N = V.N;
    const BlobLayout L = blob_layout(N, st.K1);
    double *h = blobs + it.blob_off;
    for (int e = threadIdx.x; e < L.off_pose; e += blockDim.x) {
        if (e >= L.off_lat && e < L.off_lat + L.K1) continue;
        double v = 0.0;
        if (e == 0) v = (double)N;
        else if (e == 1) v = (double)L.K1;
        else if (e == 2) v = st.D;
        else if (e >= L.off_T && e < L.off_T + N) v = V.E.times[e - L.off_T];
        else if (e >= L.off_c && e < L.off_c + 18 * N) {
            const int q = e - L.off_c, i = q / 18, d = (q % 18) / 6, k = q % 6;
            v = V.E.m.b[d * 6 * N + 6 * i + k];
        }
        h[e] = v;
    }
    if (threadIdx.x == 0) {
        int k = 0;
        for (double t = 0.0; t <= st.D; t += 0.15) h[L.off_lat + k++] = t;
    }
}

// (kBackendWarps * 32, 1): lets ptxas hold the machine and the dynamics penalty in registers (162, no spills; three CTAs per SM)
__global__ void __launch_bounds__(kBackendWarps * 32, 1) k_backend_backward(const BackendArgs B, const BackendRoundItem *items, int count,
                                                                         const double *records) {
    const int j = blockIdx.x * kBackendWarps + threadIdx.x / 32;
    if (j >= count) return;
    const WarpTeam team{(int)(threadIdx.x & 31)};
    const BackendRoundItem it = items[j];
    const int s = it.slot;
    BackendSlot &sl = B.slots[s];
    const SlotView V = carve(B, s);
    double f;
    if (it.rc == 0) {
        const double *o = records + it.out_off;
        double pos = 0.0, other = 0.0;
        const double *pose_rec = B.pose_on ? B.pose_rec + 4 * it.pose_off : nullptr;
        f = host::backend_backward(V.E, sl.energy, o, V.L.x, B.rho, B.pose_on ? &B.pose : nullptr, pose_rec, B.dyn_on ? &B.dyn : nullptr,
                                   host::lbfgs_eval_grad(sl.M, V.L), &pos, &other, team);
        if (team.lane() == 0) {
            if (sl.good_evals++ == 0) {
                B.result[sl.problem].f0 = f;
                B.result[sl.problem].f0_set = 1;
            }
            sl.last_status = 0;
            B.status[s].n_inside = (int64_t)o[1 + 19 * V.N];
        }
    } else {
        if (team.lane() == 0) sl.last_status = it.rc;
        f = __longlong_as_double(0x7ff8000000000000LL);  // the host's NAN
    }
    int ask = 0;
    if (team.lane() == 0) ask = host::lbfgs_step(B.P, sl.M, V.L, f, 0);
    advance(B, s, V, ask, team);
}

}  // namespace

cudaError_t launch_backend_init(const BackendArgs &B, const int *slot_problem, int count, cudaStream_t st) {
    if (count <= 0) return cudaSuccess;
    k_backend_init<<<(count + kBackendWarps - 1) / kBackendWarps, kBackendWarps * 32, 0, st>>>(B, slot_problem, count);
    return cudaGetLastError();
}
cudaError_t launch_backend_blob(const BackendArgs &B, const BackendRoundItem *items, int count, double *blobs, cudaStream_t st) {
    if (count <= 0) return cudaSuccess;
    k_backend_blob<<<count, 128, 0, st>>>(B, items, blobs);
    return cudaGetLastError();
}
cudaError_t launch_backend_backward(const BackendArgs &B, const BackendRoundItem *items, int count, const double *records, cudaStream_t st) {
    if (count <= 0) return cudaSuccess;
    k_backend_backward<<<(count + kBackendWarps - 1) / kBackendWarps, kBackendWarps * 32, 0, st>>>(B, items, count, records);
    return cudaGetLastError();
}

}  // namespace svsdf
