// oracle/ref_path_scaled_shim.cpp — TEST INFRASTRUCTURE: the reference's own source of the hot path with its `useScale` switch on
// (sw_manager.hpp:17) and getScale = this project's schedule.  oracle/ref_extract_scale.py prepares oracle/_ref/scaled/ (a copy of
// ref_path_shim.cpp next to the edited fragments); this file compiles that copy and adds the schedule's C entry points.
// The scaled getStateOnTrajStamp(t, xt, Rt, St) asserts `time_stamp > traj_duration`, an inverted condition: inert only because
// the build defines NDEBUG (oracle/Makefile).
#include "_ref/scaled/ref_path_shim.cpp"

extern "C" {
int ref_scaled() { return useScale ? 1 : 0; }
// sched = a_x, a_y, b_x, b_y, w_x, w_y, phi_x, phi_y
void ref_set_scale(void *h, const double *sched) {
    SweptVolumeManager &sv = ((RefCtx *)h)->sv;
    for (int d = 0; d < 2; ++d) {
        sv.sc_a[d] = sched[d]; sv.sc_b[d] = sched[2 + d]; sv.sc_w[d] = sched[4 + d]; sv.sc_phi[d] = sched[6 + d];
    }
}
}  // extern "C"
