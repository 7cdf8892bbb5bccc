// host::pose_penalty (csrc/host/minco.hpp) behind a C entry point, for tests/test_oracle_pose_penalty.py: the chain rule every back end
// applies to the pose penalty's sample records, compiled as the runtime unit is compiled (no contraction).
#include "host/minco.hpp"

extern "C" double pose_chain(double weight, int res, int N, const double *T, const double *b, const double *rec, double *gradC,
                             double *gradT, double *partial) {
    svsdf::host::PoseParams p;
    p.weight = weight;
    p.res = res;
    return svsdf::host::pose_penalty(p, N, T, b, rec, gradC, gradT, partial);
}
