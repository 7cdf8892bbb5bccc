// C entry points of the swept-volume contour checker (oracle/swept_oracle.hpp) for ctypes (oracle/swept_py.py).
#include <cstring>

#include "swept_oracle.hpp"

extern "C" {
// Contours the dense field; returns a handle holding the result (release with sw_free).  sizes_out: V, S, F, clipped.
void *sw_contour(const double *field, int64_t i0, int64_t j0, int nx, int ny, double h, double iso, int64_t *sizes_out) {
    auto *M = new oracle::SweptMesh(oracle::swept_contour(field, i0, j0, nx, ny, h, iso));
    sizes_out[0] = (int64_t)(M->verts.size() / 2);
    sizes_out[1] = (int64_t)(M->segs.size() / 2);
    sizes_out[2] = (int64_t)(M->tris.size() / 3);
    sizes_out[3] = M->clipped;
    return M;
}
void sw_copy(void *handle, double *verts, int32_t *segs, int32_t *tris) {
    const auto *M = static_cast<oracle::SweptMesh *>(handle);
    if (!M->verts.empty()) std::memcpy(verts, M->verts.data(), M->verts.size() * sizeof(double));
    if (!M->segs.empty()) std::memcpy(segs, M->segs.data(), M->segs.size() * sizeof(int32_t));
    if (!M->tris.empty()) std::memcpy(tris, M->tris.data(), M->tris.size() * sizeof(int32_t));
}
void sw_free(void *handle) { delete static_cast<oracle::SweptMesh *>(handle); }
}
