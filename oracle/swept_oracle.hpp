// swept_oracle.hpp — CPU restatement of the svsdf_swept_contour contract (include/svsdf.h): marching squares over a dense field,
// one literal loop per output kind.  The checker of csrc/svsdf_swept.cu; it knows nothing of the narrow band: a NaN corner is
// "not evaluated" (never inside, its edges never cross, its cells are skipped), which is how the band's output reads.
// Build with -ffp-contract=off: every vertex coordinate is p_a + s (p_b - p_a) with s = (iso - f_a) / (f_b - f_a), rounded per operation.
#pragma once
#include <cmath>
#include <cstdint>
#include <vector>

namespace oracle {

struct SweptMesh {
    std::vector<double> verts;      // [V][2]
    std::vector<int32_t> segs;      // [S][2]
    std::vector<int32_t> tris;      // [F][3]
    int clipped = 0;
};

// Walk items of a cell: c0 (a, b), e0 (edge c0c1), c1 (a + 1, b), e1 (c1c2), c2 (a + 1, b + 1), e2 (c3c2), c3 (a, b + 1), e3 (c0c3).
enum { C0 = 0, E0, C1, E1, C2, E2, C3, E3 };
struct CasePolys {
    int n;
    int len[2];
    int item[2][6];
};
// case = in(c0) | in(c1) << 1 | in(c2) << 2 | in(c3) << 3; kSaddleSplit: cases 5 and 10 when the inside corners are not connected
static const CasePolys kCases[16] = {
    {0, {0, 0}, {{0}, {0}}},
    {1, {3, 0}, {{C0, E0, E3}, {0}}},
    {1, {3, 0}, {{E0, C1, E1}, {0}}},
    {1, {4, 0}, {{C0, C1, E1, E3}, {0}}},
    {1, {3, 0}, {{E1, C2, E2}, {0}}},
    {1, {6, 0}, {{C0, E0, E1, C2, E2, E3}, {0}}},
    {1, {4, 0}, {{E0, C1, C2, E2}, {0}}},
    {1, {5, 0}, {{C0, C1, C2, E2, E3}, {0}}},
    {1, {3, 0}, {{E2, C3, E3}, {0}}},
    {1, {4, 0}, {{C0, E0, E2, C3}, {0}}},
    {1, {6, 0}, {{E0, C1, E1, E2, C3, E3}, {0}}},
    {1, {5, 0}, {{C0, C1, E1, E2, C3}, {0}}},
    {1, {4, 0}, {{E1, C2, C3, E3}, {0}}},
    {1, {5, 0}, {{C0, E0, E1, C2, C3}, {0}}},
    {1, {5, 0}, {{E0, C1, C2, C3, E3}, {0}}},
    {1, {4, 0}, {{C0, C1, C2, C3}, {0}}},
};
static const CasePolys kSaddleSplit5 = {2, {3, 3}, {{C0, E0, E3}, {E1, C2, E2}}};
static const CasePolys kSaddleSplit10 = {2, {3, 3}, {{E0, C1, E1}, {E2, C3, E3}}};

// field: ny rows of nx values, corner (i0 + a, j0 + b) at field[b nx + a], position (fl((i0 + a) h), fl((j0 + b) h))
inline SweptMesh swept_contour(const double *field, int64_t i0, int64_t j0, int nx, int ny, double h, double iso) {
    SweptMesh M;
    const int64_t n = (int64_t)nx * ny;
    auto F = [&](int a, int b) { return field[(int64_t)b * nx + a]; };
    auto X = [&](int a) { return (double)(i0 + a) * h; };
    auto Y = [&](int b) { return (double)(j0 + b) * h; };
    auto ev = [&](int a, int b) { return !std::isnan(F(a, b)); };
    auto in = [&](int a, int b) { return F(a, b) <= iso; };
    std::vector<int32_t> idH(n, -1), idV(n, -1), idC(n, -1);
    int32_t V = 0;
    auto vertex = [&](double xa, double ya, double fa, double xb, double yb, double fb) {
        const double s = (iso - fa) / (fb - fa);
        M.verts.push_back(xa + s * (xb - xa));
        M.verts.push_back(ya + s * (yb - ya));
        return V++;
    };
    // 1. crossings of horizontal edges (a, b) - (a + 1, b), row-major
    for (int b = 0; b < ny; ++b)
        for (int a = 0; a + 1 < nx; ++a)
            if (ev(a, b) && ev(a + 1, b) && in(a, b) != in(a + 1, b))
                idH[(int64_t)b * nx + a] = vertex(X(a), Y(b), F(a, b), X(a + 1), Y(b), F(a + 1, b));
    // 2. crossings of vertical edges (a, b) - (a, b + 1), row-major
    for (int b = 0; b + 1 < ny; ++b)
        for (int a = 0; a < nx; ++a)
            if (ev(a, b) && ev(a, b + 1) && in(a, b) != in(a, b + 1))
                idV[(int64_t)b * nx + a] = vertex(X(a), Y(b), F(a, b), X(a), Y(b + 1), F(a, b + 1));
    // 3. inside corners, row-major; one on the border clips
    for (int b = 0; b < ny; ++b)
        for (int a = 0; a < nx; ++a)
            if (ev(a, b) && in(a, b)) {
                idC[(int64_t)b * nx + a] = V++;
                M.verts.push_back(X(a));
                M.verts.push_back(Y(b));
                if (a == 0 || b == 0 || a == nx - 1 || b == ny - 1) M.clipped = 1;
            }
    // 4. cells, row-major: segments (inside on the left) and fan triangles of each inside polygon
    for (int b = 0; b + 1 < ny; ++b)
        for (int a = 0; a + 1 < nx; ++a) {
            if (!(ev(a, b) && ev(a + 1, b) && ev(a + 1, b + 1) && ev(a, b + 1))) continue;
            const int cas = (int)in(a, b) | (int)in(a + 1, b) << 1 | (int)in(a + 1, b + 1) << 2 | (int)in(a, b + 1) << 3;
            const double m = ((F(a, b) + F(a + 1, b)) + (F(a, b + 1) + F(a + 1, b + 1))) * 0.25;
            const CasePolys *P = &kCases[cas];
            if (cas == 5 && !(m <= iso)) P = &kSaddleSplit5;
            if (cas == 10 && !(m <= iso)) P = &kSaddleSplit10;
            const int64_t c = (int64_t)b * nx + a;
            const int32_t id[8] = {idC[c], idH[c], idC[c + 1], idV[c + 1], idC[c + nx + 1], idH[c + nx], idC[c + nx], idV[c]};
            for (int p = 0; p < P->n; ++p) {
                const int L = P->len[p];
                const int *it = P->item[p];
                for (int k = 0; k < L; ++k)
                    if ((it[k] & 1) && (it[(k + 1) % L] & 1)) {
                        M.segs.push_back(id[it[k]]);
                        M.segs.push_back(id[it[(k + 1) % L]]);
                    }
                for (int k = 1; k + 1 < L; ++k) {
                    M.tris.push_back(id[it[0]]);
                    M.tris.push_back(id[it[k]]);
                    M.tris.push_back(id[it[k + 1]]);
                }
            }
        }
    return M;
}

}  // namespace oracle
