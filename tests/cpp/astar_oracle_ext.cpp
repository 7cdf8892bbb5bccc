// Test-side extension of the CPU oracle's A* (oracle/frontend_oracle.hpp astar_search), built by tests/astar_oracle_ext.py into a
// temporary directory:
//   * ext_astar runs the oracle's own astar_search with an expansion budget (its max_expansions argument) for n start/goal pairs;
//   * with counts_out it also runs an instrumented copy of the same search loop that counts, per search, the branches that set the
//     reference's A* apart from a textbook one: closed nodes re-opened, open nodes improved without re-keying, and pops whose key ties
//     the next key of the open list (decided by insertion order).  The copy must reproduce the oracle's path and expansion count; the
//     return value is the number of searches where it does not.
#include <cstring>
#include <iterator>
#include <map>
#include <vector>

#include "../../oracle/frontend_oracle.hpp"

using namespace oracle;

namespace {

struct Counts {
    int reopened = 0, improved_open = 0, tie_pops = 0;
};

// astar_search (frontend_oracle.hpp) line for line, plus the three counters
AstarResult counted_search(const Shape &S, const ShapeKernels &K, const FrontMap &M, const MapGeom &G, const double start[2],
                           const double goal[2], int max_expansions, Counts &C) {
    AstarResult R;
    const double xmax = G.ox + M.X * G.res, ymax = G.oy + M.Y * G.res;
    auto in_map = [&](const double p[2]) { return !(p[0] < G.ox || p[1] < G.oy || p[0] > xmax || p[1] > ymax); };
    if (!in_map(start) || !in_map(goal)) return R;
    const int sx = grid_index_1d(start[0], G.ox, G.res, M.X), sy = grid_index_1d(start[1], G.oy, G.res, M.Y);
    const int gx = grid_index_1d(goal[0], G.ox, G.res, M.X), gy = grid_index_1d(goal[1], G.oy, G.res, M.Y);
    struct Node { int id = 0; double g = 0, f = 0, yaw = 0; int father = -1; };
    const int NS = M.X * M.Y;
    std::vector<Node> nodes((size_t)NS + 1);
    auto slot_xy = [&](int s, int &x, int &y) { if (s == NS) { x = sx; y = sy; } else { x = s / M.Y; y = s % M.Y; } };
    std::multimap<double, int> open;
    Node &st = nodes[NS];
    st.g = 0; st.f = astar_heuristic(sx, sy, gx, gy); st.id = 1; st.yaw = 0.0;
    open.insert({st.f, NS});
    nodes[(size_t)sx * M.Y + sy].id = 1; nodes[(size_t)sx * M.Y + sy].g = st.g; nodes[(size_t)sx * M.Y + sy].f = st.f;
    while (!open.empty()) {
        auto it = open.begin();
        const int cur = it->second;
        if (std::next(it) != open.end() && std::next(it)->first == it->first) C.tie_pops++;
        open.erase(it);
        nodes[cur].id = -1;
        int cx, cy_;
        slot_xy(cur, cx, cy_);
        if (cx == gx && cy_ == gy) {
            R.success = true;
            std::vector<int> chain;
            int p = cur;
            while (nodes[p].father != -1) { chain.push_back(p); p = nodes[p].father; }
            chain.push_back(p);
            for (auto q = chain.rbegin(); q != chain.rend(); ++q) {
                int x, y;
                slot_xy(*q, x, y);
                R.path.push_back((x + 0.5) * G.res + G.ox);
                R.path.push_back((y + 0.5) * G.res + G.oy);
                R.path.push_back(nodes[*q].yaw);
            }
            return R;
        }
        if (R.expansions >= max_expansions) return R;
        R.expansions++;
        uint8_t ok[9], parts[9];
        double cyaw[9];
        expand_node(S, K, M, G, cx, cy_, nodes[cur].yaw, K.kernel_size, ok, cyaw, parts);
        int n = 0;
        for (int i = -1; i < 2; i++)
            for (int j = -1; j < 2; j++, n++) {
                if (!ok[n]) continue;
                const int nx = cx + i, ny = cy_ + j, ns = nx * M.Y + ny;
                Node &nb = nodes[ns];
                if (nb.id == 0) nb.yaw = cyaw[n];
                const double ec = std::sqrt((double)(i * i + j * j));
                const double tg = ec + nodes[cur].g;
                if (nb.id == 0) {
                    nb.father = cur; nb.g = tg; nb.f = tg + astar_heuristic(nx, ny, gx, gy) + 0.0; nb.id = 1;
                    open.insert({nb.f, ns});
                } else if (nb.id == 1) {
                    if (tg < nb.g) { nb.father = cur; nb.g = tg; nb.f = tg + astar_heuristic(nx, ny, gx, gy) + 0.0; C.improved_open++; }
                } else {
                    if (tg < nb.g) {
                        nb.father = cur; nb.g = tg; nb.f = tg + astar_heuristic(nx, ny, gx, gy) + 0.0; nb.id = 1;
                        open.insert({nb.f, ns});
                        C.reopened++;
                    }
                }
            }
    }
    return R;
}

}  // namespace

extern "C" {

// path_out [n][max_path][3], len_out [n] (0 = no path or longer than max_path), exp_out [n]; counts_out [n][3] may be NULL
int ext_astar(const char *name, const double *poly_params, int ks, int K, double safeh, const uint8_t *occ, int X, int Y, double ox, double oy,
              double map_res, int n, const double *start_xy, const double *goal_xy, int max_path, int max_expansions, double *path_out,
              int *len_out, int *exp_out, int *counts_out) {
    Shape S;
    S.id = shape_id_from_name(name);
    S.set_poly_params(poly_params[0], poly_params[1], poly_params[2]);
    ShapeKernels SK = init_shape_kernels(S, ks, K, map_res, safeh);
    FrontMap M;
    M.build(occ, X, Y, ks);
    MapGeom G;
    G.ox = ox; G.oy = oy; G.res = map_res;
    int differ = 0;
#pragma omp parallel for schedule(dynamic) reduction(+ : differ)
    for (int q = 0; q < n; ++q) {
        AstarResult R = astar_search(S, SK, M, G, start_xy + 2 * q, goal_xy + 2 * q, max_expansions);
        const int len = (int)(R.path.size() / 3);
        len_out[q] = (R.success && len <= max_path) ? len : 0;
        exp_out[q] = R.expansions;
        if (len_out[q]) std::memcpy(path_out + (size_t)q * max_path * 3, R.path.data(), R.path.size() * sizeof(double));
        if (counts_out) {
            Counts C;
            AstarResult Rc = counted_search(S, SK, M, G, start_xy + 2 * q, goal_xy + 2 * q, max_expansions, C);
            if (Rc.success != R.success || Rc.expansions != R.expansions || Rc.path != R.path) differ++;
            counts_out[3 * q] = C.reopened; counts_out[3 * q + 1] = C.improved_open; counts_out[3 * q + 2] = C.tie_pops;
        }
    }
    return differ;
}

}  // extern "C"
