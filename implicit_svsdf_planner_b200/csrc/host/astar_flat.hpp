// host/astar_flat.hpp — the per-search bookkeeping of the A* front end WITHOUT containers: flat arrays and a binary heap, written so
// that the same code compiles for the device (SVSDF_HD).  k_astar_search (csrc/svsdf_frontend.cu, svsdf_front_astar_device) runs it in
// thread 0 of one CTA per search, with its arrays and heap in global memory and the node test spread over the CTA's warps: no host
// round trip per expansion (DESIGN.md §7 rank 3 (vi); the lock-step host version of (v) pays a launch, two copies and the host's
// open-list pass per round).  The same code is also checked on the host: tests/cpp/astar_host_main.cpp runs it beside host/astar.hpp
// and the oracle's literal AstarPathSearch and requires identical paths and expansion counts.
//
// Same semantics as host/astar.hpp (AstarPathSearcher::AstarPathSearch / getPath, front_end_Astar.hpp:243-390):
//   * node states 0 unseen / 1 open / -1 closed, yaw fixed when a node is first seen, open nodes improved in place WITHOUT re-keying,
//     closed nodes re-opened when improved, a start-node object (slot NS) separate from the grid node of the start cell;
//   * the open list is a std::multimap<double, node> there: begin() is the smallest key and equal keys leave in insertion order.  Here:
//     a binary min-heap ordered by (f, sequence number of the insertion) — the same total order.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define SVSDF_HD __host__ __device__
#else
#define SVSDF_HD
#endif

namespace svsdf {
namespace host {

struct FlatHeapEntry {
    double f;
    uint32_t seq;
    int32_t slot;
};

// Storage of ONE search, provided by the caller (device: a slice of a global-memory pool):
//   id [NS + 1] int8, g / f / yaw [NS + 1] double, father [NS + 1] int32 (NS = X * Y, slot NS = the start-node object), heap [heap_cap].
struct FlatSearch {
    int X, Y, NS;
    int sx, sy, gx, gy;
    int8_t *id;
    double *g, *f, *yaw;
    int32_t *father;
    FlatHeapEntry *heap;
    int heap_n, heap_cap;
    uint32_t seq;
    int cur;
    int64_t expansions;
    int status;  // 0 running, 1 path found (cur = goal slot), 2 open list empty, 3 expansion limit, -1 heap overflow

    // Only id[] has to be cleared between searches (and father[] of slots a path can reach is written when they are first
    // opened): g / f / yaw / father of a slot are written when its id goes from 0 to 1 and read only while it is non-zero.  The
    // start cell's grid slot is marked open without a father; it is never pushed (nothing improves g = 0), so never popped and
    // never a father.

    SVSDF_HD static double heuristic(int ax, int ay, int bx, int by) {  // getHeu (front_end_Astar.hpp:165-183), dz = 0
        const double p = 1.0 / 1000;
        int dx = ax - bx, dy = ay - by;
        dx = dx < 0 ? -dx : dx;
        dy = dy < 0 ? -dy : dy;
        const int dz = 0;
        const int dmin = dx < dy ? (dx < dz ? dx : dz) : (dy < dz ? dy : dz);
        const int dmax = dx > dy ? (dx > dz ? dx : dz) : (dy > dz ? dy : dz);
        const int dmid = dx + dy + dz - dmin - dmax;
        const double h = sqrt(3.0) * dmin + sqrt(2.0) * (dmid - dmin) + (dmax - dmid);
        return h * (1 + p);
    }
    SVSDF_HD static bool before(const FlatHeapEntry &a, const FlatHeapEntry &b) { return a.f < b.f || (a.f == b.f && a.seq < b.seq); }
    SVSDF_HD bool push(double key, int slot) {
        if (heap_n >= heap_cap) { status = -1; return false; }
        FlatHeapEntry e{key, seq++, slot};
        int i = heap_n++;
        while (i > 0) {
            const int p = (i - 1) >> 1;
            if (!before(e, heap[p])) break;
            heap[i] = heap[p];
            i = p;
        }
        heap[i] = e;
        return true;
    }
    SVSDF_HD FlatHeapEntry pop() {
        const FlatHeapEntry top = heap[0];
        const FlatHeapEntry last = heap[--heap_n];
        int i = 0;
        for (;;) {
            int c = 2 * i + 1;
            if (c >= heap_n) break;
            if (c + 1 < heap_n && before(heap[c + 1], heap[c])) ++c;
            if (!before(heap[c], last)) break;
            heap[i] = heap[c];
            i = c;
        }
        if (heap_n > 0) heap[i] = last;
        return top;
    }
    SVSDF_HD void slot_xy(int s, int &x, int &y) const {
        if (s == NS) { x = sx; y = sy; } else { x = s / Y; y = s % Y; }
    }
    // AstarPathSearch up to the first pop (:243-300).  The caller has zeroed id[].
    SVSDF_HD void begin(int sx_, int sy_, int gx_, int gy_) {
        sx = sx_; sy = sy_; gx = gx_; gy = gy_;
        heap_n = 0; seq = 0; cur = -1; expansions = 0; status = 0;
        g[NS] = 0; f[NS] = heuristic(sx, sy, gx, gy); id[NS] = 1; yaw[NS] = 0.0; father[NS] = -1;
        push(f[NS], NS);
        const int c = sx * Y + sy;
        id[c] = 1; g[c] = g[NS]; f[c] = f[NS];
    }
    // One iteration of the main loop up to the neighbour expansion: pops the best open node.  Returns true when `cur` has to be
    // expanded (its cell and yaw go to the node test); false when the search has ended (status says how).
    SVSDF_HD bool pop_next(int64_t max_expansions, int &cx, int &cy, double &cyaw) {
        if (status != 0) return false;
        if (heap_n == 0) { status = 2; return false; }
        const FlatHeapEntry e = pop();
        cur = e.slot;
        id[cur] = -1;
        slot_xy(cur, cx, cy);
        if (cx == gx && cy == gy) { status = 1; return false; }
        if (expansions >= max_expansions) { status = 3; return false; }
        ++expansions;
        cyaw = yaw[cur];
        return true;
    }
    // AstarGetSucc's bookkeeping (:192-240) for the node popped last: ok9 / yaw9 = the node test's answer for its 9 cells (di-major)
    SVSDF_HD void apply(int cx, int cy, const unsigned char *ok9, const double *yaw9) {
        const double gcur = g[cur];
        int k = 0;
        for (int i = -1; i < 2; i++)
            for (int j = -1; j < 2; j++, k++) {
                if (!ok9[k]) continue;
                const int nx = cx + i, ny = cy + j, ns = nx * Y + ny;
                if (id[ns] == 0) yaw[ns] = yaw9[k];
                const double ec = sqrt((double)(i * i + j * j));
                const double tg = ec + gcur;
                if (id[ns] == 0) {
                    father[ns] = cur; g[ns] = tg; f[ns] = tg + heuristic(nx, ny, gx, gy) + 0.0; id[ns] = 1;
                    if (!push(f[ns], ns)) return;
                } else if (id[ns] == 1) {
                    if (tg < g[ns]) { father[ns] = cur; g[ns] = tg; f[ns] = tg + heuristic(nx, ny, gx, gy) + 0.0; }
                } else if (tg < g[ns]) {
                    father[ns] = cur; g[ns] = tg; f[ns] = tg + heuristic(nx, ny, gx, gy) + 0.0; id[ns] = 1;
                    if (!push(f[ns], ns)) return;
                }
            }
    }
    // getPath (:370-390): number of nodes from the start to `cur`; out (optional, capacity max_path): (x, y, yaw) per node, start first.
    // Both walks stop after NS + 1 nodes (there are only NS + 1 slots); a longer father chain returns -1.  A valid search has none:
    // edge costs are positive and the self-neighbour never improves g, so father pointers cannot form a cycle.
    SVSDF_HD int path(double ox, double oy, double res, int max_path, double *out) const {
        int n = 1;
        for (int s = cur; father[s] != -1; s = father[s])
            if (++n > NS + 1) return -1;
        if (n > max_path || !out) return n;
        int s = cur;
        for (int k = n - 1; k >= 0; --k) {
            int x, y;
            slot_xy(s, x, y);
            out[3 * k] = (x + 0.5) * res + ox;  // getGridCubeCenter
            out[3 * k + 1] = (y + 0.5) * res + oy;
            out[3 * k + 2] = yaw[s];
            s = father[s];
        }
        return n;
    }
};

}  // namespace host
}  // namespace svsdf
