// svsdf_types.h — POD types shared by the host runtime and the sm_90a kernels.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SVSDF_HD __host__ __device__
#else
#define SVSDF_HD
#endif

namespace svsdf {

// Shape registry ids. Keys mirror the reference's shapeConstructors map
// (src/swept_volume/include/swept_volume/sw_manager.hpp:187-235); unknown names fall back to the
// rectangle Polygon (sw_manager.hpp:363-372).
enum ShapeId : int {
    SH_STAR = 0,
    SH_HORSESHOE,
    SH_PIE,
    SH_PIE2,
    SH_ARC,
    SH_TUNNEL,
    SH_CUTDISK,
    SH_TRAPEZOID,
    SH_RHOMBUS,
    SH_HEART,
    SH_ROUNDEDX,
    SH_BIGX,
    SH_ROUNDEDCROSS,
    SH_VESICA,
    SH_MOON,
    SH_UNEVENCAPSULE,
    SH_CIRCLE,
    SH_POLYGON,
    SH_MESH,   // triangle-mesh functor, BasicShape::getonlySDF_igl (Shape.hpp:332-340); selected by svsdf_config.mesh_*
    SH_COUNT
};

constexpr int kMaxPolyEdges = 64;
constexpr int kMeshStride = 10;          // doubles per face record: a, b, c, rmax (see ShapeFn<SH_MESH>)
constexpr int kMaxMeshFaces = 1 << 20;  // SH_MESH: faces of the triangle soup
constexpr int kFwnMaxDepth = 24;        // SH_MESH: deepest hierarchy the device traversal's explicit stack holds (svsdf_create checks)
constexpr int kMaxPieces = 64;       // pieces per trajectory supported by the per-warp accumulators
constexpr int kWarpsPerBlock = 8;    // k_outer block = 256 threads
constexpr int kGsipWarps = 22;       // k_gsip block = 704 threads: one warp per ring sample (<= 21 per round)
constexpr double kMaxDuration = 300.0;  // sw_manager.hpp:380: durations >= 300 s are not accepted by updateTraj

// Parameters of the robot-shape SDF functor. Trigonometric constants the reference evaluates on the host
// at construction (cos(20.5), sin(43) ... radians of the literal, Shape.hpp:855,1235,1276,1320) are
// evaluated on the host here too and passed in, so host/device libm differences cannot enter.
struct ShapeParams {
    int id;
    int has_xform;      // 0: trans == 0 and Rotate == I (all shipped yamls) -> pre-transform skipped (bit-exact)
    double trans[2];    // poly_params[0..1]              (Shape.hpp:287)
    double rot[4];      // Rotate(0,0),(0,1),(1,0),(1,1)  (Shape.hpp:288-294)
    double cst[4];      // per-shape host-computed constants (see shape_registry.cpp)
    double radius;      // Circle
    double rout;        // conservative circumradius about the body origin (incl. |trans|): sdf(q) >= |q| - rout for every q.
                        // Lets choiceTInit's layer-1 scan skip lattice samples that provably cannot be the minimum
                        // (thread_choice_t_init).  >= 1e30 disables the pruning (mesh functor).
    double prune_scale, prune_rmin;  // generalisation for functors that are only approximately distances far away (mesh: the float
                        // winding number w scales the distance by 1 - 2w): sdf(q) >= (|q| - rout) / prune_scale for |q| >= prune_rmin.
                        // Analytic shapes: 1 and 0.
    int poly_n;         // Polygon edge count
    int pad_;
    double poly_sx[kMaxPolyEdges], poly_sy[kMaxPolyEdges], poly_ex[kMaxPolyEdges], poly_ey[kMaxPolyEdges];
    const double *mesh_tri;  // SH_MESH: device pointer, kMeshStride doubles per face (a, b, c, rmax), vertices already R v + trans (Shape.hpp:296-302)
    int mesh_nf;
    int fwn_nn;              // SH_MESH: nodes of the 4-way winding-number hierarchy (host/fwn_bvh.hpp), 0 = none
    float fwn_boxmag;        // SH_MESH: >= |every x / y coordinate of the child boxes| (error term of the float box bounds)
    int pad3_;
    // device copies of FwnBvh's arrays: child words [nn][4]; expansion rows [nn][23][4] float (one lane per child); child boxes
    // [nn][4][6] float: lo x, lo y, hi x, hi y rounded OUTWARDS by two ulps (they contain the double vertices), squared z gap to
    // the plane z = 0 rounded down, pad; leaf triangles in float [nf][12]
    const unsigned int *fwn_child;
    const float *fwn_data;
    const float *fwn_cbox;
    const float *fwn_trif;
};

// Deformable robot (svsdf_set_scale; the reference's getScale hook, sw_manager.hpp:495-503): per axis d = x, y
// s_d(t) = a_d + sin(w_d t + phi_d) b_d, s_z = 1.  Passed by value to the scaled kernels only.  An accepted schedule keeps
// every s_d(t) in [kScaleMin, kScaleMax] (svsdf_set_scale).
constexpr double kScaleMin = 1e-6, kScaleMax = 1e6;
struct ScaleSched {
    double a[2], b[2], w[2], phi[2];
};

// Trajectory blob: one contiguous, 16-byte aligned buffer that the kernels pull into shared memory with a
// single TMA bulk copy (cp.async.bulk.shared::cluster.global).  All offsets are in doubles.
//   [0]  header (4 doubles: N, K1, D, reserved)
//   [4]  T[Npad]              piece durations (Npad = N rounded up to even)
//   [..] c[N][3][6]           per piece, per dim (x,y,yaw), ascending powers (== MINCO b rows 6i..6i+5)
//   [..] lat[K1pad]           layer-1 lattice times t_k = 0.15 accumulated k times (host, IEEE adds)
//   [..] pose[4][K1pad]       SoA rows x, y, cos yaw, sin yaw at lat[k] (conflict-free lane-strided reads) —
//                             filled on device by k_pose_table
struct BlobLayout {
    int N, K1;
    int off_T, off_c, off_lat, off_pose, K1pad, total;  // in doubles; total is even (16-byte multiple)
};

SVSDF_HD inline BlobLayout blob_layout(int N, int K1) {
    BlobLayout L;
    L.N = N;
    L.K1 = K1;
    int Npad = (N + 1) & ~1;
    int K1pad = (K1 + 1) & ~1;
    L.off_T = 4;
    L.off_c = L.off_T + Npad;
    L.off_lat = L.off_c + 18 * N;
    L.off_pose = L.off_lat + K1pad;
    L.K1pad = K1pad;
    L.total = L.off_pose + 4 * K1pad;
    L.total = (L.total + 1) & ~1;
    return L;
}

// Pose windows of choiceTInit layers 2 and 3 (k_pose_windows): the samples of a layer-2 window depend only on the layer-1 winner kb
// (seed lat[kb], or 0 for kb = -1), those of a layer-3 window only on (kb, m2), m2 the layer-2 sample that set the minimum (-1: none,
// the seed stays lat[kb]).  Window w holds kWinLen records, sample m at [kWinLen w + m]; the records past a window's last sample
// (t > term) are computed but never read.  Layer 2: window kb + 1, (K1 + 1) windows; layer 3: window kWin3Stride (kb + 1) + m2 + 1.
// One 32-byte record per sample: a lane's read is one sector.
constexpr int kWinLen = 21;
constexpr int kWin3Stride = kWinLen + 1;
struct alignas(32) PoseRec {
    double x, y, c, s;  // position and cos / sin of the yaw
};
SVSDF_HD inline int64_t win2_records(int K1) { return (int64_t)(K1 + 1) * kWinLen; }
SVSDF_HD inline int64_t win3_records(int K1) { return (int64_t)(K1 + 1) * kWin3Stride * kWinLen; }

// Batched k_outer: a warp's batches whose descents share one pass over the CTA's point queue (KernelArgs::outer_chunk).  The host
// takes the largest chunk <= kOuterChunkMax that the launch has rounds for and that leaves the kernel's residency what it is at 1.
constexpr int kOuterChunkMax = 4;
// dynamic shared memory of k_outer in doubles: [ blob | 8 warps x (19N + 1) accumulators | chunk x 8 warps x 32 x 4 work area ]
SVSDF_HD inline size_t outer_smem_doubles(int blob_doubles, int N, int chunk) {
    return (size_t)blob_doubles + (size_t)kWarpsPerBlock * (19 * N + 1) + (size_t)chunk * kWarpsPerBlock * 128;
}
// the dynamic shared memory k_outer / k_gsip opt in to (cudaFuncAttributeMaxDynamicSharedMemorySize); the host refuses larger launches
constexpr int kMaxDynSmemBytes = 200 * 1024;

// Penalty parameters (star.yaml: weight_p 60, safety_hor 0.7; smoothedL1 mu = 0.01 is a literal in the
// reference, back_end_optimizer.hpp:1052)
struct CostParams {
    double weight_p;
    double safety_hor;
};

// Kernel argument block
struct KernelArgs {
    const double *blob;        // trajectory blob (global)
    int blob_doubles;
    const double *points_xy;   // P x 2, packed (x, y)
    int64_t P;
    CostParams cp;
    // per-point outputs (optional, may be null)
    double *out_sdf, *out_tstar, *out_grad;   // grad: P x 3
    int *out_rounds;                           // GSIP rounds per point (0 for outside points)
    // reduction outputs
    double *partials;          // [gridDim.x][19N+1] block partial sums (K1)
    int want_reduce;
    int want_gsip;             // 0: stop after the outer solve (getSDFofSweptVolume semantics)
    int batched;               // k_outer: run choiceTInit / gradient / chain rule one point per lane (large P)
    int outer_chunk;           // batched k_outer: batches per warp that share one descent pass (1 .. kOuterChunkMax; sizes the work area)
    // inside-point bookkeeping
    unsigned char *inside_flag;  // P
    double *inside_tstar;        // P (sparse: written for inside points only)
    int *inside_list;            // compacted, ascending point index
    int *n_inside;               // device scalar
    double *gsip_contrib;        // [n_inside][20]: cost, 18 gdC entries ([d][q]), gdT
    int *gsip_piece;             // [n_inside]
    unsigned long long *eval_counter;  // optional: executed lane-evaluations (profiling builds)
    // pose windows of choiceTInit layers 2 / 3 (k_pose_windows); null: the layer evaluates the trajectory at every sample
    const PoseRec *win2, *win3;
};

// svsdf_cost_grad_multi (svsdf_kernels_multi.cuh): n problems in one set of launches.  The KernelArgs of a multi launch hold the
// BASES of the packed buffers; MultiProblem says where problem k's pieces start.  Each problem keeps the decomposition of its
// single-problem call: its virtual grid `grid` (outer_plan with the single-problem k_outer's occupancy) and its `batched` schedule.
constexpr int kMaxMultiProblems = 65535;  // problems per multi evaluation (k_finalize_multi's grid.y)
struct MultiProblem {
    int64_t blob_off;    // doubles into the packed blobs (even: every blob starts 16-byte aligned, as the TMA load needs)
    int64_t pt_off;      // points into points_xy / inside_tstar / inside_list
    int64_t flag_off;    // bytes into inside_flag (multiple of 16: k_compact's uint4 loads)
    int64_t part_off;    // doubles into partials ([grid][19N + 1])
    int64_t out_off;     // doubles into out / tot ([1 + 19N + 1])
    int64_t P;
    int blob_doubles, N, K1, grid;
};
struct MultiArgs {
    int n;                       // problems
    const MultiProblem *prob;    // [n]
    const int *cta_map;          // [CTAs of the launch][2]: (problem, virtual CTA) of every physical k_outer_multi CTA
    int *ins_count;              // [n] inside points per problem (k_compact_multi)
    int *ins_off;                // [n + 1] exclusive prefix of ins_count: problem k owns inside slots [ins_off[k], ins_off[k + 1])
    unsigned int *compact_ticket;  // k_compact_multi's last-CTA counter (zero between calls)
    unsigned int *tickets;       // [n] k_finalize_multi's per-problem counters (zero between calls)
    double *tot, *out;           // per problem at out_off
};

// K3 (svsdf_extract.cu): query-point extraction from the packed map kernel
constexpr int kMaxWaypoints = 66;   // interior waypoints of <= 64 pieces (+ optional end points)
constexpr int kMaxMapLayers = 64;   // z layers of a 3-D map (svsdf_set_map3d)
constexpr int kMaxKeepout = 160;    // keep-out polyline samples (synthetic scenes only)
struct ExtractArgs {
    const unsigned char *map;  // (X + 2h) x row_bytes, MSB-first bits along y (PCSmap_manager.h:81-108)
    int X, Y, h, row_bytes;
    double ox, oy, res;        // boundary_xyzmin (x, y) and grid resolution
    int W;                     // number of waypoint boxes
    int bx1[kMaxWaypoints], bx2[kMaxWaypoints], by1[kMaxWaypoints], by2[kMaxWaypoints];  // clamped index boxes
    // "OutOfLastOne": the box whose cells waypoint w skips is the box of waypoint w - 1; for w = 0 it is the box around
    // tmp_pos = (999, 999, 999) (plan_manager.cpp:152), i.e. after projInMap the far corner cell of the map
    int px1, px2, py1, py2;
    // one launch handles ONE z layer of the map: act[w] = the layer lies in waypoint w's z range, excl[w] = it lies in the z range
    // of the box waypoint w skips (a skipped cell must be inside the last box in all three dimensions, PCSmap_manager.h:207-209)
    unsigned char act[kMaxWaypoints], excl[kMaxWaypoints];
    int rx1, wy1, nW;          // bounding rectangle: first row, first 32-cell word, words per row
    long long n_items;         // rows * nW
    int n_keepout;
    double clearance;
    double keepout[2 * kMaxKeepout];
};

// The clamped index box of the voxels around a centre c (x, y, z) with half sizes half: corner = c -+ half -> projInMap
// (PCSmap_manager.h:128-135: clamped to [lo, hi], hi = lo + size * res) -> getGridIndex (Gridmap3D.cpp:137-174: floor, clamped to
// the last cell).  idx[a] = {first, last}, both inclusive.  Shared by the query-point extraction (host) and the pose-sampled
// obstacle penalty (device), so both see the same cells.
SVSDF_HD inline void map_index_box(const double c[3], const double half[3], const double lo[3], const double hi[3], const int size[3],
                                   double res, int idx[3][2]) {
    for (int a = 0; a < 3; ++a)
        for (int side = 0; side < 2; ++side) {
            double v = c[a] + (side ? half[a] : -half[a]);
            v = v < lo[a] ? lo[a] : v;
            v = v > hi[a] ? hi[a] : v;
            int i = (int)floor((v - lo[a]) / res);
            i = i < 0 ? 0 : i;
            i = i >= size[a] ? size[a] - 1 : i;
            idx[a][side] = i;
        }
}

// The pose-sampled obstacle penalty (svsdf_set_pose_penalty; the reference's grad_cost_p, back_end_optimizer.hpp:956-1028): one
// record (costp, gradp_x, gradp_y, grad_yaw) per sample j = 0 .. res of every piece, piece-major.  PoseProblem: where a problem's
// trajectory blob starts (doubles into PoseArgs::blobs) and where its N (res + 1) records go (records into PoseArgs::rec).
struct PoseProblem {
    int64_t blob_off, rec_off;
};
struct PoseArgs {
    const unsigned char *map;  // Z layers of (X + 2h) x row_bytes, MSB-first bits along y (svsdf_set_map3d)
    int X, Y, Z, h, row_bytes;
    int64_t layer;             // bytes per layer
    double lo[3], hi[3], res;  // boundary_xyzmin, boundary_xyzmax (lo + size * res) and the voxel edge
    double half[3];            // the gather box's half sizes (bdx / 2, bdy / 2, bdz / 2)
    double safety_hor;
    int res_samples;           // integralIntervs
    int n;                     // problems (grid.y)
    const double *blobs;
    const PoseProblem *prob;   // [n]
    double *rec;               // [..][4]
};

// svsdf_swept_contour[_multi] (svsdf_swept.cu): the narrow-band marching-squares mesher of n problems (n = 1: the single call).
// Problem k owns tiles tile0 .. (the classify / compact CTAs) and whole marching-squares blocks blk0 .. blk0 + nblk - 1; its corners
// start at corner kSweptBlock * blk0 of the concatenation, so one k_sw_scan over the blocks gives every problem its own prefix.
constexpr int kSweptTile = 16;           // classification / compaction tile: 16 x 16 corners, one CTA of 256 threads
constexpr int kSweptMaxSamples = 2112;   // path samples: at most ceil(T_i / 0.15) per piece, D < 300 s, N <= 64
constexpr int kSweptBlock = 1024;        // corners per CTA of the marching-squares passes (256 threads x 4)
struct SweptProblem {
    int64_t i0, j0;
    int nx, ny;
    int tiles_x, nblk;         // tiles per row; marching-squares blocks (ceil(nx ny / kSweptBlock))
    int64_t tile0, blk0;       // first tile, first block
    int samp0, n_samp;         // its samples in SweptArgs::samp
};
struct SweptArgs {
    int n_prob;
    const SweptProblem *prob;  // [n_prob], tile0 and blk0 ascending
    int *stat;                 // [n_prob][8]: [0] non-finite value seen, [1] clipped, [2..6] channel totals, [7] needed corners
    double h, iso;
    const double *samp;        // [..][3]: sample x, y and its reach (a corner farther than reach from every sample is > iso)
    unsigned char *need;       // per corner of the concatenation: corner is evaluated
    double *field;             // per corner
    int *tile_off;             // [tiles + 1] needed corners per tile, then their exclusive prefix (k_sw_scan)
    double *pts;               // [P][2] needed corners (problem by problem, tile-major, row-major in a tile)
    int64_t *idx;              // [P] their corner index in the concatenation
    const double *val;         // [P] their values (the evaluation's output)
    int64_t P;
    int *blk;                  // [5][n_blocks + 1] per-CTA counts of the marching-squares channels, then their prefix
    int *vid;                  // per corner [3]: vertex (local to its problem) of the horizontal edge, the vertical edge and the corner
    double *verts;             // [V][2], problem by problem
    int *segs, *tris;          // [S][2], [F][3], problem by problem; vertex ids local to the problem
    int tiles, n_blocks;       // over all problems
};

// svsdf_map_clearance[_multi] (svsdf_clearance.cu): the occupied map columns near n trajectories.  Problem k covers the words of its
// reach rectangle (the 32-cell words of its rows that hold its columns), one item per word, row-major, padded to whole CTAs of 256
// (cta0[k] ..); a last segment covers the whole map and counts its occupied columns.  The CTA order is problem order, then map order.
struct ClearanceProblem {
    int64_t cta0;              // first CTA
    int64_t n_items;           // rows * nW (0: the rectangle misses the map)
    int i0, wy0, nW;           // first row, first word of a row, words per row
    int all;                   // every occupied column of the rectangle is in the band (d_max = +inf or no far-field bound)
    int samp0, n_samp;         // its samples in ClearanceArgs::samp
    int occ_only;              // the last segment: the whole map, counts the occupied columns, no band
    int pad_;
};
struct ClearanceArgs {
    const unsigned char *map;  // Z layers of (X + 2h) x row_bytes, MSB-first bits along y (svsdf_set_map / svsdf_set_map3d)
    int X, Y, h, row_bytes, Z;
    int64_t layer;             // bytes per layer
    double ox, oy, res;        // boundary_xyzmin (x, y) and grid resolution
    int64_t n_items;           // 256 x the CTAs of all segments
    const double *samp;        // [..][3]: sample x, y and its reach (a centre farther than reach from every sample is > d_max)
    unsigned *band;            // [n_items] band bits of the word (k_cl_count)
    int *blk;                  // [n_blocks + 1] band cells per CTA, then their exclusive prefix (k_sw_scan)
    unsigned long long *n_occ; // occupied columns of the map
    int *ij;                   // [P][2] band cells, problem by problem, each in map order: (i, j)
    double *pts;               // [P][2] their centres
    int n_prob;                // problems + 1 (the occupied-column segment)
    const ClearanceProblem *prob;
};

// K5 (svsdf_frontend.cu): collision kernels of the A* front end
constexpr int kMaxYawKernels = 64;
constexpr int kMaxKernelSize = 32;  // kernel rows are held as 32-bit masks
struct FrontParams {
    int kernel_size, kernel_count;
    double res, safemargin;      // kernelresu (occupancy_resolution), max(front_end_safeh, res / 2)
    int X, Y, h, row_bytes;      // map (svsdf_set_map)
    int out_words;               // 32-cell words per output row: ceil(Y / 32)
    double ox, oy, map_res;      // boundary_xyzmin (x, y) and grid resolution of the map
};
// k_expand_nodes: sample parameters of checkSubSWCollision (kt = 0, 0.02, ... accumulated on the host, <= 1)
struct SubSwParams {
    int nkt;
    double half_box;             // kernel_size / 2 + 1 (integer division), world units (front_end_Astar.hpp:224)
    double kt[64];
};
// k_astar_search: n whole searches (svsdf_front_astar_device)
struct AstarArgs {
    int n, max_path;
    int64_t max_expansions;
    const int *cells;          // [n][4] start x, y, goal x, y cell indices (16-byte aligned); start x = -1: start or goal outside the map
    unsigned char *pool;       // one slot per CTA, slot_bytes each (16-byte aligned): heap, g, f, yaw, father, id — NS + 1 entries each
    int64_t slot_bytes;
    int *next;                 // search counter, zero at launch
    double *paths;             // [n][max_path][3]
    int *len, *expansions, *status;  // [n] each
};

}  // namespace svsdf
