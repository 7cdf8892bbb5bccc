/* svsdf.h — C ABI of libsvsdf_b200.so: the H100-native drop-in for the SVSDF collision cost + gradient path of
 * ZJU-FAST-Lab/Implicit-SVSDF-Planner.  Plain pointers and sizes only; no C++/torch types cross this boundary.
 * All matrices use the reference's memory layouts (Eigen default column-major) so a maintainer can pass
 * `.data()` of the existing Eigen objects (see INTEGRATION.md for the binding stubs).
 *
 * Reference interfaces replaced (paths relative to the reference project's src/):
 *   R1  TrajOptimizer::addSaftyPenaOnSweptVolumeParallelTrueSDF(void*, const VectorXd& T, const MatrixX3d& coeffs,
 *         double& cost, VectorXd& gradT, MatrixX3d& gradC)
 *         planner_algorithm/include/planner_algorithm/back_end_optimizer.hpp:774-869      -> svsdf_cost_grad
 *   R2  SweptVolumeManager::getTrueSDFofSweptVolume<true>(pos_eva, time_seed_f, grad_prel, set_ts)
 *         swept_volume/include/swept_volume/sw_manager.hpp:916-1018                        -> svsdf_query
 *       SweptVolumeManager::getSDFofSweptVolume<false,true>  sw_manager.hpp:844-866         -> svsdf_query (outer_only=1)
 *       SweptVolumeManager::updateTraj                      sw_manager.hpp:376-385         -> svsdf_set_traj
 *   R3  TrajOptimizer::costFunctionLmbmParallel(void*, const double* x, double* g, int n)
 *         back_end_optimizer.hpp:344-408; callback type lmbm_evaluate_t utils/include/utils/lmbm.h:206-209
 *                                                                                          -> svsdf_evaluate
 *   R4  TrajOptimizer::optimize_traj_lmbm(initS, finalS, opt_x, N, traj)
 *         planner_algorithm/src/back_end_optimizer.cpp:3-97 (outer solver on the host)     -> svsdf_optimize
 *   R5  shape::BasicShape::getonlySDF / getonlyGrad1 and the shapeConstructors registry
 *         utils/include/utils/Shape.hpp:266-270, sw_manager.hpp:187-235,350-373            -> svsdf_shape_sdf/_grad1
 *   R6  TrajOptimizer::setParam / parallel_points / parallel_points_num
 *         back_end_optimizer.hpp:877-932, plan_manager/src/plan_manager.cpp:168-175         -> svsdf_create/_set_points
 *   R7  MINCO_S3NU::setConditions, setParameters, getEnergy..., propogateGrad utils/include/utils/minco.hpp:397-655
 *                                                                                          -> svsdf_minco_*
 *
 * Threading: a context is not thread-safe; use one context per CUDA stream / GPU (the reference has the same
 * restriction: one optimisation per TrajOptimizer instance, back_end_optimizer.hpp:344-408 mutates members).
 * Errors: every int-returning function returns SVSDF_OK (0) or a negative svsdf_status; no exceptions cross
 * the ABI.  The library has no CPU fallback: without a usable CUDA device svsdf_create fails with
 * SVSDF_ERR_CUDA.
 */
#ifndef SVSDF_H_
#define SVSDF_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct svsdf_ctx svsdf_ctx;

typedef enum {
    SVSDF_OK = 0,
    SVSDF_ERR_INVALID = -1,   /* bad argument (null pointer, N out of range, duration >= 300 s, ...) */
    SVSDF_ERR_CUDA = -2,      /* CUDA runtime error or no device; see svsdf_last_error */
    SVSDF_ERR_NOT_READY = -3, /* points / boundary conditions not set */
    SVSDF_ERR_NONFINITE = -4  /* cost or gradient became NaN/Inf */
} svsdf_status;

/* Mirrors the subset of `struct Config` (utils/include/utils/config.hpp) the hot path reads. */
typedef struct {
    const char *shape;        /* registry key = basename of yaml `inputdata` ("star", "sdHorseshoe", ...);
                                 unknown / NULL -> Polygon fallback (rectangle 12 x 0.2 unless polygon_xy given) */
    double poly_params[3];    /* yaml poly_params: body-frame offset x, y and yaw (degrees) of the shape */
    double weight_p;          /* yaml weight_p   (star.yaml: 60.0) */
    double safety_hor;        /* yaml safety_hor (star.yaml: 0.7)  */
    double rho;               /* yaml rho        (star.yaml: 3.8)  */
    int device;               /* CUDA device ordinal */
    int strict_fp;            /* 1 (default): kernels compiled with -fmad=false, bit-compatible with the un-fused
                                 x86-64 arithmetic of the reference; 0: FMA-contracted build (~5-10 % faster, gradient
                                 only within the reference's ~1e-5 contraction noise floor) */
    const double *polygon_xy; /* optional polygon vertices (x0,y0,x1,y1,...) for the fallback shape */
    int polygon_n;            /* number of vertices (<= 64) */
    /* Optional triangle mesh.  When mesh_nf > 0 the robot shape is the reference's mesh functor
       BasicShape::getonlySDF_igl (utils/Shape.hpp:332-340: (1 - 2 * winding number) * distance to the mesh, gradient by
       the same central differences, :35-53) instead of a registry shape; `shape` is then ignored.  poly_params are
       applied to the vertices (R v + trans, Shape.hpp:285-302) at creation; the arrays are copied. */
    const double *mesh_vertices; /* mesh_nv x 3, row-major (x, y, z) */
    int mesh_nv;
    const int32_t *mesh_faces;   /* mesh_nf x 3, 0-based vertex indices */
    int mesh_nf;
} svsdf_config;

/* Fill a config with the reference's star.yaml defaults. */
void svsdf_default_config(svsdf_config *cfg);

int svsdf_create(const svsdf_config *cfg, svsdf_ctx **out);
void svsdf_destroy(svsdf_ctx *ctx);
const char *svsdf_last_error(const svsdf_ctx *ctx);
/* Shape registry lookup: returns the internal id (>= 0); unknown names map to the Polygon fallback id. */
int svsdf_shape_id(const char *name);
/* Radius R (about the body origin, pre-transform included) such that the configured shape functor satisfies
   sdf(q) >= |q| - R for every body-frame point q.  The kernels use it to skip lattice samples of choiceTInit's first layer
   (sw_manager.hpp:538-581) that provably cannot be the minimum; exposed so that the bound can be tested against the oracle
   without a GPU.  Writes a value >= 1e300 when no bound is used (mesh functor).  Host-only, no context needed. */
int svsdf_shape_bound_radius(const svsdf_config *cfg, double *radius_out);
/* Read a Wavefront .obj (what igl::read_triangle_mesh does for yaml `inputdata`, utils/Shape.hpp:284-285): vertices
   (nv x 3 doubles) and fan-triangulated faces (nf x 3, 0-based), malloc'ed; release both with svsdf_free. */
int svsdf_read_obj(const char *path, double **vertices_out, int *nv_out, int32_t **faces_out, int *nf_out);
/* Host-side view of the mesh functor's winding-number hierarchy (csrc/host/fwn_bvh.hpp: the 4-way BVH with order-2
   expansions that igl::fast_winding_number builds, fast_winding_number.cpp:380-457) — for tests and diagnostics, no GPU
   needed.  vertices: nv x 3 doubles as they enter the BVH (shape frame), faces: nf x 3.  Outputs (any may be NULL):
   n_nodes_out; children_out [n_nodes][4] (triangle index | 0x80000000 + node index | 0xffffffff empty; capacity in nodes given by
   node_capacity); data_out [n_nodes][23][4] floats; w_out[n] = winding number at q (n x 3 doubles, float query, accuracy 2.0). */
int svsdf_mesh_fwn_host(const double *vertices, int nv, const int32_t *faces, int nf, int *n_nodes_out, int node_capacity,
                        uint32_t *children_out, float *data_out, int64_t n, const double *q, double *w_out);
void svsdf_free(void *p);

/* R6: parallel_points.  pts: P rows of `stride` doubles (x, y, [z ...]); z is ignored like the reference
 * does (back_end_optimizer.hpp:791).  `pts` is consumed before the call returns (packed into pinned memory by a few host threads, chunk
 * by chunk, each chunk handed to the copy engine at once); the call does not wait for the host -> device transfer itself: whatever is
 * called next on this context runs behind it on the context's stream. */
int svsdf_set_points(svsdf_ctx *ctx, const double *pts, int64_t P, int stride);
/* Same, but the points already live on the device as packed (x, y) pairs; no copy is made of host data. */
int svsdf_set_points_device(svsdf_ctx *ctx, const double *dev_xy, int64_t P);

/* R2: updateTraj.  T: N durations; coeffs: MINCO `b`, 6N x 3 column-major. */
int svsdf_set_traj(svsdf_ctx *ctx, int N, const double *T, const double *coeffs);

/* Deformable robots: the reference's `useScale` switch and its `getScale(t)` hook (sw_manager.hpp:17, :495-503) as a
 * schedule.  Per axis d = x, y: s_d(t) = a_d + sin(w_d t + phi_d) b_d; s_z = 1.  The reference's commented example is
 * a = (0.8, 0.8), b = (0.6, 0.4), w = (1.5, 1.8), phi = (-1.0, 0.0).  Valid: every value finite, a_d - |b_d| >= 1e-6 and
 * a_d + |b_d| <= 1e6 (every s_d(t) in [1e-6, 1e6], so det = sy sx is a normal number and St.inverse() is finite and non-zero;
 * a_d - |b_d| > 0 alone admits a = 1e-160, whose det underflows, and a = 1e160, whose det overflows) and
 * |w_d| * 300 + |phi_d| < 1e6 (the sin argument stays in the range of the fast reduction).  svsdf_scale_matrix applies the
 * same test. */
typedef struct svsdf_scale {
    double a[2], b[2], w[2], phi[2];
} svsdf_scale;
/* NULL: rigid robot (the default).  A schedule turns on the scaled descent, FD gradient and chain rule for every later
 * query, cost and evaluation on this context; the seed scan (choiceTInit) stays rigid as in the reference.  The
 * schedule is copied.  Returns SVSDF_ERR_INVALID (and keeps the previous setting) for an invalid schedule. */
int svsdf_set_scale(svsdf_ctx *ctx, const svsdf_scale *scale);
/* S(t) and St.inverse() as 3x3 column-major matrices, with the arithmetic of the kernels: the pinned sin, Eigen 3.3's
 * size-3 inverse (1/det with det = sy sx; Sinv = diag(sy/det', sx/det', (sx sy)/det') where 1/det' is rounded once).
 * Either output may be NULL.  No context and no GPU needed. */
int svsdf_scale_matrix(const svsdf_scale *scale, double t, double S_out[9], double Sinv_out[9]);

/* ---- Speed and yaw-rate limits: the back end's dynamics penalty ------------------------------------------------------------
 * The yaml's back-end limits (vmax, omgmax, weight_v, weight_omg, smoothingEps, integralIntervs), which the reference reads
 * (back_end_optimizer.hpp:72-79, :884-896) and never penalises: addTimeIntPenalty (:411-533) computes violaVel = |vel_xy|^2 - vmax^2
 * and violaOmg = vel_yaw^2 - omgmax^2, and nothing uses them.  Here the penalty fills the callback's dyn_cost slot (:358, :387):
 *   cost = sum over pieces i and samples j = 0 .. integralIntervs of node step (weight_v smoothedL1(violaVel) + weight_omg
 *          smoothedL1(violaOmg)), node = 1/2 at both ends of a piece, step = T_i / integralIntervs; smoothedL1 as :316-340.
 * The exact arithmetic and summation order are those of host::dynamics_penalty (csrc/host/minco.hpp).  The penalty is soft. */
typedef struct {
    double vmax, omgmax, weight_v, weight_omg, smoothingEps;
    int integralIntervs;
} svsdf_dynamics;
/* star.yaml's values: vmax 10, omgmax 10, weight_v 10, weight_omg 10, smoothingEps 1e-2, integralIntervs 4. */
void svsdf_default_dynamics(svsdf_dynamics *dyn);
/* NULL: no dynamics penalty (the default).  Otherwise every later svsdf_evaluate, svsdf_optimize, svsdf_optimize_batch (each context
 * of the pool with its own setting), svsdf_optimize_lockstep and svsdf_optimize_device of this context adds the penalty after the
 * safety term and before the MINCO adjoint and rho * sum(T); svsdf_last_costs counts it in cost_other.  The limits are copied.
 * Returns SVSDF_ERR_INVALID, and keeps the previous setting, for a non-finite value, vmax or omgmax <= 0, a negative weight,
 * smoothingEps <= 0 or integralIntervs outside 1 .. 64. */
int svsdf_set_dynamics(svsdf_ctx *ctx, const svsdf_dynamics *dyn);
/* The penalty of one trajectory (N >= 1 pieces, T[N], coeffs: MINCO b, 6N x 3 column-major) on the host: writes (not adds) the cost,
 * gradC[18N] (column-major like coeffs) and gradT[N], with the bits both back ends add.  No context and no GPU needed.  Returns
 * SVSDF_ERR_INVALID, writing nothing, for invalid limits (as svsdf_set_dynamics), N < 1 or a NULL pointer. */
int svsdf_dynamics_penalty(const svsdf_dynamics *dyn, int N, const double *T, const double *coeffs, double *cost, double *gradC,
                           double *gradT);

/* ---- Pose-sampled obstacle penalty: the discrete-pose collision cost ---------------------------------------------------------
 * The reference's second collision cost, which it computes and never applies: addTimeIntPenalty (back_end_optimizer.hpp:411-533) calls
 * grad_cost_p (:956-1028) at the samples j = 0 .. integralIntervs of every piece.  At the sample's pose x = (x, y, yaw) it gathers the
 * occupied voxels of the 3-D map in the box x -+ half (getPointsInAABB, PCSmap_manager.h:160-182; the box's z range is centred on the
 * yaw, as in the reference), keeps those whose body-frame offset p_rel = Rz(yaw)^T (c - x) has every |p_rel_a| <= half_a, and sums
 * smoothedL1(safety_hor - sdf(p_rel), 0.01) and its gradient in position and yaw over them.  The per-sample sums are integrated with
 * the trapezoid rule: cost = sum over i, j of node step weight costp_ij, node = 1/2 at both ends of a piece, step = T_i /
 * integralIntervs.  Unlike the SVSDF term, whose query points are fixed when they are set, the voxels are gathered afresh around the
 * trajectory at every evaluation; between samples the body is not seen (a fast trajectory can pass an obstacle unpenalised).  The
 * body is rigid here even under svsdf_set_scale (the reference passes St and never uses it); safety_hor is the context's.  The exact
 * arithmetic and summation order: svsdf_pose.cu (the records) and host::pose_penalty (csrc/host/minco.hpp, the chain rule).
 * Not available for the mesh functor. */
typedef struct {
    double weight;        /* weight_p */
    int integralIntervs;  /* samples j = 0 .. integralIntervs per piece */
    double half[3];       /* the gather box's half sizes: kernel_size * occupancy_resolution / 2 in the reference */
} svsdf_pose_penalty;
/* star.yaml's values: weight 60, integralIntervs 4, half 8.5 on each axis. */
void svsdf_default_pose_penalty(svsdf_pose_penalty *p);
/* NULL: no pose penalty (the default).  Otherwise every later svsdf_evaluate, svsdf_optimize, svsdf_optimize_batch (each context of
 * the pool with its own setting), svsdf_optimize_lockstep and svsdf_optimize_device of this context adds the penalty after the
 * safety term and before the dynamics penalty; svsdf_last_costs counts it in cost_pos.  These calls then need a 3-D map
 * (svsdf_set_map3d) and return SVSDF_ERR_NOT_READY, before any launch, without one.  The values are copied.  Returns
 * SVSDF_ERR_INVALID, and keeps the previous setting, for a non-finite value, weight < 0, integralIntervs outside 1 .. 64, a half
 * size <= 0, or a context of the mesh functor. */
int svsdf_set_pose_penalty(svsdf_ctx *ctx, const svsdf_pose_penalty *p);
/* The penalty p of one trajectory (N pieces as svsdf_cost_grad takes it) against the context's 3-D map and shape, on the device:
 * writes (not adds) the cost, gradC[18N] (column-major like coeffs) and gradT[N], with the bits the back ends add, and, when
 * samples_out is not NULL, the N (integralIntervs + 1) raw sample records (costp, gradp_x, gradp_y, grad_yaw) of grad_cost_p, piece
 * by piece.  p need not be the context's setting.  Returns SVSDF_ERR_INVALID for invalid values or trajectories (refused as
 * svsdf_set_pose_penalty and svsdf_cost_grad refuse them) and SVSDF_ERR_NOT_READY without a 3-D map. */
int svsdf_pose_penalty_eval(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, const svsdf_pose_penalty *p, double *cost,
                            double *gradC, double *gradT, double *samples_out);

/* ---- Swept-volume outline and mesh: the planner's own field contoured on the GPU ---------------------------------------------
 * svsdf_swept_contour meshes the level set f(p) = iso of f = getSDFofSweptVolume<false,true> (exactly what svsdf_query(...,
 * outer_only = 1) returns, bit for bit per point) on the z = 0 plane, for the trajectory (N, T, coeffs) as svsdf_query takes it and
 * with the context's shape, pre-transform, scale schedule and build (strict / fast).  Where the planner's local search misses the
 * global minimum, the outline shows what the planner sees.  No interior (GSIP) branch: inside the volume the outer solve's value
 * (negative there) is what is interpolated.
 *   Grid: corner (i, j) sits at (fl(i h), fl(j h)) (i, j int64, one rounded product, no origin), so grids of different boxes line up.
 *     The box is snapped outwards to this lattice; corners i0 .. i0 + nx - 1, j0 .. j0 + ny - 1; field index (j - j0) nx + (i - i0).
 *     Automatic box (has_box = 0): the trajectory's bounding box padded by the band bound below, so that every corner outside it is
 *     provably > iso and the result is never clipped.  Unavailable (SVSDF_ERR_INVALID) when the shape has no far-field bound
 *     (svsdf_shape_bound_radius >= 1e300).
 *   Inside: f <= iso (the sdf <= 0 convention of the interior flag; iso = 0 is the boundary, iso = safety_hor where the penalty starts).
 *   Vertices: one per crossing edge (exactly one end inside), shared by the cells that own the edge; with a the edge's lower-index
 *     corner s = (iso - f_a) / (f_b - f_a), p = p_a + s (p_b - p_a) per coordinate, every operation rounded once (no contraction), so
 *     the strict and fast builds give the same vertices from the same field.  Inside corners are vertices too.
 *     Order: crossings of horizontal edges (row-major), then of vertical edges, then inside corners (row-major).
 *   Saddles (two diagonal corners inside): m = ((f00 + f10) + (f01 + f11)) * 0.25; m <= iso connects the inside corners.
 *   Segments (2 int32 each, vertex indices) have the inside on their left: outer loops run counter-clockwise, holes clockwise.
 *   Triangles (3 int32, counter-clockwise) fill the inside: per cell each inside polygon (inside corners and crossing vertices walked
 *     counter-clockwise from the lower-left corner) is fan-triangulated from its first vertex.  Segments and triangles come cell by
 *     cell (row-major), within a cell in that walk order.
 *   clipped = 1 when an inside corner lies on the box border (only a user box can do this).  Loops are closed, and the boundary of the
 *     fill equals the segment set, exactly when clipped = 0.
 * Narrow band: only corners of cells that can hold the contour are evaluated (n_evaluated of the box's nx ny).  A cell is skipped only
 * when a bound proves its four corners > iso: f(p) >= min_t |p - x(t)| / s_max - R (R = the shape's far-field radius, s_max the largest
 * scale factor) with x(t) covered by samples x_k and radii delta_k from the velocity coefficients (DESIGN.md §7).  The field of a
 * skipped corner is NaN.  A fixed number of kernel launches per call (none of the evaluation's when no corner is needed); the
 * context's resident points and everything svsdf_cost_grad depends on are left as they were.
 * Errors: SVSDF_ERR_INVALID (nothing allocated) for a non-finite h or h <= 0, a non-finite iso, a non-finite or inverted box, a box over
 * max_corners (0: 2^25; at most 2^28), or a bad trajectory; SVSDF_ERR_NONFINITE when an evaluated corner's value is not finite.
 * The library allocates the output arrays; release them with svsdf_swept_free. */
typedef struct {
    double h;              /* grid spacing (> 0) */
    double iso;            /* level */
    int has_box;           /* 0: automatic box */
    double box[4];         /* xmin, ymin, xmax, ymax (has_box = 1) */
    int64_t max_corners;   /* cap on nx * ny; 0 = 2^25 */
    int want_field;        /* 1: return the field (nx * ny doubles, NaN where not evaluated) */
} svsdf_swept_params;
typedef struct {
    int64_t i0, j0;        /* lattice index of the box's lower-left corner */
    int nx, ny;            /* corners per row / column */
    int64_t n_vertices, n_segments, n_triangles;
    double *vertices;      /* n_vertices x 2 (x, y) */
    int32_t *segments;     /* n_segments x 2 */
    int32_t *triangles;    /* n_triangles x 3 */
    double *field;         /* ny x nx or NULL */
    int clipped;
    int64_t n_evaluated;   /* corners whose field was evaluated */
} svsdf_swept_mesh;
int svsdf_swept_contour(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, const svsdf_swept_params *params,
                        svsdf_swept_mesh *out);
void svsdf_swept_free(svsdf_swept_mesh *mesh);

/* ---- Map clearance: a trajectory checked against every occupied cell of the map ----------------------------------------------
 * svsdf_map_clearance evaluates the swept-volume SDF of the trajectory (N, T, coeffs) at the centre of every occupied map column and lists
 * the cells whose value is <= d_max.  It is the check the reference declares as PlannerManager::getMinSVSDF (plan_manager.hpp:45) and
 * never defines: is the optimised trajectory collision free against the whole map, not only against the back end's query points?
 *   Obstacles: the occupied cells of the context's map (svsdf_set_map, svsdf_set_map_device or svsdf_set_map3d).  A column (i, j) counts
 *     once when any of its z layers is occupied (the back end zeroes z too, so every voxel it would penalise is covered).  Only cells
 *     inside the map count: the map kernel's padding and the outside of the map are NOT obstacles here, unlike the reference's
 *     isOccupied, which treats out-of-range indices as occupied (Gridmap3D.cpp:199-202).
 *   Centre of cell (i, j): ((i + 0.5) res + ox, (j + 0.5) res + oy), rounded as svsdf_extract_points[3d] rounds it, bit for bit.
 *   Value: exactly what svsdf_query(..., outer_only = 0) returns for that centre on this context (getTrueSDFofSweptVolume<true>: the
 *     interior (GSIP) depth where the centre is inside), for every shape, pre-transform, scale schedule and build.
 *   List: every occupied cell with value <= d_max, in ascending i * Y + j order; n_within, n_colliding, min_sdf and argmin are computed
 *     from it (argmin: the first cell in list order among ties; +INFINITY and -1 for an empty list).
 *   d_max: >= 0 or +INFINITY.  Only the cells near the path are evaluated (n_evaluated of n_occupied): a column is skipped only when the
 *     band bound of svsdf_swept_contour with iso = d_max proves its outer value > d_max >= 0, and then that outer value is the answer.
 *     d_max = +INFINITY, or a shape without a far-field bound, evaluates every occupied column.
 * Errors (nothing allocated): SVSDF_ERR_INVALID for a NaN or negative d_max, a bad trajectory or non-finite coefficients;
 * SVSDF_ERR_NOT_READY without a map; SVSDF_ERR_NONFINITE when an evaluated value is not finite.  A fixed number of kernel launches per
 * call, whatever the map size (none of the evaluation's when no column is near the path); the context's resident points,
 * last_n_inside and everything svsdf_cost_grad depends on keep their values.  Release the arrays with svsdf_clearance_free. */
typedef struct {
    int64_t n_occupied;   /* occupied map columns (cells (i, j) with any occupied z layer) */
    int64_t n_evaluated;  /* columns whose value was computed (the band) */
    int64_t n_within;     /* listed cells: value <= d_max */
    int64_t n_colliding;  /* listed cells with value <= 0 */
    double  min_sdf;      /* minimum over the listed cells; +INFINITY when none */
    int64_t argmin;       /* index into the list (first in list order among ties); -1 when none */
    int32_t *ij;          /* n_within x 2: cell index (i, j) */
    double  *xy;          /* n_within x 2: cell centre */
    double  *sdf;         /* n_within */
    double  *tstar;       /* n_within */
} svsdf_clearance;
int svsdf_map_clearance(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, double d_max, svsdf_clearance *out);
void svsdf_clearance_free(svsdf_clearance *c);
/* svsdf_map_clearance_multi: svsdf_map_clearance of n trajectories against the context's map in one set of launches.  out[k] equals
 * svsdf_map_clearance(ctx, N_k, T_k, coeffs_k, d_max, ...) on the same context bit for bit (counts, list and summary), and status_out[k]
 * is the status that call would return (SVSDF_OK or SVSDF_ERR_NONFINITE; a problem whose status is not OK has no arrays allocated).
 *   0 <= n <= 65535; n = 0 does nothing.  The call is refused before any work (SVSDF_ERR_INVALID, nothing allocated) for a bad d_max,
 *   any bad trajectory (N outside 1 .. 64, bad durations, non-finite coefficients), or when the map cells in the 32-cell words of the
 *   problems' reach rectangles number more than 2^31 - 1 together (never for n = 1); SVSDF_ERR_NOT_READY without a map.
 *   Each problem evaluates only the occupied columns of its reach rectangle (the bounding box of its samples' reach, padded outwards):
 *   the band is that of the single call.  The occupied columns of the map are counted once per call.  A fixed number of kernel
 *   launches, whatever n and the map size (none of the evaluation's when no problem has a band); the context's resident points,
 *   last_n_inside and everything svsdf_cost_grad and svsdf_cost_grad_multi depend on keep their values.  Release each out[k] with
 *   svsdf_clearance_free. */
typedef struct {
    int N;
    const double *T;       /* N */
    const double *coeffs;  /* 18 N, column-major 6N x 3 */
} svsdf_clearance_problem;
int svsdf_map_clearance_multi(svsdf_ctx *ctx, int n, const svsdf_clearance_problem *problems, double d_max, svsdf_clearance *out,
                              int *status_out);

/* svsdf_swept_contour_multi: svsdf_swept_contour of n trajectories in one set of launches, with one set of parameters (h, iso,
 * max_corners, want_field and the box: has_box = 1 gives every problem that box, has_box = 0 each its own automatic box).  out[k] is
 * bit for bit svsdf_swept_contour(ctx, N_k, T_k, coeffs_k, params, ...) on the same context (grid, vertices, segments, triangles with
 * problem-local vertex ids, clipped, n_evaluated, field); status_out[k] is the status that call returns, SVSDF_OK or
 * SVSDF_ERR_NONFINITE (then out[k] holds nothing).  Release each out[k] with svsdf_swept_free.
 *   0 <= n <= 65535; n = 0 does nothing.  Refused before any work (SVSDF_ERR_INVALID, nothing allocated) for any parameter or
 *   trajectory the single call refuses, a shape without a far-field bound and no box, or when the problems' grids hold more than
 *   2^31 - 1 corners together (never for n = 1).  The number of kernel launches does not depend on n or the grids (none of the
 *   evaluation's when no problem needs a corner); the host synchronises three times.  The context's resident points, last_n_inside
 *   and everything svsdf_cost_grad and svsdf_cost_grad_multi depend on keep their values. */
int svsdf_swept_contour_multi(svsdf_ctx *ctx, int n, const svsdf_clearance_problem *problems, const svsdf_swept_params *params,
                              svsdf_swept_mesh *out, int *status_out);

/* R2: per-point swept-volume SDF query on the trajectory given by (N, T, coeffs).
 * pts: P x 3 (x, y, z) host doubles (z ignored).  Outputs (host, may be NULL): sdf[P], tstar[P], grad3[3P]
 * (body-frame FD gradient for sdf > 0; world-frame unit direction for the interior branch, exactly what the
 * reference returns), rounds[P] (GSIP rounds, 0 for outside points).  outer_only = 1 stops after
 * getSDFofSweptVolume (no interior branch). */
int svsdf_query(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, int64_t P, const double *pts,
                double *sdf, double *tstar, double *grad3, int *rounds, int outer_only);

/* R1: accumulate the swept-volume penalty over the context's query points into cost / gradT[N] / gradC[6N x 3
 * column-major] (they already hold the energy terms, as in the reference). */
int svsdf_cost_grad(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, double *cost_io,
                    double *gradT_io, double *gradC_io);

/* R3: boundary conditions (3x3 column-major: column k = k-th derivative of (x, y, yaw)) and piece count. */
int svsdf_set_boundary(svsdf_ctx *ctx, const double *initS, const double *finalS, int N);
/* R3: LMBM / L-BFGS compatible callback: x = [tau (N), xi (3(N-1))] -> cost, g.  `instance` is a svsdf_ctx*. */
double svsdf_evaluate(void *instance, const double *x, double *g, const int n);
/* Cost split of the last svsdf_evaluate: out3 = (cost_pos, cost_other, cost_total)  (back_end_optimizer.hpp:396-398) */
int svsdf_last_costs(const svsdf_ctx *ctx, double *out3);
/* Durations and MINCO coefficients of the last svsdf_evaluate (T_out[N], coeffs_out[18N] column-major). */
int svsdf_get_traj(const svsdf_ctx *ctx, double *T_out, double *coeffs_out);

/* Host L-BFGS parameters (utils/include/utils/lbfgs_ref.hpp:20-130; yaml: mem_size, past, min_step, g_epsilon). */
typedef struct {
    int mem_size;
    int past;
    double delta;
    double g_epsilon;
    int max_iterations;
    int max_linesearch;
    double min_step, max_step;
    double f_dec_coeff, s_curv_coeff, cautious_factor, machine_prec;
    /* Non-smooth handling (the SVSDF cost has kinks and finite-difference gradients; the reference drives it with LMBM for
       that reason, back_end_optimizer.cpp:29-36).  When the line search fails on a quasi-Newton direction the memory is
       dropped and the search restarts along -g, at most this many times in a row without an accepted step; when it fails on
       -g itself the run ends with status 3 (no decrease along the steepest-descent direction to line-search precision:
       the counterpart of LMBM_NOMOREPROGRESS, lmbm.h:182).  0 = plain lbfgs_ref.hpp behaviour (negative line-search code). */
    int nonsmooth_restarts;
} svsdf_lbfgs_params;
void svsdf_default_lbfgs_params(svsdf_lbfgs_params *p);

typedef struct {
    double final_cost;
    int iterations;     /* accepted line-search steps */
    int evaluations;    /* cost+gradient evaluations */
    int status;         /* lbfgs_ref.hpp return code (0 convergence, 1 stop, 3 no more progress at a kink, <0 error) */
    double seconds;     /* wall-clock of the whole optimisation */
    double gpu_seconds; /* sum of device time of the cost kernels (CUDA events) */
} svsdf_opt_stats;

/* Progress / cancel hook, same contract as lmbm_progress_t (lmbm.h:211-213): non-zero return cancels. */
typedef int (*svsdf_progress_t)(void *user, const double *x, const int k);

/* R4: optimise opt_x in place from the given start (opt_x has N + 3(N-1) entries).  Returns >= 0 on success
 * (0 is remapped to 1 like optimize_traj_lmbm does), negative solver code otherwise; the last iterate is
 * returned either way.  T_out / coeffs_out (may be NULL) receive the final trajectory. */
int svsdf_optimize(svsdf_ctx *ctx, const double *initS, const double *finalS, double *opt_x, int N,
                   const svsdf_lbfgs_params *params, svsdf_progress_t progress, void *user, double *T_out,
                   double *coeffs_out, svsdf_opt_stats *stats);

/* Host L-BFGS on an arbitrary callback (same role as lbfgs::lbfgs_optimize, utils/include/utils/lbfgs_ref.hpp:434):
 * minimises eval(instance, x, g, n) from x (in/out).  Re-entrant.  Returns the lbfgs_ref.hpp status code. */
typedef double (*svsdf_eval_t)(void *instance, const double *x, double *g, const int n);
int svsdf_lbfgs_minimize(svsdf_eval_t eval, void *instance, double *x, int n, const svsdf_lbfgs_params *params,
                         svsdf_progress_t progress, void *user, svsdf_opt_stats *stats);

/* R7: host MINCO_S3NU. q: 3 x (N-1) column-major. Outputs may be NULL. */
int svsdf_minco_forward(const double *initS, const double *finalS, int N, const double *q, const double *T,
                        double *coeffs_out, double *energy, double *gradC_out, double *gradT_out);
int svsdf_minco_propagate(const double *initS, const double *finalS, int N, const double *q, const double *T,
                          const double *gradC, const double *gradT, double *gradQ_out, double *gradT_out);
/* tau <-> T maps (back_end_optimizer.hpp:199-289) */
void svsdf_forward_T(int n, const double *tau, double *T);
void svsdf_backward_T(int n, const double *T, double *tau);

/* R5: shape functor over n body-frame points (rel: n x 3, z ignored by the 2-D shapes). */
int svsdf_shape_sdf(svsdf_ctx *ctx, int64_t n, const double *rel, double *sdf_out);
int svsdf_shape_grad1(svsdf_ctx *ctx, int64_t n, const double *rel, double *grad3_out);

/* Device-resident evaluation for benchmarking and batch mode: runs R1 on the given trajectory with every input
 * already in HBM, leaves the result on the device, and returns the device time of the kernels in milliseconds
 * (CUDA events on the context's stream).  out_host (1 + 19N + 1 doubles: cost, gradC[18N] col-major, gradT[N],
 * n_inside) may be NULL. */
int svsdf_cost_grad_device(svsdf_ctx *ctx, int N, const double *T, const double *coeffs, int repeats,
                           float *ms_per_eval, double *out_host);

/* ---- The reference's own outer solver as a plug-in (SURVEY.md §8f rank 4) ------------------------------------------------------------
 * The back end of the reference is driven by LMBM, shipped as a prebuilt Fortran library (src/utils/include/utils/lmbm.so behind
 * lmbm.h / lmbm.cpp).  It is not redistributed here, but a deployment that has it can plug it in: svsdf_lmbm_open loads the library from
 * `path` — by default a PRIVATE COPY of the file, so that every handle has its own instance of the library's static state (lmbm.cpp:4-6
 * keeps the callback in file-scope statics and the Fortran code keeps COMMON / SAVE data): handles can then run concurrently from
 * different threads, which one shared instance cannot.  svsdf_lmbm_params mirrors lmbm::lmbm_parameter_t (lmbm.h:15-174);
 * svsdf_lmbm_default_params fills the struct's member initialisers (what back_end_optimizer.cpp:29 uses). */
typedef struct svsdf_lmbm svsdf_lmbm;
typedef struct {
    float timeout;
    int bundle_size, ini_corrections, max_corrections, exponent_distmeasure, max_iterations, max_evaluations, past, verbose, update_method,
        scaling_strategy;
    double delta_past, f_rel_eps, f_lower_bound, terminate_param1, terminate_param2, distance_measure, sufficient_dec, max_stepsize;
} svsdf_lmbm_params;
void svsdf_lmbm_default_params(svsdf_lmbm_params *p);
int svsdf_lmbm_open(const char *path, int private_copy, svsdf_lmbm **out);
void svsdf_lmbm_close(svsdf_lmbm *h);
const char *svsdf_lmbm_last_error(void);
/* lmbm::lmbm_optimize(n, x, &fx, eval, instance, progress, &param) (lmbm.h:214-221); returns LMBM's code (>= 0 success). */
int svsdf_lmbm_minimize(svsdf_lmbm *h, svsdf_eval_t eval, void *instance, double *x, int n, const svsdf_lmbm_params *params,
                        svsdf_progress_t progress, double *f_out);
/* Makes svsdf_optimize (and svsdf_optimize_batch for this context) run LMBM instead of the built-in L-BFGS: the context takes its own
 * private instance of the library at `path` (NULL: back to L-BFGS).  params NULL = defaults. */
int svsdf_set_lmbm_library(svsdf_ctx *ctx, const char *path, const svsdf_lmbm_params *params);

/* ---- Mid end (SURVEY.md §8f rank 4; host only, no GPU and no context) ---------------------------------------------------------
 * OriTraj (src/planner_algorithm/include/planner_algorithm/mid_end.hpp, src/mid_end.cpp): the warm-start optimisation between the A*
 * front end and the SVSDF back end — MINCO energy + cubic pull of the inner waypoints towards their A* cells + trapezoid integral of
 * the velocity / body-rate / attitude penalties through the multicopter flatness map (utils/flatness.hpp) + rho * sum(T).
 * svsdf_mid_config mirrors the yaml keys OriTraj::setParam reads; svsdf_mid_default_config fills config/star.yaml's values.
 * Layouts: initS / finalS 3x3 column-major; Q 3 x (N - 1) column-major (inner waypoints); rot_list (N - 1) rotation matrices, 3x3
 * column-major each (recent_se3_path[ind].getRotMatrix(), plan_manager.cpp:159); x = [tau (N), xi (3 (N - 1))]. */
typedef struct {
    double rho_mid_end, vmax, omgmax, weight_v, weight_omg, weight_pr, weight_ar, smoothingEps;
    int integralIntervs;
    double vehicleMass, gravAcc, horizDrag, vertDrag, parasDrag, speedEps;
    int mem_size, past;
    double min_step, g_epsilon, relCostTolMidEnd;
    int max_iterations, cancel_after; /* mid_end.cpp:51 (10000) and earlyExit's `k > 1e2` (mid_end.hpp:626) */
    int solver;                       /* 0: the reference's patched L-BFGS behaviour (utils/lbfgs.hpp:375, 759-779) — the same warm start as
                                         the reference; 1: this build's L-BFGS (Lewis-Overton line search, restarts) — converges further */
} svsdf_mid_config;
void svsdf_mid_default_config(svsdf_mid_config *cfg);
/* OriTraj::costFunction (mid_end.hpp:277-325): cost and gradient at x. */
int svsdf_mid_cost(const svsdf_mid_config *cfg, int N, const double *initS, const double *finalS, const double *Q, const double *rot_list,
                   const double *x, double *cost_out, double *grad_out);
/* OriTraj::getOriTraj (mid_end.cpp:3-92): T_init = config.inittime * ones(N) in the reference.  Returns the solver status (>= 0 success,
 * 2 = stopped by the `k > cancel_after` rule); opt_x_out [N + 3 (N - 1)] is what the back end starts from (plan_manager.cpp:192-199),
 * T_out [N], coeffs_out [18 N] (column-major 6N x 3) the resulting spline. */
int svsdf_mid_get_ori_traj(const svsdf_mid_config *cfg, int N, const double *initS, const double *finalS, const double *Q,
                           const double *T_init, const double *rot_list, double *opt_x_out, double *T_out, double *coeffs_out,
                           double *final_cost_out, int *iterations_out);

/* ---- Batch variants (leading problem dimension; BASELINE config 5, SURVEY.md §8b / §8e) -----------------------------------
 * Independent problems are spread over a POOL of contexts (one worker thread per context; several contexts may sit on the
 * same GPU — each has its own stream, so the host side of one problem (MINCO, line search) and the latency-bound tail of its
 * kernels overlap the kernels of another — or on different GPUs of the process).  Problems are handed out dynamically: a
 * worker takes the next index when it finishes one (`next`: optional source of indices shared with other processes, e.g. a
 * counter in the torch.distributed store; return < 0 or >= n_problems to stop; NULL = internal counter 0, 1, 2, ...).
 * Results do not depend on which context solved a problem (bit-reproducible kernels).
 *
 * svsdf_problem: one optimisation.  Query points are either given (points != NULL: P rows of `stride` doubles) or built on
 * the device from the context's map around the waypoints (svsdf_extract_points semantics; the map must have been set on every
 * context of the pool). */
typedef struct {
    const double *initS, *finalS;   /* 3x3 column-major boundary states */
    double *opt_x;                  /* in: start, out: result; N + 3 (N - 1) entries */
    const double *points;           /* explicit query points or NULL */
    int64_t P;
    int stride;
    const double *waypoints_xy;     /* W x 2 (used when points == NULL) */
    int W;
    double half;
    const double *keepout_xy;       /* optional keep-out samples (synthetic scenes), n_keepout x 2 */
    int n_keepout;
    double clearance;
    double *T_out, *coeffs_out;     /* optional: final durations [N] and MINCO coefficients [18 N] */
} svsdf_problem;
typedef int (*svsdf_next_problem_t)(void *user);
/* stats_out[n_problems] (optional), status_out[n_problems] (svsdf_optimize return values), points_out[n_problems] (optional:
 * number of query points of each problem).  Returns SVSDF_OK when every problem ran (individual solver codes are in
 * status_out), the first API error otherwise. */
int svsdf_optimize_batch(svsdf_ctx *const *ctxs, int n_ctx, const svsdf_problem *problems, int n_problems, int N,
                         const svsdf_lbfgs_params *params, svsdf_next_problem_t next, void *next_user,
                         svsdf_opt_stats *stats_out, int *status_out, int64_t *points_out);
/* One cost + gradient evaluation per problem with HOST buffers (the batch form of svsdf_set_points + svsdf_cost_grad):
 * pts[k]: P[k] rows of `stride` doubles; T: [n][N]; coeffs: [n][18 N] column-major per problem; cost_io [n], gradT_io [n][N],
 * gradC_io [n][18 N] accumulate like svsdf_cost_grad. */
int svsdf_cost_grad_batch(svsdf_ctx *const *ctxs, int n_ctx, int n_problems, int N, const double *const *pts, const int64_t *P,
                          int stride, const double *T, const double *coeffs, double *cost_io, double *gradT_io, double *gradC_io);

/* ---- Many problems on ONE context: one set of launches per evaluation round ----------------------------------------------------
 * svsdf_cost_grad_multi: the cost and gradient of n problems (each with its own N, T, coefficients and query points; the context's
 * robot shape, pre-transform, penalty weights and scale schedule are shared) in one upload, one launch of each cost kernel (two k_outer
 * launches when both point schedules occur) and one download.  Every problem gets the bits svsdf_set_points + svsdf_cost_grad give it
 * on the same context, n_inside included: it keeps its own k_outer decomposition (the grid its single call would launch and the same
 * sparse / batched schedule) and its own reduction order.  The dynamic shared memory of a k_outer launch is sized by its largest
 * trajectory, so one long trajectory lowers the residency of the whole launch (speed only, not the bits).  0 <= n <= 65535; P = 0 is
 * allowed (the cost is then 0).  An invalid problem (N outside 1..64, a bad duration, null outputs, P < 0, stride < 2, null points)
 * refuses the whole call with SVSDF_ERR_INVALID before any work.  Returns SVSDF_ERR_NONFINITE, after accumulating every problem, when
 * a cost is not finite. */
typedef struct {
    int N;
    const double *T, *coeffs;                   /* [N] durations, [18 N] MINCO coefficients (column-major 6N x 3) */
    const double *points;                       /* P rows of `stride` doubles (x, y first) */
    int64_t P;
    int stride;
    double *cost_io, *gradT_io, *gradC_io;      /* accumulate like svsdf_cost_grad: [1], [N], [18 N] */
    int64_t *n_inside_out;                      /* optional: interior points of the problem */
} svsdf_multi_problem;
int svsdf_cost_grad_multi(svsdf_ctx *ctx, int n, const svsdf_multi_problem *problems);

/* svsdf_optimize_lockstep: n back ends on one context, in lock-step.  Up to max_in_flight problems (<= 0: min(n, 1024)) are in flight,
 * each a machine of the built-in L-BFGS (the solver of svsdf_optimize, unchanged) in a slot; a problem that finishes hands its slot
 * to the next.  The calling thread advances the machines round by round: every live problem asks for an evaluation, and ONE
 * svsdf_cost_grad_multi-style round evaluates all of them, with each problem's host half (tau -> T, MINCO, energy; afterwards the
 * adjoint and rho * sum(T)) and its solver step spread over OpenMP threads.  Per problem, opt_x, T_out, coeffs_out, status_out
 * (svsdf_optimize's return value) and stats_out (final cost, iterations, evaluations, status) equal svsdf_optimize on the same
 * inputs bit for bit, whatever max_in_flight and the order in which problems are taken; stats seconds / gpu_seconds are the problem's
 * wall time (from entering its slot to leaving it) and the device time of the rounds it took part in.  f0_out (optional) receives
 * the cost of the first evaluation, i.e. at the start point.  Inputs are checked like svsdf_optimize's (2 <= N <= 64, non-null
 * initS / finalS / opt_x, P >= 0, stride >= 2, points when P > 0): one invalid problem refuses the call.  A context with an LMBM library
 * (svsdf_set_lmbm_library) is refused with SVSDF_ERR_INVALID.  Returns SVSDF_OK, or the error of a failed round (every problem of that
 * round then ends with it, as svsdf_optimize ends on a failed evaluation).  svsdf_lockstep_rounds: the rounds of the last call. */
typedef struct {
    int N;
    const double *initS, *finalS;               /* 3x3 column-major */
    double *opt_x;                              /* in: start, out: result; N + 3 (N - 1) entries */
    const double *points;                       /* P rows of `stride` doubles */
    int64_t P;
    int stride;
    double *T_out, *coeffs_out;                 /* optional: [N], [18 N] */
    double *f0_out;                             /* optional: cost at the start point */
} svsdf_lockstep_problem;
int svsdf_optimize_lockstep(svsdf_ctx *ctx, const svsdf_lockstep_problem *problems, int n, const svsdf_lbfgs_params *params, int max_in_flight,
                            svsdf_opt_stats *stats_out, int *status_out);
int svsdf_lockstep_rounds(const svsdf_ctx *ctx, int64_t *rounds);

/* svsdf_optimize_device: svsdf_optimize_lockstep with the back end on the device.  Every problem in flight keeps its L-BFGS state, its
 * MINCO spline and its query points (uploaded once, when it enters a slot) in device memory; one warp per problem runs the host's own
 * solver and MINCO code (host/lbfgs.hpp, host/minco.hpp) between the evaluations, so the machines never leave the device.  A round is
 * one small download of every slot's state, the host's launch plan (each problem keeps the grid of its single call), one small upload
 * and the launches; the launches per round do not depend on n.  Same problems, checks, refusals and results as svsdf_optimize_lockstep
 * (bit for bit svsdf_optimize per problem: opt_x, T_out, coeffs_out, f0_out, stats and status_out), plus: max_in_flight above 65535 is
 * refused.  An invalid trajectory ends its problem with a NaN cost and SVSDF_ERR_INVALID; a round that fails gives its error to every
 * problem in it and the call returns that error.  stats seconds: from the start of the call to the end of the problem's last round;
 * gpu_seconds: device time of the rounds it took part in.  rounds_out (optional): the rounds of the call (also svsdf_lockstep_rounds).
 * Solver parameters that svsdf_optimize refuses end every problem at once with that code, nothing launched.  At most 2^31 - 1 query points
 * in one call.  After a CUDA error only the return value and status_out (that error for every problem not finished) are written.
 * No progress hook. */
int svsdf_optimize_device(svsdf_ctx *ctx, const svsdf_lockstep_problem *problems, int n, const svsdf_lbfgs_params *params, int max_in_flight,
                          svsdf_opt_stats *stats_out, int *status_out, int64_t *rounds_out);
/* svsdf_round_times: device time (ms) of the rounds of the last svsdf_optimize_lockstep / svsdf_optimize_device call: the evaluation
 * kernels (pose table to finalize) and the back-end kernels (blobs and the device L-BFGS / MINCO; 0 for svsdf_optimize_lockstep, whose
 * machines are advanced round by round on the host). */
int svsdf_round_times(const svsdf_ctx *ctx, double *eval_ms, double *backend_ms);

/* ---- "next" row (SURVEY.md §8f rank 1): query-point construction on the device --------------------------------------
 * R8  PlannerManager::generateTraj point collection  plan_manager/src/plan_manager.cpp:156-175
 *     PCSmapManager::getPointsInAABBOutOfLastOne       map_manager/include/map_manager/PCSmap_manager.h:184-219
 *     on the byte-packed map kernel of PCSmapManager::generateMapKernel2D (PCSmap_manager.h:81-108), z = 0 layer.
 * svsdf_set_map copies the packed map ((X + 2h) rows of ceil((Y + 2h)/8) bytes, h = (kernel_size-1)/2, MSB first) to the
 * device; svsdf_set_map_device adopts a device buffer (e.g. the NCCL-broadcast one) without copying.  origin = the
 * map's boundary_xyzmin (x, y), res = grid resolution. */
int svsdf_set_map(svsdf_ctx *ctx, const unsigned char *kernel_bytes, int X, int Y, int kernel_size, double origin_x,
                  double origin_y, double res);
int svsdf_set_map_device(svsdf_ctx *ctx, const unsigned char *dev_kernel_bytes, int X, int Y, int kernel_size,
                         double origin_x, double origin_y, double res);
/* The reference's 3-D map: generateMapKernel's layout (PCSmap_manager.h:39-78: (X + 2h) x (Y + 2h) x ceil((Z + 2h)/8) bytes, z bits
 * MSB first), origin = boundary_xyzmin (x, y, z).  Re-packed into Z layers of the 2-D layout on upload; layer 0 is what
 * svsdf_set_map would have been given (generateMapKernel2D), so the front-end entry points work on it unchanged.  Z <= 64. */
int svsdf_set_map3d(svsdf_ctx *ctx, const unsigned char *kernel_bytes, int X, int Y, int Z, int kernel_size,
                    const double *origin_xyz, double res);
/* svsdf_extract_points on a 3-D map: waypoints_xyz W x 3, half_xyz = the box half sizes (bdx/3, bdy/3, bdz/3 in
 * plan_manager.cpp:165).  Every occupied voxel of every layer inside a box (and outside the last box in at least one dimension)
 * is a query point; voxels stacked above the same (x, y) give several points with that (x, y) — the cost loop zeroes z
 * (back_end_optimizer.hpp:791).  Output order: layer by layer, ascending (i*Y + j) within a layer. */
int svsdf_extract_points3d(svsdf_ctx *ctx, const double *waypoints_xyz, int W, const double *half_xyz, const double *keepout_xy,
                           int n_keepout, double clearance, int64_t *n_points);
/* Builds the context's resident query-point set from the map: occupied cells inside the AABB (half-size `half` in x and
 * y) of waypoint w and outside the AABB of waypoint w-1 (for w = 0: outside the box around tmp_pos = (999, 999, 999),
 * plan_manager.cpp:152, i.e. the map's far corner cell), de-duplicated, in ascending (i*Y + j) order.
 * waypoints_xy: W x 2.  keepout_xy / clearance (optional, n_keepout = 0 to disable; not part of the reference): drop
 * cells closer than `clearance` to any keep-out sample.  n_points receives the count. */
int svsdf_extract_points(svsdf_ctx *ctx, const double *waypoints_xy, int W, double half, const double *keepout_xy,
                         int n_keepout, double clearance, int64_t *n_points);
/* Copies the context's resident points (packed x, y) back to the host (tests). */
int svsdf_get_points(svsdf_ctx *ctx, double *xy_out, int64_t capacity, int64_t *n_points);

/* ---- Next row (SURVEY.md 8f rank 3): collision kernels of the A* front end -----------------------------------------------
 *   R9  BasicShape::initShape (yaw-indexed occupancy kernels of the shape)      utils/include/utils/Shape.hpp:386-430, 194-216
 *       SweptVolumeManager::kernelConv<true> / visit_kernels_by_distance / checkKernelValue
 *                                                                                swept_volume/include/swept_volume/sw_manager.hpp:1033-1169
 * svsdf_front_init builds the kernel_yaw_num kernels (kernel_size x kernel_size cells of size occupancy_resolution, cell set
 * iff getonlySDF(cell centre, Rz(yaw_k)) <= max(front_end_safeh, occupancy_resolution / 2)) on the device with the context's
 * shape functor; yaml keys kernel_size (odd, <= 32), kernel_yaw_num (<= 64), occupancy_resolution, front_end_safeh.
 * Not available for the Polygon / mesh functors (the reference defines no rotated kernels for them).
 * svsdf_front_get_kernels: yaw_out [K], cells_out [K][ks][ks] (0/1), bytes_out [K][ks][(ks+7)/8] (MSB first) — any may be NULL.
 * svsdf_front_cspace: with the map of svsdf_set_map (packed for the same kernel_size), free[k][x][y] = kernelConv(k, (x, y)) for
 *   every yaw kernel and cell, as 32-cell words: word [k][x][w], bit (31 - t) <-> y = 32 w + t, 1 = no collision; cells beyond
 *   Y read 0.  words_out (host, K * X * ceil(Y/32) words) may be NULL; ms_out = device time of the kernel; dev_words_out = the
 *   device copy (valid until the next call).
 * svsdf_front_check_kernel_value: checkKernelValue(father_yaw, child_yaw, ind) for n nodes: ok_out[i] = a free yaw kernel was
 *   found within the reference's breadth-first search (at most 11 kernels around the father's), child_yaw_out[i] = its yaw
 *   (father_yaw when none). */
/* svsdf_front_expand: the neighbour loop of AstarPathSearcher::process (planner_algorithm/include/planner_algorithm/
 *   front_end_Astar.hpp:192-240) for n nodes at once (e.g. the current node of each problem of a batch): for node i (cell index
 *   node_ij[2i..], yaw node_yaw[i]) and each of its 9 cells (di, dj in -1..1, di-major): ok_out[9i + m] =
 *   isIndexValid && !occupied && checkKernelValue(fy, cy, vi) && checkSubSWCollision((father centre, fy), (child centre, cy),
 *   occupied cell centres within kernel_size/2 + 1 of the child) (sw_manager.hpp:1171-1210, PCSmap_manager.h:137-158);
 *   child_yaw_out[9i + m] = cy.  parts_out (optional): bit 0 valid and free, bit 1 kernel test, bit 2 sub-swept-volume test. */
int svsdf_front_expand(svsdf_ctx *ctx, int64_t n, const int32_t *node_ij, const double *node_yaw, unsigned char *ok_out,
                       double *child_yaw_out, unsigned char *parts_out);
/* svsdf_front_astar: AstarPathSearcher::AstarPathSearch + getPath (front_end_Astar.hpp:243-390; z = 0 layer) for n start/goal
 *   pairs on the map of svsdf_set_map, all searches advancing in lock-step so that every iteration is ONE svsdf_front_expand
 *   launch over the current node of every unfinished search (host logic: csrc/host/astar.hpp; per search it is the
 *   reference's: multimap open list, no re-keying of improved open nodes, re-opening of closed ones, yaw fixed at first
 *   visit).  paths_out [n][max_path][3] = (x, y, yaw) per node, start first; len_out[n] = nodes on the path (0: no path or
 *   longer than max_path); expansions_out[n] / rounds_out (optional): expansions per search / number of lock-step rounds. */
int svsdf_front_astar(svsdf_ctx *ctx, int n, const double *start_xy, const double *goal_xy, int max_path, double *paths_out,
                      int32_t *len_out, int32_t *expansions_out, int64_t *rounds_out);
/* svsdf_front_astar_device: the same n searches as svsdf_front_astar (same paths, yaws and expansion counts), each run whole on the
 *   device in ONE kernel launch — no host step between expansions (k_astar_search: one CTA per search in flight, the bookkeeping of
 *   csrc/host/astar_flat.hpp in its thread 0, the neighbour tests of svsdf_front_expand on its 9 warps).  Same inputs and layouts:
 *   paths_out [n][max_path][3], start node first; len_out[q] = 0 when there is no path or it is longer than max_path; entries of a
 *   row past len_out[q] are unspecified.  max_expansions >= 1 is the per-search budget (the test of the reference's loop: a pop
 *   that is not the goal ends the search once max_expansions nodes have been expanded).  expansions_out, status_out and ms_out may
 *   be NULL.  status_out[q]: 0 start or goal outside the map (isInMap; the search did not run), 1 path returned, 2 open list ran
 *   empty, 3 max_expansions reached, 4 path found but longer than max_path, -1 an internal guard tripped (heap overflow or a father
 *   chain longer than X * Y + 1; neither happens in a correct search).  ms_out = device time of the search kernel.  Needs
 *   max_path >= 1 and n >= 0 (n = 0 returns at once); one search slot (45 bytes per map cell) must fit the 2 GiB search pool.
 *   SVSDF_FORCE_GRID_ASTAR = n > 0 in the environment at svsdf_create sets the kernel's grid (tests). */
int svsdf_front_astar_device(svsdf_ctx *ctx, int n, const double *start_xy, const double *goal_xy, int max_path, int64_t max_expansions,
                             double *paths_out, int32_t *len_out, int32_t *expansions_out, int32_t *status_out, float *ms_out);
int svsdf_front_init(svsdf_ctx *ctx, int kernel_size, int kernel_yaw_num, double occupancy_resolution, double front_end_safeh);
int svsdf_front_get_kernels(svsdf_ctx *ctx, double *yaw_out, unsigned char *cells_out, unsigned char *bytes_out);
int svsdf_front_cspace(svsdf_ctx *ctx, uint32_t *words_out, float *ms_out, const uint32_t **dev_words_out);
int svsdf_front_check_kernel_value(svsdf_ctx *ctx, int64_t n, const double *father_yaw, const int32_t *ind_xy,
                                   unsigned char *ok_out, double *child_yaw_out);

/* The device sin/cos used on the path (fdlibm restatement, csrc/svsdf_sincos.cuh), exposed for parity tests. */
int svsdf_sincos(svsdf_ctx *ctx, int64_t n, const double *x, double *sin_out, double *cos_out);

/* Measurement helpers */
/* Device time (ms, CUDA events on the context's stream) of the kernels of the last svsdf_cost_grad_device
 * evaluation: out4 = { k_pose_table, k_outer, k_compact + k_gsip, k_finalize }. */
int svsdf_last_kernel_ms(const svsdf_ctx *ctx, float *out4);
int svsdf_kernel_launches(const svsdf_ctx *ctx, int64_t *count);       /* kernels launched by this ctx so far */
int svsdf_executed_evals(svsdf_ctx *ctx, int enable, uint64_t *count); /* lane-level SDF evaluations counter */
int svsdf_fp64_peak(svsdf_ctx *ctx, double *tflops);                   /* measured DFMA peak (2 flop/FMA) */
int svsdf_device_ptr_points(svsdf_ctx *ctx, const double **dev_xy);    /* device pointer of the packed points */

#ifdef __cplusplus
}
#endif
#endif /* SVSDF_H_ */
