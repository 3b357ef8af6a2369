/*
 * sicp_b200.h — C ABI of libsicp_b200.so: the H100 (sm_90a) ICP inner loop behind the
 * simpleICP Python API.
 *
 * The reference (pglira/simpleICP) has no FFI/plugin layer (SURVEY.md §0.9); its boundary is the
 * Python class surface exported at python/simpleicp/__init__.py:12-14.  This header is the
 * C boundary a binding of that surface needs: one entry point per reference method on the hot
 * path, each citing the reference code it replaces (paths relative to the reference repo).
 *
 * Conventions
 *  - extern "C", plain pointers and sizes, no torch / C++ types.
 *  - Every function returns a sicp_status; sicp_last_error(ctx) gives the message.
 *  - Pointers marked [h|d] may be host or device memory (detected with
 *    cudaPointerGetAttributes); [h] must be host memory.  The caller owns every buffer it passes
 *    and allocates every output; the library never frees or keeps caller memory.  Any alignment
 *    of the element type is accepted; outputs that are misaligned or on another device than the
 *    context's are written through the library's own device buffer.
 *  - All point arrays are row-major n x 3 float64 (NumPy's layout for PointCloud.X,
 *    python/simpleicp/pointcloud.py:81-84).  Indices are int64 like NumPy's.
 *  - A context is bound to one device and one CUDA stream (e.g. torch's current stream); calls
 *    on one context are not thread-safe, different contexts are independent.
 *  - Angles are radians at this boundary (the Python facade converts degrees,
 *    python/simpleicp/simpleicp.py:146-148).
 */
#ifndef SICP_B200_H
#define SICP_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The version changes when a struct layout or an existing entry point's meaning changes.  Added
 * entry points leave it as it is (sicp_get_batch_outputs came in at version 5): bindings look
 * them up by name. */
#define SICP_ABI_VERSION 5

typedef enum {
  SICP_OK = 0,
  SICP_ERR_BAD_ARG = 1,       /* argument checks, simpleicp.py:326-353, pointcloud.py:158-159   */
  SICP_ERR_NO_OVERLAP = 2,    /* "Point clouds do not overlap ...", simpleicp.py:165-170         */
  SICP_ERR_TOO_FEW_CORR = 3,  /* "Too few correspondences!" (< 6), simpleicp.py:209-214          */
  SICP_ERR_CUDA = 4,
  SICP_ERR_SINGULAR = 5,      /* normal equations not positive definite                          */
  SICP_ERR_STATE = 6          /* call order violated (e.g. match before set_clouds)              */
} sicp_status;

typedef struct sicp_ctx sicp_ctx;

/* Nearest-neighbour engine selection (both engines are exact). */
typedef enum {
  SICP_NN_AUTO = 0,  /* uniform-grid search, TMA brute force for queries the grid cannot bound */
  SICP_NN_GRID = 1,  /* grid only, ring expansion until proven exact                           */
  SICP_NN_BRUTE = 2  /* TMA-staged tiled brute force for every query                           */
} sicp_nn_engine;

/* Normal sign convention.  The reference's sign is whatever LAPACK dgeev returns
 * (pointcloud.py:191-197, np.linalg.eig) — see DESIGN.md "normal sign". */
typedef enum {
  SICP_SIGN_DGEEV = 0,     /* reproduce np.linalg.eig's sign (Hessenberg-QR path of dgeev)       */
  SICP_SIGN_CANONICAL = 1  /* largest-magnitude component positive                              */
} sicp_sign_mode;

/* Algorithm variant of reject + solve (option key "variant").  The default is the Python package's
 * algorithm (the north-star path).  The linearised variants restate the C++ driver
 * (c++/src/corrpts.cpp:59-156, c++/src/simpleicp.cpp:54-80; pinned to those sources, see
 * tests/test_cpp_reference_pin.py): median/MAD over ALL distances with the upper middle element
 * (std::nth_element at n/2), sigma = 1.4826 MAD, one linear solve A x = l per iteration, cloud
 * moved by the RIGID dH = H(euler(x), t), residuals A x - l, sample standard deviation, no
 * parameter uncertainties and no observed/fixed parameters.  They differ in the matrix that is
 * REPORTED: H * dH (the C++ driver, c++/src/simpleicp.cpp:66) or dH * H, the transform really
 * applied to the cloud and the composition order of the Rust / Julia / MATLAB drivers
 * (rust/src/icp.rs:164, julia/simpleicp.jl:272, matlab/simpleicp.m:55).  Those three ports differ
 * from the C++ arithmetic in two more points that are NOT reproduced: they move the cloud by the
 * linearised matrix I + [x]_x itself (rust/src/icp.rs:339-344, matlab/simpleicp.m:146-152) -- not
 * a rotation, so distances are not preserved and the search could not stay in the static grid
 * of the untouched cloud -- and they average the two middle elements of an even-sized sample
 * (rust/src/icp.rs:392-404).  Both effects are second order in the per-iteration angles.
 * Normals stay in the float32 storage of the default variant (the C++ code keeps float64), see
 * DESIGN.md.                                                                                    */
typedef enum {
  SICP_VARIANT_PYTHON = 0,
  SICP_VARIANT_LINEARIZED = 1,        /* C++ arithmetic, reports dH * H                          */
  SICP_VARIANT_LINEARIZED_CPP = 2     /* C++ arithmetic, reports H * dH (the C++ driver itself)  */
} sicp_variant;

/* ---- life cycle --------------------------------------------------------------------------- */
int32_t sicp_abi_version(void);
int32_t sicp_create(int32_t device, void* cuda_stream, sicp_ctx** out);
int32_t sicp_destroy(sicp_ctx* ctx);
const char* sicp_last_error(sicp_ctx* ctx); /* ctx may be NULL: last error of the calling thread */
int32_t sicp_set_option(sicp_ctx* ctx, const char* key, double value);
/*  keys: "nn_engine" (sicp_nn_engine), "sign_mode" (sicp_sign_mode), "variant" (sicp_variant),
 *        "grid_target_occupancy"
 *        (points per occupied cell, default 3), "grid_max_rings" (ring limit before the
 *        brute-force pass takes over, default 8), "grid_sort_cells" (0/1), "host_sync_every"
 *        (iterations queued between host reads in sicp_run, default 4), "match_group" (lanes per
 *        query in the grid search: 0 = by K, 1, 4, 8, 16), "fused" (1: iterations after the first
 *        run their reject + solve in the barrier-free kernel, 0: always the cooperative kernel),
 *        "warm_start" (1: the grid search of an iteration starts from the previous iteration's
 *        neighbour as upper bound), "keep_knn" (see sicp_get_knn), "knn_coop" (k-NN search: 1 cooperative
 *        lanes per query (k <= 16), 0 one thread per query, -1 (default) by the number of queries),
 *        "upload_threads" (worker threads that stage a cloud given in PAGEABLE host memory --
 *        e.g. a NumPy array -- through pinned buffers, default 2; 0: plain cudaMemcpyAsync, which
 *        the driver stages on the calling thread; pinned and device sources never use them),
 *        "upload_chunk_kb" (slice size of that staging, default 2048), "normals_scratch_mb"
 *        (bound of the movable-normals estimate's neighbour scratch, default 64: it runs in
 *        launches of 2^20 x normals_scratch_mb / (4 k) queries), "joint_solver" (the solve of
 *        sicp_register_joint: 0 dense, the default; 1 sparse, see there), "defaults" (any value:
 *        every option back to its default)                                */

/* ---- clouds: SimpleICP.add_point_clouds (simpleicp.py:58-73) + PointCloud.X ---------------- */
int32_t sicp_set_clouds(sicp_ctx* ctx, const double* fix_xyz /*[h|d] n_fix x 3*/, int64_t n_fix,
                        const double* mov_xyz /*[h|d] n_mov x 3*/, int64_t n_mov);

/* ---- selection: PointCloud.idx_selected / select_n_points (pointcloud.py:91-147) ----------- */
/* idx ascending fixed-cloud indices; idx == NULL selects all n_fix points.                    */
int32_t sicp_set_selected(sicp_ctx* ctx, const int64_t* idx /*[h|d] K or NULL*/, int64_t K);

/* PointCloud.select_in_range (pointcloud.py:149-171) as used at simpleicp.py:158-170:
 * keep[i] = 1 iff the nearest point of H0 * X_mov to selected fixed point i is STRICTLY closer
 * than max_range.  n_kept == 0 returns SICP_ERR_NO_OVERLAP.                                    */
int32_t sicp_select_in_range(sicp_ctx* ctx, const double H0[16], double max_range,
                             uint8_t* keep /*[h|d] K*/, int64_t* n_kept /*[h]*/);

/* ---- normals: PointCloud.estimate_normals (pointcloud.py:173-203) ---------------------------
 * k-NN (self included) in the fixed cloud, covariance (ddof=1), symmetric 3x3 eigen-solve;
 * normal = eigenvector of the smallest eigenvalue, planarity = (l_mid - l_min) / l_max, float32.
 * Outputs may be NULL (kept on the device for sicp_match either way).                          */
int32_t sicp_estimate_normals(sicp_ctx* ctx, int32_t neighbors, float* nx, float* ny, float* nz,
                              float* planarity /*[h|d] K each*/);
/* The reference's "columns already present" hook (simpleicp.py:176-178).                       */
int32_t sicp_set_normals(sicp_ctx* ctx, const float* nx, const float* ny, const float* nz,
                         const float* planarity /*[h|d] K each*/);
/* Movable-side attributes (optional; the default run has none).  Arrays of n_mov floats in the
 * movable cloud's own frame, NaN where not estimated; all four NULL clears them; a new movable
 * cloud (sicp_set_clouds / sicp_register) clears them too.
 *  - planarity: second branch of CorrPts.reject_wrt_planarity (corrpts.py:157-162): when pc_mov
 *    carries a planarity column, a correspondence must pass min_planarity on BOTH sides; NaN
 *    fails.  The median / MAD of the distance rejection are taken over that set.
 *  - max_angle_rad in [0, pi/2]: CorrPts.reject_wrt_to_angle_between_normals — the hook the
 *    reference declares, calls after the distance rejection (simpleicp.py:207, commented out)
 *    and leaves `raise NotImplementedError` (corrpts.py:190-193).  Here: a correspondence that
 *    survived both rejections is dropped when acos|n_fix . (R n_mov)| > max_angle_rad, R the
 *    rotation of the iteration's transform.  Negative: no angle test.
 * Both act in sicp_match/sicp_reject/sicp_solve, sicp_iterate and sicp_run.  sicp_register and
 * sicp_register_batch take their clouds themselves and clear them; they estimate the movable
 * attributes on the device instead when sicp_register_params.mov_neighbors > 0.               */
int32_t sicp_set_mov_normals(sicp_ctx* ctx, const float* nx, const float* ny, const float* nz,
                             const float* planarity /*[h|d] n_mov each*/, double max_angle_rad);
/* neighbour indices of the last sicp_estimate_normals (test/inspection hook), K x neighbors; they
 * are only kept when option "keep_knn" was 1 during that call.                                  */
int32_t sicp_get_knn(sicp_ctx* ctx, int64_t* idx /*[h|d] K x k*/, double* dist2 /*[h|d] or NULL*/);

/* ---- one ICP iteration, stage by stage ------------------------------------------------------ */
/* CorrPts.match (corrpts.py:124-137, 195-211): pc2_idx[i] = argmin_j |H x_mov_j - x_fix_sel_i|,
 * dist[i] = (H x_mov_pc2idx - x_fix_sel_i) . n_i.                                              */
int32_t sicp_match(sicp_ctx* ctx, const double H[16], int64_t* pc2_idx /*[h|d] K or NULL*/,
                   double* dist /*[h|d] K or NULL*/);

/* CorrPts.reject_wrt_planarity + reject_wrt_point_to_plane_distances (corrpts.py:139-188):
 * (double)planarity_f32 >= min_planarity (NaN drops), then |d - median| <= 3 * MAD with the
 * RAW median absolute deviation (SciPy scale=1.0, corrpts.py:186).
 * stats[4] = {median, mad, mean(d kept), popstd(d kept)}.                                      */
int32_t sicp_reject(sicp_ctx* ctx, double min_planarity, uint8_t* keep /*[h|d] K or NULL*/,
                    int64_t* n_kept /*[h]*/, double stats[4] /*[h] or NULL*/);

typedef struct {
  double x0[6];           /* start values alpha1..3 [rad], tx,ty,tz (simpleicp.py:223-227)       */
  double observed[6];     /* rbp_observed_values, radians                                      */
  double obs_weight[6];   /* rbp_observation_weights: 0 free, +inf fixed, else observed          */
  double distance_weight; /* > 0; <= 0 or NaN means "None": 1/std(d kept)^2 (simpleicp.py:233)   */
} sicp_lsq_params;

/* SimpleICPOptimization.estimate_parameters (optimization.py:65-124): argmin over the free
 * parameters of sum (w n.(R(x) p2 + t - p1))^2 + sum (w_j (x_j - obs_j))^2, solved to
 * convergence (Levenberg-Marquardt on the exact Euler model).  residuals = unweighted signed
 * distances at the solution, in kept order.  stats[2] = {mean, population std} of them.        */
int32_t sicp_solve(sicp_ctx* ctx, const sicp_lsq_params* p, double x[6] /*[h]*/,
                   double H[16] /*[h]*/, double* residuals /*[h|d] n_kept or NULL*/,
                   double stats[2] /*[h] or NULL*/, double* distance_weight_used /*[h] or NULL*/);

/* SimpleICPOptimization.estimate_parameter_uncertainties (optimization.py:126-170) for the last
 * sicp_solve / sicp_run: sigma[j] = sqrt(Cxx_jj), NaN for fixed parameters.                     */
int32_t sicp_uncertainties(sicp_ctx* ctx, double sigma[6] /*[h]*/);

/* ---- the fused loop: SimpleICP.run iterations (simpleicp.py:184-281) ------------------------ */
typedef struct {
  double min_planarity;
  double min_change;       /* percent, simpleicp.py:355-379                                     */
  int32_t max_iterations;
  int32_t reserved;
  sicp_lsq_params lsq;     /* x0 = observed values on iteration 0, as the reference              */
} sicp_run_params;

typedef struct {
  int64_t n_kept;
  double median, mad;          /* of the planarity survivors                                    */
  double mean_dist, std_dist;  /* kept distances before the solve ("orig:0" row on iteration 0)  */
  double x[6];
  double mean_res, std_res;    /* residuals after the solve (log row, stop rule)                */
  double distance_weight;
  int32_t lm_iterations;
  int32_t n_bruteforce;        /* queries answered by the brute-force engine                    */
} sicp_iter_record;

typedef struct {
  int32_t iterations;          /* number of iterations run (the reference's it + 1)             */
  int32_t converged;           /* 1 if the stop rule fired, 0 if max_iterations was reached     */
  double x[6];
  double H[16];
  double sigma[6];
  int64_t n_residuals;
  double loop_ms;              /* device time of the iteration loop (CUDA events)               */
} sicp_run_result;

int32_t sicp_run(sicp_ctx* ctx, const sicp_run_params* p, sicp_run_result* out /*[h]*/,
                 sicp_iter_record* log /*[h] max_iterations entries or NULL*/);
/* The rigid transform the last sicp_run / sicp_solve actually applied to the movable cloud.  Equal
 * to the result's H except for SICP_VARIANT_LINEARIZED_CPP, whose reported H = H * dH is a
 * different product of the same increments (c++/src/simpleicp.cpp:62-66: the cloud is moved by
 * dH on the left, the report multiplies on the right).                                         */
int32_t sicp_get_transform(sicp_ctx* ctx, double T[16] /*[h]*/);
/* residuals of the final iteration in kept order (simpleicp.py:324, 4th return value).          */
int32_t sicp_get_residuals(sicp_ctx* ctx, double* residuals /*[h|d] cap*/, int64_t cap,
                           int64_t* n /*[h]*/);

/* One iteration (match + reject + solve) with no host round trip except the record; used by the
 * benchmark to time the hot path in isolation.  x_in/out: cumulative parameters.              */
int32_t sicp_iterate(sicp_ctx* ctx, const sicp_run_params* p, const double x_in[6],
                     sicp_iter_record* rec /*[h] or NULL: fully asynchronous*/);

/* PointCloud.select_n_points (pointcloud.py:121-147) applied to the CURRENT selection on the
 * device: keeps the points at rint(linspace(0, m-1, n)) (numpy arithmetic; the linearised
 * variants round half away from zero as c++/src/pointcloud.cpp:92-96 does); no-op when n >= m.
 * idx_out (may be NULL) receives the resulting selection, sicp_set_selected's K is updated.     */
int32_t sicp_select_n_points(sicp_ctx* ctx, int64_t n, int64_t* idx_out /*[h|d] min(n, m) or NULL*/);

/* ---- SimpleICP.run as ONE call (simpleicp.py:75-324) --------------------------------------------
 * add_point_clouds + [select_in_range] + select_n_points + estimate_normals + the iteration loop
 * + the final transform_by_H, scheduled so that the host->device transfer of the movable cloud
 * overlaps the fixed-side work (grid, subsample, normals).  Equivalent to sicp_set_clouds,
 * sicp_set_selected(NULL), [sicp_select_in_range], sicp_select_n_points, sicp_estimate_normals,
 * sicp_run, sicp_transform in sequence; every stage-by-stage call remains valid afterwards
 * (sicp_get_residuals, sicp_get_knn, sicp_match ...).
 * mov_neighbors = k > 0 adds pc_mov.estimate_normals(k) before the run (pointcloud.py:173-203):
 * every movable point gets a normal and a planarity from its k nearest movable neighbours (itself
 * included), estimated on the device right after the movable grid is built, and the loop runs
 * as after sicp_set_mov_normals(those arrays, max_angle_rad).  k must be in [2, 64] and at most
 * the number of movable points; the linearised variants have no movable-side branch
 * (c++/src/corrpts.cpp:27-30) and refuse k > 0.  Violations are SICP_ERR_BAD_ARG before any
 * device work.  A zero-initialised struct is the run without movable attributes.               */
typedef struct {
  int64_t correspondences;       /* simpleicp.py:78 (default 1000)                                */
  int32_t neighbors;             /* simpleicp.py:79 (default 10)                                  */
  int32_t mov_neighbors;         /* 0: no movable attributes; k: estimate them (see above)        */
  double max_overlap_distance;   /* <= 0 or +inf: clouds fully overlap (simpleicp.py:81)          */
  sicp_run_params run;
  double max_angle_rad;          /* read only when mov_neighbors > 0: as sicp_set_mov_normals'
                                    (negative: no angle test, else <= pi/2)                       */
} sicp_register_params;
int32_t sicp_register(sicp_ctx* ctx, const double* fix_xyz /*[h|d] n_fix x 3*/, int64_t n_fix,
                      const double* mov_xyz /*[h|d] n_mov x 3*/, int64_t n_mov,
                      const sicp_register_params* p, sicp_run_result* out /*[h]*/,
                      sicp_iter_record* log /*[h] max_iterations entries or NULL*/,
                      double* mov_xyz_out /*[h|d] n_mov x 3 or NULL*/,
                      int64_t* n_selected /*[h] or NULL*/);

/* ---- many independent pairs in one call (BASELINE.json configs[4]; SURVEY.md section 8e) --------
 * SimpleICP.run (simpleicp.py:75-324) for n_pairs independent (fixed, movable) pairs on ONE GPU
 * with ONE set of kernel launches per stage and per iteration for the whole batch: the grids of
 * all 2 n_pairs clouds are built in one segmented counting sort, the searches of all pairs run in
 * one launch, reject + solve run one block per pair, every pair has its own stop flag.  Results
 * per pair equal those of sicp_register on that pair.
 * fix_xyz[i] / mov_xyz[i] point to the i-th pair's clouds (host, ideally pinned, or device);
 * correspondences must be <= 4096 (one block per pair).
 * max_overlap_distance finite and > 0: PointCloud.select_in_range on every fixed point of pair i
 * under that pair's initial transform, then the subsample over the survivors, as sicp_register
 * does.  A pair without a survivor gets SICP_ERR_NO_OVERLAP and takes no part in the loop.
 * observed (n_pairs x 6, radians, or NULL): row i replaces both run.lsq.x0 and run.lsq.observed
 * for pair i (rbp_observed_values per pair; in the linearised variants only the initial
 * transform); every other parameter is common to the batch.
 * mov_neighbors > 0: every pair's movable cloud gets its normals and planarities on the device
 * (as sicp_register does; k must not exceed any pair's movable point count), max_angle_rad as
 * there.
 * n_selected (or NULL) receives the selected fixed points of each pair (sicp_register's value).
 * out[i].status is the sicp_status of pair i (a pair without overlap or without enough
 * correspondences fails alone); the call itself fails only on bad arguments or CUDA errors.
 * It is sicp_register_pairs over its 2 n_pairs clouds (pair i = clouds 2i and 2i + 1), whose
 * limits of 2^32 points no input an 80 GB GPU can hold reaches (2^32 points take 103 GB).       */
typedef struct {
  int32_t status;
  int32_t iterations;
  int32_t converged;
  int32_t reserved;
  int64_t n_kept;
  double H[16];
  double x[6];
  double sigma[6];
  double mean_res, std_res;   /* of the final residuals (exact, two-pass)                       */
} sicp_pair_result;
int32_t sicp_register_batch(sicp_ctx* ctx, int32_t n_pairs, const double* const* fix_xyz /*[h|d]*/,
                            const int64_t* n_fix, const double* const* mov_xyz /*[h|d]*/,
                            const int64_t* n_mov, const sicp_register_params* p,
                            const double* observed /*[h] n_pairs x 6, radians, or NULL*/,
                            sicp_pair_result* out /*[h] n_pairs*/,
                            int64_t* n_selected /*[h] n_pairs or NULL*/);

/* ---- many scans against ONE resident fixed cloud (a map) ----------------------------------------
 * sicp_set_map uploads a fixed cloud and builds its grid once (the cell plan sicp_register_batch
 * would make for it).  It stays on the context until it is replaced, released (map_xyz NULL or
 * n_map 0) or the context is destroyed; no other call (sicp_set_clouds, sicp_register,
 * sicp_register_batch) touches it.  n_map must be below 2^32.
 * sicp_register_to_map is SimpleICP.run (simpleicp.py:75-324) for n_scans (map, scan i) pairs,
 * with the parameters, limits, `observed` rows, per-scan status and n_selected of
 * sicp_register_batch: the result of scan i equals that of sicp_register_batch with the map as
 * the fixed cloud of every pair, bit for bit.  The map is neither uploaded nor gridded again.
 * With max_overlap_distance the overlap filter only searches the map points inside the box of
 * each scan's movable grid mapped by its prior and grown by max_overlap_distance (plus a rounding
 * margin): the filter's work grows with the scans' footprints, not with the map.  Survivor
 * offsets are 32-bit: n_scans x n_map must be below 2^32 (SICP_ERR_BAD_ARG otherwise), and the
 * filter keeps an n_scans x n_map bit mask on the device.  n_map >= neighbors is required.
 * SICP_ERR_STATE when no map is set.                                                            */
int32_t sicp_set_map(sicp_ctx* ctx, const double* map_xyz /*[h|d] n_map x 3*/, int64_t n_map);
int32_t sicp_register_to_map(sicp_ctx* ctx, int32_t n_scans, const double* const* mov_xyz /*[h|d]*/,
                             const int64_t* n_mov, const sicp_register_params* p,
                             const double* observed /*[h] n_scans x 6, radians, or NULL*/,
                             sicp_pair_result* out /*[h] n_scans*/,
                             int64_t* n_selected /*[h] n_scans or NULL*/);

/* ---- many pairs drawn from ONE set of clouds (scan sequences, loop closures, several priors) ----
 * sicp_register_pairs registers n_pairs pairs whose clouds come from n_clouds clouds: pair i is
 * (xyz[fix_id[i]], xyz[mov_id[i]]).
 *  - Equality: out[i] and n_selected[i] equal, bit for bit, what sicp_register_batch returns for
 *    pair i of the expanded list (fix_xyz[i] = xyz[fix_id[i]], mov_xyz[i] = xyz[mov_id[i]]) with
 *    the same p and observed: every field, every variant, with and without max_overlap_distance
 *    and mov_neighbors.  sicp_get_batch_outputs afterwards returns the same bits as after that
 *    call (transformed clouds, residuals, log, T).
 *  - Shared clouds: fix_id[i] == mov_id[i] is allowed, a cloud may be fixed in one pair and movable
 *    in another, and a cloud no pair references is not read (its pointer may be NULL).
 *  - Done once per cloud: each referenced cloud is uploaded once (any memory kind) and gridded once
 *    under sicp_register_batch's cell plan; that grid is both its fixed and its movable grid.  With
 *    mov_neighbors, each cloud that is movable in some pair gets its normals estimated once.  The
 *    loop is per pair, as in sicp_register_batch.
 *  - SICP_ERR_BAD_ARG, before any device work: the checks of sicp_register_batch's parameters
 *    (n_pairs in [1, 65535], correspondences <= 4096, ...), n_clouds < 1, an id outside
 *    [0, n_clouds), a referenced cloud with a NULL pointer or no point, a cloud that is fixed in a
 *    pair with fewer than `neighbors` points, a cloud that is movable in a pair with fewer than
 *    mov_neighbors points, sum n over the referenced clouds >= 2^32, or sum over pairs of
 *    n[fix_id[i]] >= 2^32 (the overlap filter's keep flags and their prefix sum are per pair and
 *    32-bit).
 *  - The map (sicp_set_map) is not touched.  sicp_timings: upload_ms is the upload of the clouds
 *    that are fixed in some pair, grid_fix_ms their grid build; the clouds that are only movable
 *    cross PCIe on a second stream meanwhile, and grid_mov_ms is their grid build (0 without
 *    them).
 *  - Device memory: the clouds once (24 B per point) and their one grid, plus sicp_register_batch's
 *    per-pair buffers and 4 B of overlap flags per fixed point of each pair.                   */
int32_t sicp_register_pairs(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                            const int64_t* n /*[h] n_clouds*/, int32_t n_pairs,
                            const int32_t* fix_id /*[h] n_pairs*/, const int32_t* mov_id /*[h] n_pairs*/,
                            const sicp_register_params* p,
                            const double* observed /*[h] n_pairs x 6, radians, or NULL*/,
                            sicp_pair_result* out /*[h] n_pairs*/,
                            int64_t* n_selected /*[h] n_pairs or NULL*/);

/* ---- many clouds registered JOINTLY (multi-scan ICP, linearised) ---------------------------------
 * sicp_register_joint estimates one pose T_c (world <- cloud, row-major 4 x 4) per cloud from the
 * edges (fix_id[e], mov_id[e]): per iteration every edge is matched and rejected as pair
 * (a, b) of sicp_register_pairs under SICP_VARIANT_LINEARIZED from R_e = T_a^-1 T_b, and ONE least-
 * squares problem over the kept rows of all edges gives a linearised increment x_c per free cloud;
 * T_c <- dH(x_c) T_c.  DESIGN.md §6.9 states the rule.
 *  - Rules: always the linearised ones, whatever the context's "variant" option.  p is read as
 *    sicp_register_pairs reads it (correspondences, neighbors, max_overlap_distance,
 *    run.min_planarity, run.min_change, run.max_iterations).
 *  - Reduction: with two clouds, one edge (0, 1), cloud 0 fixed with T_0 = I and H0[1] = H(x0), the
 *    result equals sicp_register_pairs' under SICP_VARIANT_LINEARIZED with observed row x0 up to
 *    rounding.
 *  - SICP_ERR_BAD_ARG, before any device work: every check of sicp_register_pairs under a
 *    linearised variant (n_edges in [1, 65535], correspondences <= 4096, zero observation weights,
 *    ...), mov_neighbors != 0, a self edge, a non-finite H0 entry, no free cloud or more than 256
 *    free clouds among the referenced ones (16 384 under option "joint_solver" 1), or a free cloud
 *    whose component of the edge graph holds no fixed cloud.  A cloud no edge references is not read (its pointer may be NULL).
 *  - Outputs: H_out[c] = the final T_c; fixed and unreferenced clouds get H0 (identity for a NULL
 *    H0) bit for bit.  out[e]: status, the call's iterations and convergence, the edge's last
 *    n_kept, H = final T_a^-1 T_b, x = the edge's last increment in frame a, mean_res / std_res of
 *    the final linear-model residuals (two-pass), sigma NaN (the a-posteriori covariances of every
 *    pose and every edge come from sicp_get_joint_covariances).  Converged when at an iteration i > 0
 *    every edge with >= 6 kept rows meets the stop rule.
 *  - Failures: an edge without overlap under R_e gets SICP_ERR_NO_OVERLAP and takes no part (the
 *    call returns SICP_ERR_NO_OVERLAP if that leaves a free cloud without a path to a fixed one);
 *    an edge with < 6 kept rows contributes nothing to that iteration, and reports
 *    SICP_ERR_TOO_FEW_CORR if that was its last; a joint normal matrix that is not positive
 *    definite returns SICP_ERR_SINGULAR.  On any error H_out is not written.
 *  - After SICP_OK, sicp_get_batch_outputs (n_pairs = n_edges) returns per edge cloud b moved by the
 *    final T_a^-1 T_b, the final linear-model residuals in kept order, the log and T = that
 *    transform.  The map and the one-pair state are not touched.  sicp_timings: match_ms,
 *    reject_solve_ms and transform_ms are the loop's match, reject-and-blocks and joint solve +
 *    update times (device events, summed over the iterations run).
 *  - Option "joint_solver" (sicp_set_option), read by each call: 0 (the default) solves the joint
 *    system by a dense Cholesky, at most 256 free clouds.  1 solves the same system, with the same
 *    rule and outputs up to rounding, by a supernodal Cholesky over a nested-dissection ordering of
 *    the edge graph (DESIGN.md §6.11): at most 16 384 free clouds (more is SICP_ERR_BAD_ARG), and a
 *    factor of at most 4 GiB, computed from the edges before any upload (more is SICP_ERR_BAD_ARG,
 *    with the bytes in the message).  After a call under 1, sicp_get_joint_covariances returns
 *    SICP_ERR_STATE (sicp_get_joint_selected_covariances serves both solvers);
 *    sicp_get_batch_outputs works as after 0.                                                   */
int32_t sicp_register_joint(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                            const int64_t* n /*[h]*/, int32_t n_edges,
                            const int32_t* fix_id, const int32_t* mov_id /*[h] n_edges*/,
                            const int32_t* is_fixed /*[h] n_clouds, nonzero: pose held*/,
                            const double* H0 /*[h] n_clouds x 16 row-major, or NULL: identity*/,
                            const sicp_register_params* p,
                            double* H_out /*[h] n_clouds x 16*/,
                            sicp_pair_result* out /*[h] n_edges*/, int64_t* n_selected /*[h] or NULL*/);

/* ---- joint registration with POSE PRIORS (DESIGN.md §6.12) ---------------------------------------
 * sicp_register_joint_priors is sicp_register_joint with a weighted observation of each cloud's
 * absolute pose (GNSS/INS, odometry); sicp_register_joint is this call with both NULL.
 *  - Rule: cloud c's prior is an observed rigid pose P_c = prior_H[c] (world <- cloud) and six
 *    weights w_c = prior_w[c] = (w_wx, w_wy, w_wz, w_x, w_y, w_z) >= 0 in world axes, 1/rad^2 and
 *    1/m^2, relative to the unit weight of a point-to-plane row in metres (w = (sigma_row /
 *    sigma_prior)^2); 0: that component is not observed.  At every iteration, at the current pose
 *    T_c = (R_c, o_c), the prior observes u_c = (omega_c, do_c), the world rotation increment and
 *    the displacement of the cloud's origin, with l_c = (rotvec(R_P R_c^T), o_P - o_c); the joint
 *    minimisation adds sum_c (u_c - l_c)^T diag(w_c) (u_c - l_c).  The pose update, the per-edge
 *    records and the stop rule (every live edge's, priors take no part) are sicp_register_joint's.
 *  - Read: the prior of a free cloud some edge references with at least one non-zero weight.  The
 *    pose of any other prior (fixed, unreferenced, all weights 0) is not read and may be NaN.  A
 *    call that reads no prior runs exactly as sicp_register_joint: same launches, same bits.
 *  - Anchoring: a component of the edge graph is anchored by a fixed cloud or by a free cloud whose
 *    six weights are all > 0, both in the check before any device work (SICP_ERR_BAD_ARG) and over
 *    the edges that keep their overlap (SICP_ERR_NO_OVERLAP); so no fixed cloud at all is legal when
 *    priors anchor every component.  Priors on fewer components (e.g. position only) count in the
 *    system but not as an anchor; a system they leave indefinite is SICP_ERR_SINGULAR.
 *  - SICP_ERR_BAD_ARG, before any device work, besides sicp_register_joint's checks: exactly one of
 *    prior_H and prior_w NULL; any weight of prior_w negative or not finite (use is_fixed for an
 *    exact pose); a read prior pose with a non-finite entry, a bottom row other than (0, 0, 0, 1)
 *    or a rotation part with |R^T R - I| > 1e-6.
 *  - sicp_get_joint_covariances after this call: N includes the priors' blocks, and s0^2 =
 *    (sum_e sum_i r_ei^2 + sum_c v_c^T W_c v_c) / (sum_e n_e + sum_c m_c - 6 F), v_c = u_c - l_c the
 *    prior's linear-model residual of the final iteration (l_c at the poses that iteration started
 *    from) and m_c the number of non-zero weights of each read prior.                           */
int32_t sicp_register_joint_priors(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                                   const int64_t* n /*[h]*/, int32_t n_edges,
                                   const int32_t* fix_id, const int32_t* mov_id /*[h] n_edges*/,
                                   const int32_t* is_fixed /*[h] n_clouds, nonzero: pose held*/,
                                   const double* H0 /*[h] n_clouds x 16 row-major, or NULL: identity*/,
                                   const double* prior_H /*[h] n_clouds x 16 row-major, or NULL*/,
                                   const double* prior_w /*[h] n_clouds x 6, or NULL*/,
                                   const sicp_register_params* p,
                                   double* H_out /*[h] n_clouds x 16*/,
                                   sicp_pair_result* out /*[h] n_edges*/, int64_t* n_selected /*[h] or NULL*/);

/* ---- joint registration with RELATIVE POSE OBSERVATIONS (DESIGN.md §6.13) -----------------------
 * sicp_register_joint_relative is sicp_register_joint_priors with weighted observations of the
 * relative pose of two clouds (wheel or visual odometry, the INS trajectory between two scans, an
 * earlier pairwise result); sicp_register_joint_priors is this call with n_rel = 0.
 *  - Rule: observation k joins clouds a = rel_a[k] != b = rel_b[k] with an observed rigid transform
 *    Z_k = rel_H[k] of T_a^-1 T_b (cloud b in frame a) and six weights w_k = rel_w[k] = (w_ax, w_ay,
 *    w_az, w_x, w_y, w_z) >= 0 in frame-a axes, 1/rad^2 and 1/m^2, relative to the unit weight of a
 *    point-to-plane row in metres (w = (sigma_row / sigma_odo)^2); 0: that component is not
 *    observed.  At every iteration, at the current poses, it observes u_k = (alpha, dq), the
 *    rotation increment of T_a^-1 T_b in frame-a axes and the displacement of o_b in frame a, with
 *    l_k = (rotvec(R_Z R_ab^T), t_Z - t_ab), R_ab = R_a^T R_b, t_ab = R_a^T (o_b - o_a); the joint
 *    minimisation adds sum_k (u_k - l_k)^T diag(w_k) (u_k - l_k), linearised as the edge
 *    covariances' u_e below.  Pose update, per-edge records and stop rule are unchanged.
 *  - Read: an observation with a non-zero weight and at least one free end.  The Z of any other is
 *    not read and may be NaN.  A call that reads none runs exactly as sicp_register_joint_priors.
 *  - Anchoring: a read observation whose six weights are all > 0 joins its two clouds' components
 *    of the edge graph, in both anchoring checks of sicp_register_joint_priors; weaker ones count in
 *    the system only.
 *  - SICP_ERR_BAD_ARG, before any device work, besides sicp_register_joint_priors' checks: n_rel
 *    outside [0, 65535]; a NULL array with n_rel > 0; a cloud id outside [0, n_clouds), a = b, or a
 *    cloud that no edge references; a weight negative or not finite; a read Z with a non-finite
 *    entry, a bottom row other than (0, 0, 0, 1) or |R^T R - I| > 1e-6.
 *  - sicp_get_joint_covariances after this call: N includes the observations' blocks, and s0^2
 *    adds sum_k v_k^T W_k v_k to the numerator and sum_k m_k to the denominator (v_k the linear-model
 *    residual of the final iteration, m_k the non-zero weights of each read observation).        */
int32_t sicp_register_joint_relative(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                                     const int64_t* n /*[h]*/, int32_t n_edges,
                                     const int32_t* fix_id, const int32_t* mov_id /*[h] n_edges*/,
                                     const int32_t* is_fixed /*[h] n_clouds, nonzero: pose held*/,
                                     const double* H0 /*[h] n_clouds x 16 row-major, or NULL: identity*/,
                                     const double* prior_H /*[h] n_clouds x 16 row-major, or NULL*/,
                                     const double* prior_w /*[h] n_clouds x 6, or NULL*/,
                                     int32_t n_rel, const int32_t* rel_a, const int32_t* rel_b /*[h] n_rel*/,
                                     const double* rel_H /*[h] n_rel x 16 row-major*/,
                                     const double* rel_w /*[h] n_rel x 6*/,
                                     const sicp_register_params* p,
                                     double* H_out /*[h] n_clouds x 16*/,
                                     sicp_pair_result* out /*[h] n_edges*/, int64_t* n_selected /*[h] or NULL*/);

/* ---- growing the map and reading it back -------------------------------------------------------
 * sicp_map_insert appends to the map, for every voxel of size voxel_size it does not occupy, the
 * first new point that falls into it.  C is the concatenation of the n_clouds clouds in call
 * order, cloud i moved by H[16 i .. 16 i + 15] (row-major 4 x 4, bit for bit what sicp_transform
 * gives for that cloud and H) or, with H NULL, taken as it is.  key(p) = (floor(p.x / v),
 * floor(p.y / v), floor(p.z / v)) in IEEE double with a real division, compared as doubles.
 * Point C[j] is added iff its three coordinates are finite (NaN / inf points are skipped), no map
 * point has its key and no finite C[j'] with j' < j has its key.  The new map is the old one, in
 * its order, followed by the added points in ascending j; nothing is removed or moved.  The map's
 * grid is rebuilt by sicp_set_map's builder, so the grown map registers exactly as a fresh
 * sicp_set_map of the same points.  n_added[i] (if not NULL) = the points cloud i added.
 *  - SICP_ERR_STATE: no map.  SICP_ERR_BAD_ARG, before any device work: n_clouds < 1, a negative
 *    n[i], a NULL xyz[i] with n[i] > 0 (empty clouds add nothing), a non-finite H entry, a
 *    voxel_size that is not finite and > 0, or n_map + sum n[i] >= 2^32.
 *  - The map is replaced only when the new one is complete: after an error it is unchanged.
 *    Device memory peaks at about two maps plus the staged clouds; the staging buffers (about
 *    100 bytes per point of the largest insert) stay on the context for the next insert.
 *  - The grid builder of sicp_set_map needs finite bounding-box extents, of the finite new points
 *    and of the grown map: points whose coordinates on one axis are more than DBL_MAX apart
 *    (e.g. near +1e308 and -1e308) are refused with SICP_ERR_BAD_ARG ("point cloud contains
 *    non-finite coordinates") after the upload, and the map is unchanged.
 *  - Clears the batch outputs, as sicp_set_map does.
 *  - Each new point walks the map-grid cells its voxel covers: about (v / h + 2)^3 of them for a
 *    map cell size h, so a voxel far larger than the map's cells costs accordingly.
 * sicp_get_map sets *n to the map's size and copies min(*n, cap) points, in map order, into xyz
 * (none when xyz is NULL).  SICP_ERR_STATE: no map.                                              */
int32_t sicp_map_insert(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                        const int64_t* n /*[h]*/, const double* H /*[h] n_clouds x 16, or NULL*/,
                        double voxel_size, int64_t* n_added /*[h] n_clouds, or NULL*/);
int32_t sicp_get_map(sicp_ctx* ctx, double* xyz /*[h|d] cap x 3, or NULL*/, int64_t cap,
                     int64_t* n /*[h]*/);

/* ---- shrinking the map: crop around positions, thin to one point per voxel --------------------
 * sicp_map_crop keeps the map points near any of n_centers centres (x, y, z rows, in the map's
 * frame): with d = p - c rounded in double per axis and d2 = (dx dx + dy dy) + dz dz in double
 * with no fused multiply-add, map point p is kept iff d2 < fl(radius^2) for at least one centre c
 * (the strict comparison of sicp_select_in_range and sicp_map_distances).
 * sicp_map_thin keeps one map point per voxel: with key(p) = (floor(p.x / v), floor(p.y / v),
 * floor(p.z / v)) as sicp_map_insert computes it, map point j is kept iff no map point j' < j has
 * its key.  Thinning a map M thus gives the points of inserting M[1:] into a map of M[:1], and
 * later inserts at the same v keep the map at one point per voxel.
 * Common to both:
 *  - The new map is the kept points in their old order; nothing is moved or reordered.
 *    n_removed (if not NULL) = the points removed.
 *  - When nothing is removed, the map and its grid stay as they are (no rebuild).  Otherwise the
 *    grid is rebuilt by sicp_set_map's builder, so the shrunk map registers and gives distances
 *    exactly as a fresh sicp_set_map of the same points.
 *  - SICP_ERR_STATE: no map.  SICP_ERR_BAD_ARG, before any device work: n_centers < 1, centers
 *    NULL, a non-finite centre coordinate, or a radius / voxel_size that is not finite and > 0.
 *    SICP_ERR_NO_OVERLAP: a crop that would keep no point (a map is never empty).
 *  - The map is replaced only when the new one is complete: after an error it is unchanged.
 *  - Clears the batch outputs, as sicp_map_insert does.
 *  - Device memory peaks at about two maps (the old and the new one, coordinates and grid) plus
 *    8 bytes per map point of keep flags and their prefix sum, which stay on the context like the
 *    insert's staging buffers.
 *  - Cost: the crop is one pass over the map, O(n_map x n_centers) distance tests in the worst case
 *    (a point stops at its first centre within radius), plus the rebuild.  The thin walks, per map
 *    point, the map-grid cells its voxel covers, about (v / h + 2)^3 for a map cell size h, as an
 *    inserted point does, plus the rebuild.                                                      */
int32_t sicp_map_crop(sicp_ctx* ctx, int32_t n_centers, const double* centers /*[h] n_centers x 3*/,
                      double radius, int64_t* n_removed /*[h] or NULL*/);
int32_t sicp_map_thin(sicp_ctx* ctx, double voxel_size, int64_t* n_removed /*[h] or NULL*/);

/* ---- carving the map: remove the map points that rays of clouds pass (free space) --------------
 * sicp_map_carve removes the map points that scans see through: a parked car that has left, a
 * door that was open.  Cloud i is moved by H[16 i .. 16 i + 15] (row-major 4 x 4, bit for bit what
 * sicp_transform gives) or, with H NULL, taken as it is.  Every moved point p with three finite
 * coordinates is a ray from o = origins[3 i .. 3 i + 2] (the map's frame) or, with origins NULL,
 * from H's translation column (H[16 i + 3], H[16 i + 7], H[16 i + 11], taken as they are): where
 * a scan given in its sensor frame was taken.  For a map point m and one ray, every operation is
 * one IEEE double operation rounded on its own, with no fused multiply-add:
 *   d = p - o, u = m - o (per axis), L2 = (dx dx + dy dy) + dz dz, L = sqrt(L2),
 *   s = ((ux dx + uy dy) + uz dz) / L, e2 = ((ux ux + uy uy) + uz uz) - s s;
 *   the ray passes m iff L2 > 0, L2 finite, s > 0, s < L - margin and e2 < fl(radius^2).
 * passes[m] = the rays of this call that pass m (each ray counts once); m is removed iff
 * passes[m] >= min_passes.  Nothing is accumulated across calls.
 *  - margin protects the surfaces the rays end on: a ray meeting a surface at angle a passes within
 *    radius of it over about radius / sin(a) before its end, so surface points are carved where
 *    radius / sin(a) > margin.  min_passes > 1 makes one stray ray harmless.
 *  - The new map is the kept points in their old order; nothing is moved or added.  n_removed (if
 *    not NULL) = the points removed.  passes (if not NULL, any memory kind) receives the n_map
 *    counts of the map as it was, on SICP_OK and on SICP_ERR_NO_OVERLAP.
 *  - When nothing is removed, the map and its grid stay as they are.  Otherwise the grid is
 *    rebuilt by sicp_set_map's builder, so the carved map registers and gives distances exactly
 *    as a fresh sicp_set_map of the same points.
 *  - SICP_ERR_STATE: no map.  SICP_ERR_BAD_ARG, before any device work: n_clouds < 1, a negative
 *    n[i], a NULL xyz[i] with n[i] > 0 (empty clouds cast no ray), a non-finite H entry, origins
 *    and H both NULL, a non-finite origin, a radius that is not finite and > 0, a margin that is
 *    not finite and >= 0, min_passes < 1, or sum n[i] >= 2^32.  SICP_ERR_NO_OVERLAP: the carve
 *    would remove every point (a map is never empty).
 *  - The map is replaced only when the new one is complete: after an error it is unchanged.
 *  - Clears the batch outputs, as sicp_map_crop does; the one-pair state is not touched.
 *  - Cost: each ray walks the map-grid cells within about radius of its first L - margin, one
 *    layer of cells along its major axis at a time: about (L / h + 1) (2 radius / h + 2)^2 cells
 *    for a map cell size h, plus the rebuild when points are removed.
 *  - Device memory: the staging buffers of sicp_map_distances (about 40 B per point), 4 B of
 *    passes per map point and 24 B per cloud, all staying on the context; the keep flags and the
 *    rebuild as for sicp_map_crop (peak about two maps).  Map indices, offsets and counts are
 *    32-bit: n_map < 2^32 as for sicp_set_map and sum n[i] < 2^32, so no count (at most one per
 *    ray) can wrap.                                                                              */
int32_t sicp_map_carve(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                       const int64_t* n /*[h]*/, const double* H /*[h] n_clouds x 16, or NULL*/,
                       const double* origins /*[h] n_clouds x 3, or NULL: the translation column of H*/,
                       double radius, double margin, int32_t min_passes,
                       uint32_t* passes /*[h|d] n_map (the map as it was), or NULL*/,
                       int64_t* n_removed /*[h] or NULL*/);

/* ---- how well clouds fit the map: cloud-to-map distances --------------------------------------
 * sicp_map_distances gives every point of n_clouds clouds its nearest map point within
 * max_distance, and with neighbors = k > 0 its signed distance along that map point's normal.
 *  - Points: cloud i moved by H[16 i .. 16 i + 15] (row-major 4 x 4), bit for bit what
 *    sicp_transform gives for that cloud and H, or with H NULL taken as it is.
 *  - Nearest point: for a point p with three finite coordinates (after the move), the map point
 *    with the smallest squared distance d2 = (dx dx + dy dy) + dz dz (the search's d2 may contract
 *    to fused multiply-adds), the lower map index among ties.  p is within iff d2 < fl(max_distance^2),
 *    the comparison of sicp_select_in_range (cKDTree's distance_upper_bound).  Then idx = that map
 *    index and dist2 = its d2.  A finite point with nothing within the bound gets idx -1 and
 *    dist2 +inf; a point with a NaN or inf coordinate gets idx -1 and dist2 NaN and is not counted.
 *  - neighbors = k > 0: the normal (nx, ny, nz) and planarity of the matched map point m are the
 *    float32 values sicp_estimate_normals(k) gives for m with the map as the fixed cloud (m's k
 *    nearest map points, m included, under option "sign_mode").  plane_dist = ((px - mx) nx +
 *    (py - my) ny) + (pz - mz) nz in double, the float32 normal promoted, no fused multiply-add:
 *    sicp_match's point-to-plane expression, moved point minus map point.  planarity = that
 *    planarity.  Both are NaN where idx is -1.
 *  - n_within[i]: the within points of cloud i.
 *  - A NULL array skips that output and a NULL entry skips that cloud (any memory kind otherwise).
 *  - SICP_ERR_STATE: no map.  SICP_ERR_BAD_ARG, before any device work: n_clouds < 1, a negative
 *    n[i], a NULL xyz[i] with n[i] > 0 (empty clouds are fine), a non-finite H entry, a
 *    max_distance that is not finite and > 0 (an unbounded search is not offered), k neither 0
 *    nor in [2, 64], k above n_map, plane_dist or planarity given with k = 0, or sum n[i] >= 2^32.
 *  - Nothing else changes: the map, the batch outputs (sicp_get_batch_outputs), the one-pair state
 *    (sicp_get_knn, sicp_get_residuals) and sicp_timings' fields except kernel_launches.
 *  - Cost: a bound r walks about (2 r / h + 1)^3 map cells per point, h being the map grid's cell
 *    size; the normals add one k-NN + PCA per within point.  Device memory: the insert's staging
 *    buffers (about 40 B per point) plus 28 B per point and 40 B per within point, and the k-NN
 *    scratch of option "normals_scratch_mb"; they stay on the context like the insert's.        */
int32_t sicp_map_distances(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                           const int64_t* n /*[h]*/, const double* H /*[h] n_clouds x 16, or NULL*/,
                           double max_distance, int32_t neighbors /*0: no normals*/,
                           int64_t* const* idx        /*[h|d] per cloud n[i], or NULL*/,
                           double* const* dist2       /*[h|d] per cloud n[i], or NULL*/,
                           double* const* plane_dist  /*[h|d] per cloud n[i], or NULL*/,
                           float* const* planarity    /*[h|d] per cloud n[i], or NULL*/,
                           int64_t* n_within          /*[h] n_clouds, or NULL*/);

/* ---- which clouds overlap: the overlap graph of many posed clouds --------------------------------
 * sicp_overlap_graph answers, before any registration, which pairs of n_clouds clouds overlap
 * under approximate poses and by how much: the edges of sicp_register_pairs / sicp_register_joint.
 *  - Rule: H[16 c ..] is cloud c's pose (row-major 4 x 4, world <- cloud), or with H NULL every
 *    cloud is in one frame.  For an ordered pair (a, b), a != b, T_ab = H_a^-1 H_b is formed as
 *    sicp_register_joint forms its priors (the transposed rotation, then the product; exactly the
 *    identity with H NULL), and the sample of a is S_a = {0, s, 2 s, ...} < n[a] (X_a[::s] for
 *    s = stride).  count_ab = the points i of S_a whose overlap filter flag is set for the pair
 *    (fixed a, movable b) under T_ab and max_distance r: the n_kept of sicp_set_clouds(X_a, X_b),
 *    sicp_set_selected(S_a), sicp_select_in_range(T_ab, r), bit for bit (the same device search,
 *    d2 < fl(r^2)).
 *  - Output: one row per unordered pair a < b with count_ab + count_ba > 0, ascending in (a, b):
 *    (pair_a, pair_b, count_ab, count_ba).  A pair whose counts are both 0 is never reported.
 *    Empty clouds (n[c] = 0) take part in no pair.  *n_pairs = the number of rows; the first
 *    min(*n_pairs, cap) are written to every output array that is not NULL.  A caller whose cap was
 *    too small calls again with a larger one: the second call recomputes everything.
 *  - Culls: the world boxes of two clouds' grids, grown by r, that do not meet, and a direction
 *    (a, b) whose box (b's grid box mapped by T_ab, grown by r) holds no cell of a's grid, hold no
 *    point within r, up to a proven rounding margin: they are not searched, and nothing they hold
 *    could have been counted.  So the culls never change a count.
 *  - Cost: the clouds' upload and grids (as for sicp_register_pairs), a host sweep of N log N plus
 *    the candidate pairs, and bounded searches: about the sum over the candidate directions (a, b)
 *    of the sampled points of a inside b's cull box.
 *  - SICP_ERR_BAD_ARG, before any device work: n_clouds < 1, a negative n[i], a NULL xyz[i] with
 *    n[i] > 0, a non-finite H entry, an H whose bottom row is not (0, 0, 0, 1) or whose rotation
 *    part R has an entry of R^T R - I above 1e-6, a max_distance that is not finite and > 0,
 *    stride < 1, cap < 0, sum n[i] >= 2^32, or n_pairs NULL.  A cloud with a non-finite coordinate
 *    is refused by the grid builder, as sicp_register_pairs refuses it.
 *  - Nothing else changes: the map, the batch outputs (sicp_get_batch_outputs,
 *    sicp_get_joint_covariances) and the one-pair state.  sicp_timings: upload_ms and grid_fix_ms
 *    are this call's upload and grid build, overlap_ms the rest (culls, count, read-back).
 *  - Limits: the clouds share one grid build, so together they must fit its 2^31 cells (as for
 *    sicp_register_pairs; SICP_ERR_BAD_ARG "batch needs too many grid cells" otherwise).
 *  - Device memory: the clouds once (24 B per point) and their grid (32 B per point of records, the
 *    build's scratch and the cell tables), 4 B per candidate pair and direction counter, and up to
 *    about 72 MB of direction descriptors; all stay on the context for the next call.            */
int32_t sicp_overlap_graph(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz /*[h|d]*/,
                           const int64_t* n /*[h]*/, const double* H /*[h] n_clouds x 16, or NULL*/,
                           double max_distance, int64_t stride,
                           int32_t* pair_a, int32_t* pair_b /*[h] cap each, or NULL*/,
                           int64_t* count_ab, int64_t* count_ba /*[h] cap each, or NULL*/,
                           int64_t cap, int64_t* n_pairs /*[h]*/);

/* ---- the rest of SimpleICP.run's return value (simpleicp.py:316-324) for a batch ----------------
 * sicp_register_batch, sicp_register_to_map, sicp_register_pairs and sicp_register_joint report per pair only the
 * record above.  This call returns what else sicp_register returns, for every pair of the LAST
 * successful call of any of them on this context: X_mov_transformed (transform_by_H, pointcloud.py:205-217, as at
 * simpleicp.py:316), the final distance residuals (simpleicp.py:324, 4th return value), the
 * per-iteration records and the applied transform.  Those two calls only leave these on the
 * device; all the work happens here, and they stay readable (any number of times, same bits)
 * until the next sicp_register_batch, sicp_register_to_map, sicp_register_pairs, sicp_register_joint, sicp_set_map,
 * sicp_map_insert, sicp_map_crop, sicp_map_thin or sicp_map_carve on the context.
 *  - SICP_ERR_STATE: before any such call, after sicp_set_map, sicp_map_insert, sicp_map_crop,
 *    sicp_map_thin or sicp_map_carve, or after a
 *    batch / map / pairs / joint call that returned an error (each of these clears the outputs on
 *    entry; only a successful return of the first four makes them valid).  SICP_ERR_BAD_ARG: n_pairs differs from that call's.
 *  - A NULL array skips that output, a NULL entry skips that pair.  Nothing of a pair whose
 *    status was not SICP_OK (SICP_ERR_NO_OVERLAP included) is ever written.
 *  - mov_xyz_out[i]: pair i's movable cloud (n_mov[i] x 3) moved by the transform the run applied,
 *    bit for bit what sicp_transform gives for that cloud with T[i].
 *  - residuals[i]: the final residuals in kept order (the order of selection), out[i].n_kept
 *    values: those whose two-pass mean / std are out[i].mean_res / std_res.
 *  - log: entry i * max_iterations + j is pair i's record of iteration j for j < out[i].iterations,
 *    zero beyond; max_iterations is that call's run.max_iterations.  As in sicp_register's log,
 *    the last row's mean_res / std_res are the exact two-pass values (out[i]'s).
 *  - T: row-major 4 x 4 transform applied to pair i's cloud (what sicp_get_transform reports after
 *    sicp_register): out[i].H, except under SICP_VARIANT_LINEARIZED_CPP, where H = H * dH is a
 *    different product of the same increments.                                                   */
int32_t sicp_get_batch_outputs(sicp_ctx* ctx, int32_t n_pairs,
                               double* const* mov_xyz_out /*[h|d] per pair n_mov[i] x 3, or NULL*/,
                               double* const* residuals   /*[h|d] per pair out[i].n_kept, or NULL*/,
                               sicp_iter_record* log      /*[h] n_pairs x max_iterations, or NULL*/,
                               double* T                  /*[h] n_pairs x 16, or NULL*/);

/* ---- a-posteriori covariances of a joint registration (DESIGN.md §6.9) ------------------------
 * sicp_get_joint_covariances returns, for the LAST sicp_register_joint on this context, the
 * covariance of every cloud's pose and of every edge's relative pose, all from its final iteration
 * (the last one whose solve ran; its increments gave the returned poses):
 *  - N is that iteration's joint normal matrix over the edges with >= 6 kept rows, unweighted
 *    (after sicp_register_joint_priors also the priors' blocks, and s0 counts their residuals;
 *    after sicp_register_joint_relative also the relative observations', likewise).
 *    s0^2 = sum_e sum_i r_ei^2 / (sum_e n_e - 6 F) over those edges, r_ei the final residuals that
 *    sicp_get_batch_outputs returns and n_e = out[e].n_kept; a denominator <= 0 makes s0 and every
 *    covariance NaN.
 *  - cloud_cov[c] = Cov(u_c), u_c = (omega_c, do_c): the world-frame rotation increment (radians)
 *    and the world displacement of the cloud's origin o_c (the translation of the returned T_c), at
 *    the returned poses.  With y_c the centred unknowns of N (DESIGN.md §6.9) u_c = J_c y_c,
 *    J_c = [[I, 0], [-[o_c - c_w]x, I]] and C_c = s0^2 J_c (N^-1)_cc J_c^T.  A fixed cloud some edge
 *    references gets exact zeros, a cloud no edge references NaN.
 *  - edge_cov[e] = Cov(u_e) for e = (a, b), u_e = (alpha_e, dq_e): the rotation increment of
 *    T_a^-1 T_b in frame-a axes and the displacement of o_b expressed in frame a.  u_e = G_b u_b -
 *    G_a u_a with G_b = diag(R_a^T, R_a^T), G_a = [[R_a^T, 0], [-R_a^T [o_b - o_a]x, R_a^T]], so C_e =
 *    G_b C_bb G_b^T + G_a C_aa G_a^T - G_b C_ba G_a^T - G_a C_ab G_b^T with the cross-covariances
 *    of the two clouds.  Defined for every edge, also one that took no part in the final iteration.
 *  - Row-major 6 x 6 blocks in the variable order above.  The per-edge sigma of out[] stays NaN.
 *  - The first request after the call computes them on the device (sicp_register_joint itself does
 *    no extra work and its timings do not include it); every later one returns the same bits.
 *  - SICP_ERR_STATE whenever sicp_get_batch_outputs would return it, and when the last batched
 *    call was not a sicp_register_joint or ran under option "joint_solver" 1 ("covariances need
 *    joint_solver 0").  SICP_ERR_BAD_ARG: n_clouds or n_edges differs from that
 *    call's.  A NULL output is skipped.  Nothing else changes: the batch outputs, the map and the
 *    one-pair state.                                                                             */
int32_t sicp_get_joint_covariances(sicp_ctx* ctx, int32_t n_clouds,
                                   double* cloud_cov /*[h] n_clouds x 36, or NULL*/, int32_t n_edges,
                                   double* edge_cov /*[h] n_edges x 36, or NULL*/, double* s0 /*[h] or NULL*/);

/* ---- the same covariances under either solver (DESIGN.md §6.14) --------------------------------
 * sicp_get_joint_selected_covariances takes sicp_get_joint_covariances' arguments and returns its
 * outputs under its rule (priors and relative observations included), after a call under either
 * option "joint_solver":
 *  - After a call under 0 it is sicp_get_joint_covariances: the same launches, the same cache and
 *    the same bits, whichever of the two is asked first.
 *  - After a call under 1 it computes the blocks from the sparse solve's factor L of the final
 *    iteration's matrix N' in that solve's unknowns y'_c = (omega_c, u_c), each cloud's increment
 *    about its start origin o_c^0: Z = N'^-1 by Takahashi's recurrence (selected inversion) on the
 *    pattern of L, supernode by supernode from the roots down.  C_c = s0^2 J'_c Z_cc J'_c^T with
 *    J'_c = [[I, 0], [-[o_c - o_c^0]x, I]], equal to the dense J_c (N^-1)_cc J_c^T since y = K y'.
 *    The pattern holds every free cloud's diagonal block and the cross block of every two free
 *    clouds joined by an edge with overlap or a read relative observation.  An edge of two free
 *    clouds that the overlap filter parked before the first iteration may fall outside it: its
 *    cross block is w_a^T w_b, w_c = L^-1 E_c (non-zero only on the elimination-tree path from c's
 *    supernode to its root), exactly 0 for clouds in different components.  Equal to the dense
 *    request up to rounding.
 *  - Device memory after a call under 1: Z and y' together take the factor's bytes (the message of
 *    sicp_register_joint's factor check), allocated on the first request; SICP_ERR_CUDA if that
 *    fails.  SICP_ERR_BAD_ARG (before any launch) for an elimination tree more than 64 levels deep.
 *  - SICP_ERR_STATE and SICP_ERR_BAD_ARG as sicp_get_joint_covariances, without its solver check.
 *    sicp_get_joint_covariances keeps refusing after a call under 1, also after this request. */
int32_t sicp_get_joint_selected_covariances(sicp_ctx* ctx, int32_t n_clouds,
                                            double* cloud_cov /*[h] n_clouds x 36, or NULL*/, int32_t n_edges,
                                            double* edge_cov /*[h] n_edges x 36, or NULL*/,
                                            double* s0 /*[h] or NULL*/);

/* ---- PointCloud.transform_by_H (pointcloud.py:205-217), final application simpleicp.py:316 -- */
int32_t sicp_transform(sicp_ctx* ctx, const double H[16], double* mov_xyz_out /*[h|d] n_mov x 3*/);

/* ---- device timing of the last call of each stage, milliseconds ---------------------------- */
typedef struct {
  double upload_ms, grid_mov_ms, grid_fix_ms, overlap_ms, normals_ms, match_ms, reject_solve_ms,
      transform_ms;
  int64_t kernel_launches; /* kernels of this library launched on this context so far           */
  int64_t fused_iterations; /* last sicp_run / sicp_register: iterations whose reject + solve ran
                               in the barrier-free kernel (all but the first, normally)          */
  int64_t rerun_iterations; /* ... iterations repeated through the general kernel because the
                               order-statistic prediction of the barrier-free kernel missed       */
  double mov_normals_ms;    /* last sicp_register / batched call with mov_neighbors > 0:
                               k-NN + PCA of the movable cloud(s); 0 otherwise                    */
  int64_t overlap_candidates; /* last sicp_register_to_map: bounded searches its culled overlap
                               filter ran (map points inside the scans' grown boxes); 0 without
                               max_overlap_distance                                               */
} sicp_timings;
int32_t sicp_get_timings(sicp_ctx* ctx, sicp_timings* t /*[h]*/);

/* Measurement hook: run `reps` iterations from the current device state and return the average
 * device time (CUDA events on the context's stream) of each kernel group, in milliseconds:
 * ms[0] grid match kernel, ms[1] brute-force pass (launched, usually empty), ms[2] reject+solve
 * kernel, ms[3] whole iteration.  flush_l2 bit 0: overwrite a 256 MiB scratch buffer before every
 * iteration (outside the timed intervals) so each one starts with a cold L2; bit 1: record only
 * the two outer events (ms[0..2] = 0) — the inner events cost several microseconds of stream
 * bubbles per iteration, so the whole-iteration time is taken without them.                     */
int32_t sicp_time_stages(sicp_ctx* ctx, const sicp_run_params* p, int32_t reps, int32_t flush_l2,
                         double ms[4] /*[h]*/);
/* Diagnostics: %globaltimer stamps block 0 took in the last reject+solve kernel, microseconds
 * relative to kernel entry.  [1] median done, [2] MAD done, [3] moments accumulated, [4] grid
 * barrier passed, [5] LM solve done, [6] barrier, [7] residual pass, [8] barrier, [9] exit;
 * [10..12] / [14..16] radix levels done / gather barrier / sort done for the median / MAD;
 * [24],[25] radix levels used, [26],[27] candidates sorted (raw counts, not times; 0 when a
 * predictor select failed and no radix select followed); [28] path:
 * 0 cooperative kernel (radix select), 2 barrier-free kernel (there [2] = select done, [3] =
 * accumulation done in block 0, [4] = serial tail starts, [17] partials reduced, [18] M
 * assembled, [19] solve done, [9] exit).
 * Selection diagnostics (codes, not times; csrc/reject_solve.cuh: SelectPath, SelectOutcome):
 * [29] the selection that produced the last record's median and MAD: 0 radix, 2 per-bin key
 * store of the barrier-free kernel (not written by a barrier-free launch that missed its
 * prediction: the general kernel repeats that iteration); [30] outcome of the predictor select
 * of the last barrier-free launch: 0 used, > 0 the first check that failed.                     */
int32_t sicp_get_phase_times(sicp_ctx* ctx, double us[32] /*[h]*/);

/* Test-only: overwrite the order-statistic predictor (median, MAD and the planarity bound of
 * their population) that the next match bins the distances with, without resetting the loop.
 * The predictor only accelerates the selection: any finite med and mad > 0 must give the same
 * median and MAD, which is what tests use this for.                                            */
int32_t sicp_debug_seed_predictor(sicp_ctx* ctx, double med, double mad, double min_planarity);

/* Test-only: the number of queries the last match answered from the certificate of its warm
 * start (the search skipped because the neighbour provably cannot have changed; DESIGN.md §3.2).
 * 0 when the last match could not use certificates (brute-force engine, match_group 1, no
 * distance).                                                                                    */
int32_t sicp_debug_match_counts(sicp_ctx* ctx, int64_t* n_certified /*[h]*/);

/* Diagnostics: %globaltimer stamps (us, from the first block's entry) of the last one-pair grid
 * match run with the option "match_stamps" set.  Thread 0 of the first block writes slots 0-6,
 * thread 0 of the last block slots 8-14: kernel entry, dependent-launch wait released, state and
 * certificate loaded, certified decision made, normal loaded, histogram atomic returned, exit.
 * Slots 2-5 are only written for a query answered from its certificate; -1 marks a slot not
 * written.                                                                                      */
int32_t sicp_get_match_phase_times(sicp_ctx* ctx, double us[16] /*[h]*/);

/* Test-only: the uniform grid the searches run on.  side 0 = the fixed cloud's grid (k-NN of the
 * normals; built by sicp_estimate_normals), 1 = the movable cloud's grid (correspondences; built
 * by sicp_set_clouds).  o = origin (the cloud's bounding-box minimum), h = cell size, dims = cells
 * per axis; a point v lies in cell floor((v - o) / h) of each axis.  Tests use it to place points
 * relative to the real cell faces.  SICP_ERR_STATE if that grid has not been built.            */
int32_t sicp_debug_grid_params(sicp_ctx* ctx, int32_t side, double o[3] /*[h]*/, double* h /*[h]*/,
                               int32_t dims[3] /*[h]*/);

/* ---- .xyz text I/O (host only; SURVEY.md section 8f: file parsing dominates end-to-end time on
 * the lidar sets).  Contract of the reference readers (c++/src/simpleicp-cli.cpp:72-128,
 * rust/src/io.rs:9-37, np.genfromtxt in python/simpleicp/tests/test_simpleicp.py:102-103):
 * whitespace-separated x y z per line; '/' or '#' comment lines and blank lines are skipped.
 * sicp_xyz_load allocates *xyz (n x 3 float64, row-major); release it with sicp_xyz_free.
 * sicp_xyz_save mirrors PointCloud.write_xyz (python/simpleicp/pointcloud.py:219-226):
 * header != 0 writes the "//X Y Z" line, decimals < 0 writes round-trip precision.            */
int32_t sicp_xyz_load(const char* path, double** xyz /*out*/, int64_t* n /*out*/);
void sicp_xyz_free(double* xyz);
int32_t sicp_xyz_save(const char* path, const double* xyz /*[h] n x 3*/, int64_t n,
                      int32_t decimals, int32_t header);
const char* sicp_io_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* SICP_B200_H */
