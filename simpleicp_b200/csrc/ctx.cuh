// ctx.cuh — the context behind sicp_ctx and the stage entry points each .cu implements.
#pragma once
#include "common.cuh"
#include "grid_plan.h"
#include "joint_plan.h"
#include "reject_solve.cuh"
#include "upload.cuh"

namespace sicp {

// Cell-sorted records and cell table of the clouds of one grid build (grid.cu: grid_build), HBM
// resident (L2 resident for <= ~2M points).
struct GridBufs {
  DevBuf<Rec> recs;              // the points of all clouds, sorted by cell within each cloud
  DevBuf<uint32_t> cell_table;   // every cloud's cells + 1 end sentinel: global record positions
  DevBuf<uint32_t> cid;          // scratch: cell id per point
  DevBuf<uint32_t> fill;         // scratch: per-cell counter
  DevBuf<uint32_t> block_sums;   // scratch for the scan
  void swap(GridBufs& o) {
    recs.swap(o.recs);
    cell_table.swap(o.cell_table);
    cid.swap(o.cid);
    fill.swap(o.fill);
    block_sums.swap(o.block_sums);
  }
  void release() {
    recs.release();
    cell_table.release();
    cid.release();
    fill.release();
    block_sums.release();
  }
};

// One cloud of a grid build (filled by the host from the bounding boxes).
struct CloudPlan {
  const double* xyz;
  long long n;
  long long rec_base;   // position of its first record in the shared record array (= point offset)
  long long cell_base;  // first entry of its cell table in the shared table
  double ox, oy, oz, h, inv_h;
  int nx, ny, nz, pad;
};

// A grid of the one-pair context (sicp_set_clouds, sicp_estimate_normals, sicp_register): one
// cloud under the one-pair cell policy (grid.cu: grid_build_pair).
struct Grid {
  GridBufs bufs;
  GridView view{};
  bool built = false;
};

// Workspace of the fused reject + solve kernel (all device memory).
struct SolveWs {
  DevBuf<unsigned int> hist;        // radix histograms: 2 selects x levels x bins
  DevBuf<unsigned long long> cand;  // candidate keys for the in-block sort, 2 selects
  DevBuf<unsigned int> counters;    // small atomic counters / flags
  DevBuf<unsigned long long> minkey;  // min key above the selected bin, per select
  DevBuf<double> partials;          // per-block partial sums
  DevBuf<double> scal;              // broadcast scalars: median, mad, x, ...
  DevBuf<sicp_iter_record> rec;     // device copy of the per-iteration record ring
};

// Scratch of the ordered compactions (grid.cu: scan_u32, compact_bounds, compact_scatter) of the
// overlap filters, the map calls and the residuals.  Calls on one context run one after the other,
// so they share it; DevBuf::reserve drops what a buffer held, so a call reserves flag and scan
// before it writes its first flag.
struct CompactScratch {
  DevBuf<uint32_t> flag;    // uint32 flags (or counts) of one compaction
  DevBuf<uint32_t> scan;    // their exclusive prefix sum, n + 1 entries
  DevBuf<uint32_t> sums;    // the scan's block sums
  DevBuf<uint32_t> bounds;  // the boundaries picked from the scan
  uint32_t* host = nullptr; // pinned: the boundaries read back
  size_t host_cap = 0;
};

struct Batch;
struct MapStore;
struct OverlapStore;

struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  int num_sms = 132;
  std::string err;

  // options
  int nn_engine = SICP_NN_AUTO;
  int sign_mode = SICP_SIGN_DGEEV;
  int variant = SICP_VARIANT_PYTHON;
  double grid_target_occ = 3.0;
  int grid_max_rings = 8;
  int host_sync_every = 4;
  int grid_sort_cells = 0;  // 1: sort the records inside each cell by index (layout only)
  int match_group = 0;   // lanes cooperating on one grid query: 0 = by K, else 1, 4, 8 or 16
  int joint_solver = 0;  // sicp_register_joint's solve: 0 dense (k_joint_solve), 1 sparse (k_joint_sparse_solve)

  // clouds
  DevBuf<double> fix_xyz, mov_xyz;
  long long n_fix = 0, n_mov = 0;
  DevBuf<float4> mov_f4;  // centred float copy in caller order, for the TMA brute-force engine
  double mov_center[3] = {0, 0, 0};
  double mov_radius = 0;  // max |centred coordinate|
  Grid gmov, gfix;

  // selection (ascending fixed-cloud indices) and per-query data
  long long K = 0;
  DevBuf<long long> sel_idx;
  DevBuf<long long> sel_tmp;
  DevBuf<double> q_xyz;   // K x 3 gathered fixed points
  DevBuf<float4> q_nrm;   // (nx, ny, nz, planarity) float32 as the reference stores them
  bool have_normals = false;
  // movable-side attributes (sicp_set_mov_normals): per movable point, in its own frame
  DevBuf<float4> mov_nrm;
  DevBuf<float4> q_nrm_eff;  // K: fixed normal + effective planarity of the current match (nn.cu: effective_planarity)
  bool mov_attr = false;
  double mov_cos_max = -1.0; // cos(max angle between normals); < 0 = no angle test
  int knn_k = 0;
  DevBuf<long long> knn_idx;
  DevBuf<double> knn_d2;
  DevBuf<uint32_t> knn_pos;  // K x k record positions (cooperative k-NN kernel -> PCA kernel)
  int keep_knn = 0;          // option "keep_knn": store neighbour indices / distances for sicp_get_knn
  int knn_coop = -1;         // option "knn_coop": 1 cooperative lanes (k <= 16), 0 one thread per query, -1 by K
  int normals_scratch_mb = 64;  // option "normals_scratch_mb": bound of the movable-normals estimate's neighbour scratch

  // per-iteration arrays
  DevBuf<long long> nn_idx;
  DevBuf<double> dist;
  DevBuf<uint8_t> keep;
  DevBuf<unsigned long long> binstore;  // LH_BINS x bin_cap: distance keys of the members of every predictor-histogram bin (match -> fused reject/solve)
  int bin_cap = 0;
  DevBuf<double> m_xyz;              // K x 3: matched movable point, caller coordinates
  DevBuf<uint32_t> nn_pos;           // K: record position of the last match (warm start of the next one)
  // nn_pos, cert_c, cert_rho, m_xyz and nn_idx were all written by the last match with distance,
  // on the current movable grid and selection.  The certificates make this a correctness
  // contract, not a hint: a match answered from a certificate returns m_xyz and nn_idx as they
  // are.  Whatever rebuilds gmov, changes the selection or writes m_xyz or nn_idx outside such a
  // match must clear the flag.
  bool nn_pos_valid = false;
  long long nn_pos_K = 0;
  // certificates of the one-pair grid match (nn.cu: MatchCert), 28 B per query, valid with nn_pos
  DevBuf<double> cert_c;             // K x 3
  DevBuf<float> cert_rho;            // K
  DevBuf<unsigned int> cert_count;   // 2: queries answered from a certificate, by launch parity
  int cert_next = 0;                 // counter of the next certifying launch
  int cert_slot = -1;                // counter of the last match; -1: it could not certify
  DevBuf<unsigned long long> match_t;  // 16 %globaltimer stamps of the one-pair match (MatchCert::stamps)
  int match_stamps = 0;              // option "match_stamps": the one-pair match writes match_t
  int warm_start = 1;                // option "warm_start"
  int sphere_scan = 1;               // option "sphere_scan"
  int pdl = 1;                       // option "pdl": programmatic dependent launch between the two kernels of an iteration
  bool unresolved_clean = false;     // unresolved[K] is zero: the reject/solve kernel that read it last reset it
  DevBuf<double> resid;          // K, valid where keep
  DevBuf<double> resid_compact;  // kept order
  DevBuf<unsigned int> unresolved;  // query ids the grid could not bound + counter at [K]
  DevBuf<unsigned char> bf_scratch;
  long long n_kept = 0;
  bool matched = false, rejected = false, solved = false;
  bool expect_unresolved = true;  // last known: did some query exceed the ring limit?
  double min_planarity_last = 0.0;

  // last solve state (for uncertainties)
  double last_x[6] = {0, 0, 0, 0, 0, 0};
  double last_T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};  // transform applied to the movable cloud
  double last_sigma[6] = {0, 0, 0, 0, 0, 0};
  sicp_lsq_params last_lsq{};

  SolveWs ws;
  DevBuf<DevState> dev_state;
  int rs_parity = 0;
  CompactScratch compact;
  // grid build scratch (grid.cu: grid_build), kept apart from the select workspace
  DevBuf<unsigned long long> bbox_keys;   // 6 per cloud
  DevBuf<unsigned int> grid_occ;          // occupied cells per cloud
  DevBuf<CloudPlan> grid_plans;           // the plan table of a build of several clouds
  unsigned long long* grid_host = nullptr;  // pinned: bounding-box keys, then occupancies
  size_t grid_host_cap = 0;
  DevBuf<unsigned int> misc_counters;     // API scratch counters
  DevBuf<unsigned char> flush_buf;        // 256 MiB scratch for cold-L2 measurements
  DevBuf<unsigned long long> phase_t;     // %globaltimer stamps of the reject/solve kernel
  DevBuf<unsigned int> grid_bar;          // grid barrier of the cooperative reject/solve kernel
  DevBuf<unsigned int> lin_hist;          // predictor histogram (match kernels -> reject kernel)
  bool lin_hist_pending = false;          // filled by a match, not yet consumed by a reject
  bool lin_hist_init = false;
  bool rsb_attr_set = false;
  bool rs_attr_set = false;               // k_reject_solve's dynamic shared memory limit raised on this device
  bool rsf_attr_set = false;              // k_rs_fused's dynamic shared memory limit raised on this device
  DevBuf<RsSelect> rs_sel;                // k_rs_fused -> k_rs_solve
  DevBuf<RsScratch> rs_scratch;           // stores of k_rs_solve's rehearsal
  int n_fused_last = 0, n_rerun_last = 0; // last run: iterations through k_rs_fused / repeated after a missed prediction
  int fused = 1;                          // option "fused": 0 = always the cooperative kernel
  bool bf_attr_set = false;               // k_bf_nn's dynamic shared memory limit raised on this device
  sicp_iter_record* rec_host = nullptr;  // pinned
  double* scal_host = nullptr;           // pinned staging for small reads
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t copy_stream = nullptr;   // second stream: fixed-cloud upload overlaps the movable grid build
  PageableUploader up;                  // clouds in pageable host memory (NumPy arrays): threaded staging, upload.cuh
  int upload_threads = 2;               // option "upload_threads": 0 = plain cudaMemcpyAsync for every source (measured: 2, 3, 4 threads alike, tools/upload_probe.py)
  cudaEvent_t ev_copy = nullptr, ev_user = nullptr;
  sicp_timings tm{};

  // staging for host inputs
  DevBuf<unsigned char> stage;

  Batch* batch = nullptr;  // created by the first sicp_register_batch
  MapStore* map = nullptr; // sicp_set_map: the resident fixed cloud of sicp_register_to_map
  OverlapStore* ovl = nullptr;  // created by the first sicp_overlap_graph
};
// what the match kernels / reject kernels see of the movable-side attributes
inline const float4* mov_attr_nrm(Ctx& c) { return c.mov_attr ? c.mov_nrm.p : nullptr; }
inline float4* mov_attr_eff(Ctx& c) {
  if (!c.mov_attr) return nullptr;
  c.q_nrm_eff.reserve(c.K > 0 ? c.K : 1);
  return c.q_nrm_eff.p;
}

// ---- batched engine: many small pairs per launch (BASELINE configs[4], SURVEY.md section 8e) ----
// One descriptor per pair, resident in device memory; every batched kernel takes the pair from
// blockIdx.y (or blockIdx.x for the one-block-per-pair kernels) and reads its descriptor.
struct PairDev {
  GridView gmov, gfix;
  long long n_fix, n_mov;
  long long fix_off, mov_off;  // first point of this pair's clouds in the concatenated clouds
  // first overlap keep flag of this pair (Ctx::compact.flag, one per fixed point of the pair): the
  // fixed points of the pairs before it (0 on the map path, whose filter has its own bit rows)
  long long flag_off;
  long long K;                 // selected fixed points (<= Kmax)
  long long q_off;             // first entry of this pair in the per-query arrays
  double cm[3];                // centre of the movable grid's box (moment centring)
  // overlap filter: this pair's survivors are Batch::ovl_list[list_off, list_off + list_len), each
  // its fixed point's flag position flag_off + i (i: index in the fixed cloud)
  long long list_off, list_len;
  double obs[6];               // rbp_observed_values of this pair (radians)
};

// ---- sicp_register_joint (joint.cu): one edge of the joint problem per pair of the batch ----
constexpr int JE_NSUM = 36;  // N (21, packed lower), sum a d (6), sum a (6), sum d, sum d^2, count
constexpr int JOINT_MAX_FREE = 256;
constexpr int JOINT_SEL_MAX_PATH = 64;  // the selected inversion: elimination-tree depth, at most
constexpr int JOINT_MAX_PAD = 1568;  // 6 JOINT_MAX_FREE + 1 rounded up to the 32-wide tiles
// What k_joint_reject leaves of edge e = (a, b) for the solve and the update: the sums of its
// kept rows a = [w x n, n] (centred about c_f in frame a), its world block Nw = Ad^T N Ad and
// right-hand side gw = -Ad^T h, and Ad's inputs (cloud a's rotation, v = T_a c_f - c_w).
struct JointEdge {
  double N[21], h[6], s[6], sd, sd2;
  double Nw[36], gw[6];
  double Ra[9], v[3], cf[3];
  long long n;
  int part;  // >= 6 kept rows this iteration: the edge enters the joint system
  int pad;
};
// A pose prior of free cloud f that the call reads (DESIGN.md §6.12): the observed pose P and the
// weights w in world axes; per iteration k_joint_prior leaves the observation l = (rotvec(R_P R_c^T),
// o_P - o_c), the lever d of J_c = [[I, 0], [-[d]x, I]] in the unknowns of the solve in use, and the
// cloud's block Nw = J^T W J and right-hand side gw = J^T W l; k_joint_solve leaves the cloud's
// unknowns y (the covariances' residual v = J y - l).
struct JointPrior {
  Rigid P;
  double w[6];
  double Nw[36], gw[6];
  double l[6], lev[3], y[6];
  int f, pad;
};
// A relative pose observation the call reads (DESIGN.md §6.13): clouds ca and cb (free indices fa,
// fb; -1 for a fixed end), the observed Z of T_a^-1 T_b and the weights w in frame-a axes.  Per
// iteration k_joint_relative leaves the observation l = (rotvec(R_Z R_ab^T), t_Z - t_ab) and, with
// B_c = G_c J_c in the unknowns of the solve in use, the blocks N[0] = B_a^T W B_a, N[1] = B_b^T W B_b,
// N[2] = -B_b^T W B_a (rows b, columns a) and right-hand sides g[0] = -B_a^T W l, g[1] = B_b^T W l
// (a fixed end's left unset), and for the covariances' residual v = B_b y_b - B_a y_a - l the levers
// of J_a and J_b, o_b - o_a and R_a.
struct JointRel {
  Rigid Z;
  double w[6];
  double N[3][36], g[2][6];
  double l[6], lev[2][3], dba[3], Ra[9];
  int ca, cb, fa, fb;
};
// The relative observations of a call for the solves (all null / 0 without them): per block of the
// solve in use (the dense solve's blk_of blocks, the sparse solve's panel lists) its observations
// k[off[b] ..] in ascending order; y: per free cloud, 6 doubles, the dense solve's unknowns of the
// iteration (for the covariances)
struct JointRelArgs {
  JointRel* rel;
  const int* off;
  const int* k;
  double* y;
  int n;
};
struct JointFlags {
  int done;       // converged, last iteration or singular: every later queued kernel returns
  int converged;
  int singular;
  int pad;
};
struct JointArgs {
  const PairDev* pairs;
  DevState* state;  // per edge: R_e = T_a^-1 T_b in T / Tinv, the record state
  JointEdge* edges;
  JointFlags* flags;
  const double* dist;
  const float4* q_nrm;
  const double* m_xyz;
  uint8_t* keep;
  sicp_iter_record* rec;  // n_edges x rec_stride
  int rec_stride;
  int it, last;
  Rigid* pose;             // per cloud, world <- cloud
  const int* fix_id;       // per edge: cloud a
  const int* mov_id;       // per edge: cloud b
  const int* free_of;      // per cloud: index among the free clouds, -1
  const int* free_ids;     // per free cloud: its cloud
  // lower blocks (p >= q) of the joint matrix that some edge touches: blk_of[p F + q] indexes
  // blk_off; blk_edge[blk_off[b] ..] lists its edges ascending as 2 e + (1: cloud p is the edge's a)
  const int* blk_of;
  const int* blk_off;
  const int* blk_edge;
  int F, n_edges, npad;
  double* A;               // npad x npad, row-major, the lower triangle is used
  unsigned int* bar;       // grid barrier of k_joint_solve, {0, any} between launches
  double cw[3];            // the common world centre of the increments
  double min_planarity, min_change;
  // the pose priors the call reads (DESIGN.md §6.12), and per free cloud its prior or -1; both null
  // without priors
  JointPrior* prior;
  const int* prior_of;
  int n_prior;
};
// One supernode of the sparse solve's plan (joint_plan.h): its clouds at positions first ..
// first + ns - 1, its struct st[st_off .. st_off + nt), its updates [u0, u1) and the offset of its
// panel block table.
struct JointSuper {
  int first, ns, nt, st_off, u0, u1, table, pad;
};
// k_joint_sparse_solve (option "joint_solver" 1): the plan of joint_plan.h on the device.  j is read
// as k_joint_solve reads it, except blk_of / blk_off / blk_edge, npad and A.
struct JointSparseArgs {
  JointArgs j;
  const JointSuper* sn;
  const long long* panel;  // per supernode: offset of its column-major panel in L, in doubles
  const int* st;           // the structs (positions)
  const int* up;           // per update, 4 ints: descendant, first struct entry used, entries inside s, map offset
  const int* map;          // the row maps of the updates: panel cloud rows of s
  const int* lv_off;       // depth + 1
  const int* lv;           // the supernodes by level
  const int* perm;         // position -> free cloud
  // panel block (cloud row ri, cloud column cj) of supernode s: list blk[table + ri ns + cj] of
  // lst_edge[lst_off[list] ..] (2 e + (1: the cloud is the edge's a)), -1 for none or above the diagonal
  const int* blk;
  const int* lst_off;
  const int* lst_edge;
  // per free cloud, 3 doubles: the origin of its start pose minus c_w.  The system is solved for
  // each cloud's increment about that origin, assembled from the edges' sums with levers of metres
  // (the same solution as about c_w, DESIGN.md §6.11), and carried back to c_w for the update
  const double* dc;
  int depth;
  double* L;               // the panels
  double* x;               // 6 F: L^T x = y by positions, the working values of the back substitution
  double* xf;              // 6 F: the solution in free-cloud order
  int* bad;                // [1] a non-positive or non-finite pivot (0 between calls)
  int* conv;               // per block: its edges met the stop rule
  JointRelArgs r;          // off / k by the lists of lst_off; y unused
};
// sicp_get_joint_covariances (joint.cu: joint_cov_launch), from what the final iteration of the
// last sicp_register_joint left: the factor L of its joint matrix (upper-left n x n of A), the
// edges' final kept rows and residuals, and the returned poses.
struct JointCovArgs {
  const PairDev* pairs;
  const DevState* state;
  const uint8_t* keep;
  const double* m_xyz;
  const double* q_xyz;
  const float4* q_nrm;
  const JointEdge* edges;
  const Rigid* pose;
  const int* fix_id;
  const int* mov_id;
  const int* free_of;
  const int* free_ids;
  const double* L;    // npad x npad, row-major, lower triangle
  double* Z;          // npad x npad: L^-1 in the lower triangle of the first n rows and columns
  double* ss;         // per edge: sum of squared final residuals (0 for an edge that took no part)
  double* s0sq;       // [1]: s0^2 (NaN when the redundancy is <= 0)
  double* cov_f;      // per free cloud: C_c, row-major 6 x 6
  double* cov_e;      // per edge: C_e
  unsigned int* bar;  // grid barrier of k_joint_inv, {0, any} between launches
  int F, n_edges, npad;
  double cw[3];
  const JointPrior* prior;  // the pose priors of the call (their v^T W v and count enter s0^2)
  int n_prior;
  const JointRel* rel;      // the relative observations of the call and the final unknowns y (the
  const double* rel_y;      // same for them, DESIGN.md §6.13)
  int n_rel;
};
// sicp_get_joint_selected_covariances after a call under joint_solver 1 (joint.cu: joint_sel_launch,
// DESIGN.md §6.14): Z = N'^-1 on the pattern of the final iteration's factor s.L, by supernodes.
struct JointSelArgs {
  JointSparseArgs s;   // the plan, the factor, xf, dc and the grid barrier of the call
  JointCovArgs c;      // ss, s0sq, cov_f, cov_e and what k_joint_cov_ss reads (L, Z, npad unused)
  double* Z;           // supernode k's block of Z at panel[k] - 6 first[k]: 6 (ns + nt) x 6 ns, column-major
  double* y;           // 6 F: the final iteration's unknowns y' = (omega, u) about each start origin
  const int* pos;      // per free cloud: its position in the plan's order
  const int* parked;   // the edges of two free clouds whose cross block lies outside the pattern
  int n_parked;
  long long scratch;   // doubles of Z per block of k_joint_sel_parked, before Z is formed
};
struct JointStore {
  DevBuf<JointEdge> edges;
  DevBuf<JointFlags> flags;
  DevBuf<Rigid> pose;
  DevBuf<int> ids;  // fix_id, mov_id, free_of, free_ids, blk_of, blk_off, blk_edge
  DevBuf<double> A;
  DevBuf<unsigned int> bar;
  DevBuf<JointPrior> prior;
  int n_prior = 0;  // the pose priors of the last call
  DevBuf<JointRel> rel;
  DevBuf<double> rel_y;
  int n_rel = 0;    // the relative observations of the last call
  // the sparse solve (joint_solver 1): its panels, x, xf and dc (15 F), bad + one flag per block
  bool sparse = false;  // the last call used it (covariances by sicp_get_joint_selected_covariances)
  JointPlan sp_plan;           // its plan and solve arguments, for the selected inversion
  JointSparseArgs sp_args{};
  DevBuf<int> sel_ids;  // the selected inversion's pos and parked edges
  DevBuf<long long> sp_panel;
  DevBuf<double> sp_L, sp_x;
  DevBuf<int> sp_flags;
  JointFlags* flags_host = nullptr;  // pinned
  // what sicp_get_joint_covariances needs of the last call (set by joint_loop), and its cache:
  // per cloud and per edge row-major 6 x 6 blocks and s0, computed by the first get after the call
  int n_clouds = 0, n_edges = 0, F = 0, npad = 0;
  double cw[3] = {0, 0, 0};
  std::vector<char> role;  // per cloud: 0 no edge references it, 1 fixed, 2 free
  DevBuf<double> Z, cov;   // cov: ss (n_edges), s0^2 (1), C_c (F x 36), C_e (n_edges x 36)
  bool cov_done = false;
  std::vector<double> cov_cloud, cov_edge;
  double s0 = 0.0;
  ~JointStore() {
    if (flags_host) cudaFreeHost(flags_host);
  }
};
void joint_reject_launch(Ctx& c, const JointArgs& a, int n_edges);
void joint_solve_launch(Ctx& c, const JointArgs& a, const JointRelArgs& r);
void joint_sparse_solve_launch(Ctx& c, const JointSparseArgs& a);
// k_joint_prior: the blocks of a.n_prior pose priors at the current poses, in the unknowns of the
// dense solve (dc null) or of the sparse solve (dc: its per-free-cloud start origins minus c_w)
void joint_prior_launch(Ctx& c, const JointArgs& a, const double* dc);
// k_joint_relative: the blocks of r.n relative observations at the current poses, in the unknowns of
// the dense solve (dc null) or of the sparse solve
void joint_relative_launch(Ctx& c, const JointArgs& a, const JointRelArgs& r, const double* dc);
// k_joint_cov_ss, k_joint_inv, k_joint_cov_cloud, k_joint_cov_edge: the covariances of the last
// sicp_register_joint into a.cov_f / a.cov_e and s0^2 into a.s0sq (DESIGN.md §6.9)
void joint_cov_launch(Ctx& c, const JointCovArgs& a);
// k_joint_cov_ss, k_joint_sel_parked (parked_blocks > 0), k_joint_selinv, k_joint_sel_s0,
// k_joint_sel_cloud, k_joint_sel_edge: the covariances of the last sicp_register_joint under
// joint_solver 1 into a.c.cov_f / a.c.cov_e and s0^2 into a.c.s0sq (DESIGN.md §6.14)
void joint_sel_launch(Ctx& c, const JointSelArgs& a, int parked_blocks);

struct Batch {
  int n_pairs = 0;
  // total_fix: the fixed points of all pairs (overlap flags); total_mov: the points of the movable
  // clouds, the prefix of xyz; max_n_mov: the largest movable cloud
  long long Kmax = 0, total_fix = 0, total_mov = 0, max_n_mov = 0;
  // every cloud of the call once (batch.cu: register_pairs); gfix holds the grids of the clouds
  // fixed in some pair, which serve both roles, gmov those of the movable-only clouds
  DevBuf<double> xyz;
  GridBufs gfix, gmov;
  DevBuf<PairDev> pairs;
  // the movable-normals estimate runs over n_mov_desc descriptors: the pairs' own (mov_desc =
  // pairs), or with shared clouds one per distinct movable cloud (mov_desc = mov_pairs)
  DevBuf<PairDev> mov_pairs;
  const PairDev* mov_desc = nullptr;
  int n_mov_desc = 0;
  // per-query arrays, n_pairs x Kmax
  DevBuf<long long> sel_idx, nn_idx;
  DevBuf<double> q_xyz, dist, m_xyz;
  DevBuf<float4> q_nrm;
  // movable-side attributes (mov_neighbors > 0): per movable point of the batch (total_mov), in its
  // own frame, and the fixed normal + effective planarity of each match (n_pairs x Kmax)
  DevBuf<float4> mov_nrm, q_nrm_eff;
  bool mov_attr = false;
  double mov_cos_max = -1.0;
  DevBuf<uint32_t> knn_pos;        // n_pairs x Kmax x k (the movable-normals estimate reuses it)
  DevBuf<unsigned long long> binstore;  // n_pairs x LH_BINS x bin_cap
  int bin_cap = 0;
  DevBuf<uint32_t> nn_pos;
  DevBuf<uint8_t> keep;
  // overlap filter: the survivors of every pair in ascending order (PairDev::list_off)
  DevBuf<uint32_t> ovl_list;
  // per-pair state
  DevBuf<DevState> state;
  DevBuf<unsigned int> lin_hist;       // n_pairs x (LH_BINS + 2)
  DevBuf<sicp_iter_record> rec;        // n_pairs x max_iterations
  DevBuf<double> partials;             // n_pairs x RSF_NPART (+ slack)
  DevBuf<unsigned long long> phase_t;  // 32 (diagnostics of pair 0)
  DevBuf<int> flags;                   // n_pairs x 2: {stop, iterations_done}
  DevBuf<sicp_pair_result> results;
  int* flags_host = nullptr;                 // pinned
  sicp_pair_result* results_host = nullptr;  // pinned
  size_t flags_cap = 0, results_cap = 0;
  // What sicp_get_batch_outputs reads of the last sicp_register_batch / sicp_register_to_map /
  // sicp_register_pairs.  out_valid is cleared on entry of those calls and of the calls that
  // replace the map, and set only when one of the three returns successfully; the vectors are per
  // pair of that call.
  bool out_valid = false;
  bool out_joint = false;  // that call was a sicp_register_joint (sicp_get_joint_covariances)
  int out_n_pairs = 0, out_max_iterations = 0;
  std::vector<long long> out_n_mov, out_n_kept;  // movable points, kept residuals
  std::vector<int> out_status, out_iterations; // sicp_status (SICP_ERR_NO_OVERLAP included), iterations run
  std::vector<double> out_mean_std;            // exact mean / std of the final residuals, 2 per pair
  // buffers of sicp_get_batch_outputs: transformed clouds and compacted residuals of the requested
  // pairs, each pair at its own output offset (pairs may share a movable cloud), the ids and the
  // output offsets of the requested pairs
  DevBuf<double> xyz_out, resid_out;
  DevBuf<int> out_ids;
  DevBuf<long long> out_off;
  sicp_iter_record* rec_host = nullptr;      // pinned: the downloaded log
  size_t rec_cap = 0;
  Rigid* T_host = nullptr;                   // pinned: DevState::T of every pair
  size_t T_cap = 0;
  JointStore joint;                          // sicp_register_joint's buffers
  ~Batch() {
    if (flags_host) cudaFreeHost(flags_host);
    if (results_host) cudaFreeHost(results_host);
    if (rec_host) cudaFreeHost(rec_host);
    if (T_host) cudaFreeHost(T_host);
  }
};

// Box of one scan's overlap cull in the map frame (host-computed, batch.cu: map_cull_box): the
// map-grid cells [c0, c1] per axis and the coordinate box [lo, hi] the candidates must lie in.
struct MapCull {
  double lo[3], hi[3];
  int c0[3], c1[3];
  long long rows;  // (c1[1] - c0[1] + 1) (c1[2] - c0[2] + 1), 0 = no candidate
};

// The resident fixed cloud of sicp_register_to_map (sicp_set_map): its coordinates and ONE grid,
// built by grid_build with the map as its only cloud and the batch cell policy, so that its cell
// plan is the one a batch would make for it.  Every pair of a sicp_register_to_map call takes
// `view` as its fixed grid, with fix_off = 0.
struct MapStore {
  DevBuf<double> xyz;
  GridBufs grid;
  GridView view{};
  long long n = 0;
  // overlap filter: one bit per (scan, map point); its per-word popcounts and their prefix sum are
  // a compaction of the context (Ctx::compact)
  DevBuf<uint32_t> bits;
  DevBuf<unsigned long long> n_searched;  // bounded searches of the last filter
  DevBuf<MapCull> culls;                  // one per scan
  // sicp_map_insert (batch.cu: map_insert): the clouds of one call, moved and concatenated
  // (ins_xyz, cloud i from ins_off[i]), their finite points compacted in order (fin_xyz, with
  // their index in ins_xyz in fin_idx) and gridded as one cloud (gnew).  The flags of both
  // compactions are the context's (Ctx::compact).  These staging buffers grow to the largest
  // insert (about 100 B per point with the compaction scratch) and stay allocated, also across sicp_set_map, like the batch's
  // buffers.  xyz_next / grid_next receive the grown map, which is then swapped in; they are
  // released after the swap, so an insert's peak is about two maps and one map stays resident
  // between inserts.
  DevBuf<double> ins_xyz, fin_xyz, xyz_next;
  DevBuf<uint32_t> fin_idx, ins_off;
  DevBuf<Rigid> ins_T;
  GridBufs gnew, grid_next;
  // sicp_map_distances (batch.cu: map_distances) stages its clouds in ins_xyz (with ins_off,
  // ins_T) and compacts its within flags in Ctx::compact.  Its own buffers, per staged point: the
  // map index and d2 of the nearest map point, and with normals the plane distance and planarity
  // (28 B); per within point: the matched map point's coordinates and its (normal, planarity)
  // (40 B); and the k-NN positions of one chunk of option "normals_scratch_mb".  They stay
  // allocated like the insert's staging buffers.
  DevBuf<long long> dst_idx;
  DevBuf<double> dst_d2, dst_plane, dst_mxyz;
  DevBuf<float> dst_pl;
  DevBuf<float4> dst_nrm;
  DevBuf<uint32_t> dst_pos;
  // sicp_map_crop / sicp_map_thin (batch.cu: map_crop, map_thin) compact a keep flag per map
  // point in Ctx::compact into xyz_next; crop_c holds the crop's centres.
  DevBuf<double> crop_c;
  // sicp_map_carve (batch.cu: map_carve) stages its clouds as sicp_map_distances does; carve_o
  // holds one origin per cloud and carve_passes one count per map point (4 B); both stay
  // allocated like the staging buffers, and the keep flags are compacted as the crop's are.
  DevBuf<double> carve_o;
  DevBuf<uint32_t> carve_passes;
};

// One direction (a, b) of sicp_overlap_graph that survived the culls (batch.cu: overlap_graph):
// the rows of a's grid inside cull, searched in b's grid under the DevState of the same index
// (T = T_ab); the survivors are counted into counts[slot].
struct OverlapDir {
  MapCull cu;
  int a, b;  // indices into the call's grid views
  int slot;  // 2 p (count_ab) or 2 p + 1 (count_ba) of candidate pair p
  int pad;
};

// sicp_overlap_graph's buffers, kept on the context like sicp_map_distances' staging: every
// non-empty cloud once (24 B per point) and its grid, the grid views, the directions' states and
// descriptors, and two 32-bit counters per candidate pair.  Nothing in them outlives the call.
struct OverlapStore {
  DevBuf<double> xyz;
  GridBufs grid;
  DevBuf<GridView> views;
  DevBuf<unsigned char> dirs;  // n_dirs DevState, then n_dirs OverlapDir: one upload
  DevBuf<uint32_t> counts;
  uint32_t* counts_host = nullptr;  // pinned
  size_t counts_cap = 0;
  ~OverlapStore() {
    if (counts_host) cudaFreeHost(counts_host);
  }
};

// ---- stage entry points (each implemented in its own translation unit) ---------------------
struct HostCloud {
  const double* xyz_dev;
  long long n;
  long long point_off;  // first record of this cloud in the shared record array
};
// The grids of clouds in g, one segmented counting sort; views[i] is cloud i's grid, centres
// (3 per cloud) the centre o + 0.5 dims h of its box.  Cell sizes follow the policy (grid_plan.h).
void grid_build(Ctx& c, GridBufs& g, const std::vector<HostCloud>& clouds, const CellPolicy& policy,
                std::vector<GridView>& views, std::vector<double>& centres);
// one cloud under the one-pair cell policy, into a grid of the one-pair context
void grid_build_pair(Ctx& c, Grid& g, const double* xyz_dev, long long n);
void make_float4_copy(Ctx& c);
// Exclusive prefix sum of n uint32 or uint8 values (four launches): out[0 .. n], out[n] = the
// total.  block_sums is scratch.
void scan_u32(Ctx& c, const uint32_t* in, long long n, uint32_t* out, DevBuf<uint32_t>& block_sums);
void scan_u32(Ctx& c, const uint8_t* in, long long n, uint32_t* out, DevBuf<uint32_t>& block_sums);
// Ordered compaction of the elements j < n with flag[j] != 0, scan = the flags' exclusive prefix
// sum (scan_u32), on the scratch Ctx::compact.
// compact_bounds: scan[off[i]] for every offset (each <= n), read back; the returned pinned array
// holds them until the next call.
const uint32_t* compact_bounds(Ctx& c, const uint32_t* scan, const std::vector<long long>& off);
// compact_scatter: element j goes to o = scan[j]; pos[o] = j, and row o of the output takes row
// from[j] (row j without from) of the source, rows of 3 doubles for uint32 flags and of 1 double
// for uint8 flags.  A null pos or output is not written.
void compact_scatter(Ctx& c, const uint32_t* flag, long long n, const uint32_t* scan, uint32_t* pos,
                     const double* xyz, const long long* from, double* xyz_out);
void compact_scatter(Ctx& c, const uint8_t* flag, long long n, const uint32_t* scan, long long* pos,
                     const double* src, double* out);

// 1-NN of K transformed queries into the movable cloud; fused point-to-plane distance.
// If out_d2 != nullptr the squared NN distance is written instead of the plane distance epilogue
// being required (overlap filter).
// The transform is read from c.dev_state (T, Tinv) on the device.
// allow_bf: bound the ring expansion by grid_max_rings and answer the rest with the brute-force
// pass; otherwise the grid search runs to completion on its own (no extra launches).
// in_loop: called from launch_iteration — the counter of unresolved queries was reset by the
// previous iteration's reject/solve kernel (no memset between the kernels), and the kernel may be
// launched programmatically dependent on it (option "pdl").
void match_launch(Ctx& c, bool with_distance, double* out_d2, cudaEvent_t mid = nullptr,
                  bool allow_bf = true, double cap2 = -1.0, bool in_loop = false);

// kernel launch, optionally with the programmatic-stream-serialization attribute (common.cuh: pdl_wait)
template <typename... KArgs, typename... Args>
inline void launch_kernel(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                          bool pdl, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  SICP_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...));
}
void set_state_transform(Ctx& c, const double x[6], const Rigid* T_or_null, bool reset_loop);
// k-NN (self included) + PCA of every query of one side; out[i] = (nx, ny, nz, planarity) float32.
// b == nullptr, the one-pair context: the fixed side (c.gfix, c.q_xyz, c.K -> c.q_nrm, the lists
// kept under option "keep_knn") or the movable side (c.gmov, c.mov_xyz, c.n_mov -> c.mov_nrm).
// b != nullptr, a batch: every pair's selected fixed points in its fixed grid (Batch::q_xyz ->
// Batch::q_nrm) or its movable points in its own movable grid (Batch::xyz -> Batch::mov_nrm).
// The movable side is chunked: as many queries per launch as option "normals_scratch_mb" holds at
// k x 4 bytes of neighbour positions each.
void normals_launch(Ctx& c, Batch* b, bool movable, int k);
// cos of the angle limit as sicp_set_mov_normals stores it (< 0: no angle test)
double mov_cos_max_of(double max_angle_rad);
void reject_solve_launch(Ctx& c, const sicp_run_params& p, int it, bool do_solve, bool arm_stop,
                         int rec_slot);
void compact_residuals_launch(Ctx& c);
void rs_fused_launch(Ctx& c, const sicp_run_params& p, int it, bool arm_stop, int rec_slot, bool want_sigma);
void final_residuals_launch(Ctx& c);
void transform_launch(Ctx& c, const Rigid& T, const double* in_dev, double* out_dev, long long n);
void gather_queries_launch(Ctx& c);

// batched launches
// with_list: pick from each pair's survivor list (Batch::ovl_list) instead of its whole cloud;
// fix_xyz: the fixed coordinates the descriptors' fix_off index (Batch::xyz or MapStore::xyz)
void batch_select_gather_launch(Ctx& c, Batch& b, const double* fix_xyz, bool with_list, int round_away);
void batch_match_launch(Ctx& c, Batch& b, bool warm);
// PointCloud.select_in_range of every fixed point of every pair under its pair's DevState
// transform: Ctx::compact.flag[flag_off + i] = (squared distance of fix_xyz[fix_off + i] to the
// nearest movable point < r2)
void batch_overlap_launch(Ctx& c, Batch& b, const double* fix_xyz, long long max_n_fix, double r2);
// Culled overlap filter of sicp_register_to_map: for every scan, the map points inside its
// MapCull box get the bounded search of batch_overlap_launch (same device code, same flag);
// survivors set bit i of the scan's row of MapStore::bits (cleared by the caller).
void map_overlap_launch(Ctx& c, Batch& b, MapStore& m, const MapCull* culls_dev, long long max_rows, double r2,
                        long long n_candidates_hint);
// sicp_overlap_graph's count (nn.cu: k_overlap_count), one launch for n_dirs <= 65535 directions:
// for each direction d, the records of dirs[d].a's grid inside its MapCull (at most max_rows rows)
// with idx % stride == 0 get the bounded search of batch_overlap_launch in dirs[d].b's grid under
// state[d] (same device code, same flag); the survivors are added to counts[dirs[d].slot] (zeroed
// by the caller).  n_candidates (records in the culls) picks the lanes per search.
void overlap_count_launch(Ctx& c, const GridView* views, const DevState* state, const OverlapDir* dirs, int n_dirs,
                          long long max_rows, long long stride, double r2, uint32_t* counts, long long n_candidates);
// popcounts of MapStore::bits words (n_words of them) -> popc, and the ordered compaction of the
// set bits into list (scan[w] = exclusive prefix sum of the popcounts): ascending map indices
void map_bits_popc_launch(Ctx& c, const uint32_t* bits, long long n_words, uint32_t* popc);
void map_bits_scatter_launch(Ctx& c, const uint32_t* bits, long long n_words, long long words_per_scan,
                             const uint32_t* scan, uint32_t* list);
// sicp_map_insert's occupancy test (nn.cu: k_map_insert_flags): for each of the n_fin points of
// fin_xyz (gridded in fresh), flag[fin_idx[f]] = 1 when no point of the map grid and no point of
// fresh with a smaller index has the same voxel key floor(p / voxel) (flag is zeroed by the caller)
void map_insert_flags_launch(Ctx& c, const GridView& map, const GridView& fresh, const double* fin_xyz,
                             const uint32_t* fin_idx, long long n_fin, double voxel, uint32_t* flag);
// sicp_map_thin's keep flags (nn.cu: k_map_thin_flags): keep[j] = 1 for each of the n map points
// xyz (gridded in map, in map order) when no map point j' < j has its voxel key floor(p / voxel),
// else 0
void map_thin_flags_launch(Ctx& c, const GridView& map, const double* xyz, long long n, double voxel, uint32_t* keep);
// sicp_map_carve's ray walk (nn.cu: k_map_carve): each finite point j of the n points xyz (cloud i
// from off[i], n_clouds + 1 offsets) is a ray from origins[3 i]; passes[idx] += 1 for every map
// record idx the ray passes (radius r, r2 = fl(r r), margin), at most once per ray.  passes is
// zeroed by the caller.
void map_carve_launch(Ctx& c, const GridView& map, const double* xyz, long long n, const uint32_t* off, int n_clouds,
                      const double* origins, double r, double r2, double margin, uint32_t* passes);
// sicp_map_distances' bounded nearest search (nn.cu: k_map_nearest), one lane group per point j of
// xyz (n points): the nearest map point (lowest index among ties) when its d2 < cap2 ->
// idx[j], d2[j], within[j] = 1; else idx -1, within 0 and d2 +inf (finite point) or NaN (a NaN or
// inf coordinate).
void map_nearest_launch(Ctx& c, const GridView& map, const double* xyz, long long n, double cap2, long long* idx,
                        double* d2, uint32_t* within);
// k-NN (self included) + PCA of n query points in the map grid (normals.cu: the estimate of
// sicp_estimate_normals, chunked by option "normals_scratch_mb"): out[i] = (nx, ny, nz,
// planarity) float32; pos is the caller's scratch, grown to one chunk.  Nothing of the one-pair
// context is written.
void map_normals_launch(Ctx& c, const GridView& map, const double* q_xyz, long long n, int k, float4* out,
                        DevBuf<uint32_t>& pos);
void batch_rs_launch(Ctx& c, Batch& b, const sicp_run_params& p, int it, bool want_sigma);
void batch_finish_launch(Ctx& c, Batch& b, int max_iterations);
// sicp_get_batch_outputs, for the n_ids pairs ids (device) of the last batched run: the movable
// clouds moved by DevState::T into out + 3 off[j], and the final residuals in kept order into
// out + off[j] (off device)
void batch_transform_launch(Ctx& c, Batch& b, const int* ids, int n_ids, const long long* off, long long max_n_mov,
                            double* out);
void batch_residuals_launch(Ctx& c, Batch& b, const int* ids, int n_ids, const long long* off, double* out);

int bin_cap_for(long long K);

// helpers in capi.cu
// device ordinal of device (or managed) memory, -1 for host memory
int device_of_ptr(const void* p);
// bytes between any two of host, device and other-device memory, on the context's stream
void copy_any(Ctx& c, void* dst, const void* src, size_t bytes);
// queries per launch of a chunked k-NN + PCA: c.normals_scratch_mb MiB of k record positions each
inline long long normals_chunk_queries(const Ctx& c, int k) {
  return std::max<long long>(1024, ((long long)c.normals_scratch_mb << 20) / (4ll * k));
}
void check_mov_neighbors(const Ctx& c, const sicp_register_params& rp);
// a whole cloud host -> device on the context's stream (pageable sources through upload.cuh's
// staging threads), stream-ordered when it returns
void upload_to_device(Ctx& c, void* dst, const void* src, size_t bytes);

struct StageTimer {
  Ctx& c;
  double* slot;
  StageTimer(Ctx& c_, double* s) : c(c_), slot(s) { cudaEventRecord(c.ev0, c.stream); }
  void stop() {
    cudaEventRecord(c.ev1, c.stream);
    cudaEventSynchronize(c.ev1);
    float ms = 0;
    cudaEventElapsedTime(&ms, c.ev0, c.ev1);
    *slot = ms;
  }
};

}  // namespace sicp

struct sicp_ctx {
  sicp::Ctx c;
  int it_counter = 0;
};

// Body of every entry point that takes a context: API_BEGIN(ctx) binds `c` to it and makes its
// device current, API_END turns what the body throws into the return code, the context's and the
// thread's message, and cancels pending staged uploads.
#define API_BEGIN(ctxptr)                                    \
  if (!(ctxptr)) {                                           \
    sicp::set_thread_error("sicp_ctx is NULL");              \
    return SICP_ERR_BAD_ARG;                                 \
  }                                                          \
  sicp::Ctx& c = (ctxptr)->c;                                \
  try {                                                      \
    SICP_CUDA(cudaSetDevice(c.device));

#define API_END                                              \
  }                                                          \
  catch (const sicp::Error& e) {                             \
    c.up.cancel();                                           \
    c.err = e.msg;                                           \
    sicp::set_thread_error(e.msg);                           \
    if (e.code == SICP_ERR_CUDA) cudaGetLastError();         \
    return e.code;                                           \
  }                                                          \
  catch (const std::exception& e) {                          \
    c.up.cancel();                                           \
    c.err = e.what();                                        \
    sicp::set_thread_error(c.err);                           \
    return SICP_ERR_CUDA;                                    \
  }                                                          \
  return SICP_OK;
