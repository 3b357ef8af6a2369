// batch.cu — sicp_register_batch: SimpleICP.run (python/simpleicp/simpleicp.py:75-324) for many
// independent pairs with ONE set of launches per stage and per iteration (BASELINE.json
// configs[4]: 512 pairs of 100 000 points, 64 per GPU; SURVEY.md section 8e).
//
// A registration of a 100 000-point pair with 1000 correspondences is far too small to fill an
// H100: one match launch has 16 000 threads, one reject/solve launch one block, and the host
// drives ~30 launches per iteration-loop through a Python thread.  Here every kernel carries a
// pair dimension instead:
//   upload        every cloud once into one store (register_pairs): the clouds fixed in some pair
//                 on the context's stream (upload_to_device), the movable-only ones on the copy
//                 stream, where they cross PCIe while the fixed-side work runs
//   grids         segmented counting sort over all clouds of a side (grid.cu: grid_build)
//   overlap       (max_overlap_distance only) bounded search of every fixed point under its pair's
//                 prior, one scan + ordered scatter into per-pair survivor lists, one read-back
//                 per batch; this needs the movable grids, so the fixed-side work below follows it
//   select+gather rint(linspace) picks and their coordinates, all pairs in one launch
//   normals       k-NN + PCA, blockIdx.y = pair
//   mov normals   (mov_neighbors only) k-NN + PCA of every movable point in its pair's movable
//                 grid, in chunks of queries; the match folds them into an effective planarity
//   loop          per iteration ONE match launch over (pair, query) and ONE reject/solve launch
//                 with a block per pair (the barrier-free kernel with G = 1: predictor histogram
//                 select, or the in-block radix select when there is no usable prediction), every
//                 pair with its own device-resident state and stop flag
//   finish        exact residual statistics + result record per pair, one small download
// No host work per pair except the two copies.
//
// sicp_register_to_map runs the same stages (run_pairs) for scans against a map held on the
// context (sicp_set_map, MapStore): the fixed side is the map's grid, and the overlap filter only
// searches the map points inside each scan's box mapped by its prior (map_cull_box, map_filter).
//
// sicp_register_pairs runs them for pairs drawn from one set of clouds: each cloud is uploaded,
// gridded and (as a movable cloud) given its normals once, whatever number of pairs uses it
// (register_pairs).  sicp_register_batch is register_pairs over its 2 n_pairs clouds.
//
// sicp_get_batch_outputs returns what any of these calls left on the device and did not download:
// transformed clouds, residual vectors, the per-iteration log and the applied transforms.
#include <algorithm>
#include <cstddef>
#include <cmath>
#include <cstring>
#include <tuple>
#include <unordered_map>
#include <utility>
#include <vector>

#include "ctx.cuh"
#include "joint_plan.h"

namespace sicp {

struct JointRun;

namespace {

__global__ void k_gather_flags(const DevState* __restrict__ st, int n, int* __restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  flags[2 * i + 0] = st[i].stop;
  flags[2 * i + 1] = st[i].iterations_done;
}

// sicp_map_insert, one thread per point j of the concatenated clouds (cloud i owns [off[i],
// off[i + 1])): the point moved by its cloud's transform when there are transforms (T != NULL;
// rigid_apply as k_transform, in place, scalar accesses since clouds start at any point offset),
// and fin[j] = all three coordinates finite.
__global__ void __launch_bounds__(256)
    k_insert_stage(double* __restrict__ xyz, long long n, const uint32_t* __restrict__ off, int n_clouds,
                   const Rigid* __restrict__ T, uint32_t* __restrict__ fin) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= n) return;
  double x = xyz[3 * j + 0], y = xyz[3 * j + 1], z = xyz[3 * j + 2];
  if (T) {
    int lo = 0, hi = n_clouds;  // off[lo] <= j < off[hi]: the last cloud starting at or before j
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (off[mid] <= (unsigned long long)j) lo = mid;
      else hi = mid;
    }
    double ox, oy, oz;
    rigid_apply(T[lo], x, y, z, ox, oy, oz);
    xyz[3 * j + 0] = x = ox;
    xyz[3 * j + 1] = y = oy;
    xyz[3 * j + 2] = z = oz;
  }
  fin[j] = (isfinite(x) && isfinite(y) && isfinite(z)) ? 1u : 0u;
}

// sicp_map_crop, one thread per map point j: keep[j] = 1 iff d2 < r2 for at least one of the n_c
// centres cen, where d2 = (dx dx + dy dy) + dz dz with d = p - c and every operation rounded on
// its own (no fused multiply-add), else 0.  The block reads the centres through shared memory,
// kCropChunk at a time, and stops at the first chunk boundary where all its points are kept.
constexpr int kCropChunk = 256;
__global__ void __launch_bounds__(256)
    k_map_crop_flags(const double* __restrict__ xyz, long long n, const double* __restrict__ cen, int n_c, double r2,
                     uint32_t* __restrict__ keep) {
  __shared__ double s[3 * kCropChunk];
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  double x = 0.0, y = 0.0, z = 0.0;
  if (j < n) {
    x = xyz[3 * j + 0];
    y = xyz[3 * j + 1];
    z = xyz[3 * j + 2];
  }
  bool hit = false;
  for (int c0 = 0; c0 < n_c; c0 += kCropChunk) {
    // block-uniform: every thread has finished reading the previous chunk
    if (__syncthreads_and(hit || j >= n)) break;
    const int m = min(kCropChunk, n_c - c0);
    for (int i = threadIdx.x; i < 3 * m; i += blockDim.x) s[i] = cen[3 * (long long)c0 + i];
    __syncthreads();
    if (hit || j >= n) continue;
    for (int i = 0; i < m; ++i) {
      const double dx = __dsub_rn(x, s[3 * i + 0]), dy = __dsub_rn(y, s[3 * i + 1]), dz = __dsub_rn(z, s[3 * i + 2]);
      if (__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)) < r2) {
        hit = true;
        break;
      }
    }
  }
  if (j < n) keep[j] = hit ? 1u : 0u;
}

// sicp_map_carve's keep flags: keep[j] = passes[j] < min_passes
__global__ void __launch_bounds__(256)
    k_carve_keep(const uint32_t* __restrict__ passes, long long n, uint32_t min_passes, uint32_t* __restrict__ keep) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j < n) keep[j] = passes[j] < min_passes ? 1u : 0u;
}

// the signed distance of point j along its matched map point's normal, plane_distance's expression
// (nn.cu): ((px - mx) nx + (py - my) ny) + (pz - mz) nz in double, the float32 normal promoted, no
// fused multiply-add; and that normal's planarity.  NaN for a point without a match.
__global__ void __launch_bounds__(256)
    k_dist_plane(const double* __restrict__ xyz, long long n, const uint32_t* __restrict__ within,
                 const uint32_t* __restrict__ scan, const double* __restrict__ m_xyz, const float4* __restrict__ nrm,
                 double* __restrict__ plane, float* __restrict__ planarity) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= n) return;
  if (!within[j]) {
    plane[j] = __longlong_as_double(0x7ff8000000000000ll);
    planarity[j] = __int_as_float(0x7fc00000);
    return;
  }
  const long long f = scan[j];
  const float4 nr = nrm[f];
  const double dx = xyz[3 * j + 0] - m_xyz[3 * f + 0], dy = xyz[3 * j + 1] - m_xyz[3 * f + 1],
               dz = xyz[3 * j + 2] - m_xyz[3 * f + 2];
  plane[j] = __dadd_rn(__dadd_rn(__dmul_rn(dx, (double)nr.x), __dmul_rn(dy, (double)nr.y)), __dmul_rn(dz, (double)nr.z));
  planarity[j] = nr.w;
}

// the cell policy of every grid of this file: both sides of a batch, the map and its inserts
CellPolicy batch_policy(const Ctx& c) { return CellPolicy{CellPolicy::kBatch, c.grid_target_occ}; }

// What the stages shared by sicp_register_pairs (and through it sicp_register_batch) and
// sicp_register_to_map know about one call.
struct PairsRun {
  int n_pairs = 0;
  const sicp_register_params* rp = nullptr;
  const double* observed = nullptr;
  bool overlap = false;
  long long Kmax = 0, max_n_mov = 0;
  std::vector<long long> mo;    // prefix sums of the pairs' movable point counts, n_pairs + 1
  std::vector<DevState> hs;     // per-pair start state (the prior)
  // descriptors; the caller fills gfix, n_fix, fix_off, flag_off and mov_off, and gmov and cm of
  // the pairs whose movable grid it built (mov_slot[i] < 0)
  std::vector<PairDev> pd;
  // the movable-only clouds (upload_movable), which run_pairs grids into Batch::gmov once they have
  // arrived, and each pair's slot in that list (-1: its movable grid is in Batch::gfix)
  std::vector<HostCloud> mov_clouds;
  std::vector<int> mov_slot;
  // pairs whose descriptors the movable-normals estimate runs over, one per distinct movable cloud;
  // empty or all pairs: every pair's (each has its own movable cloud)
  std::vector<int> mov_first;
  std::vector<char> no_overlap;
  // sicp_register_joint: each pair's start transform (instead of rigid_from_x of its x0), and the
  // joint problem whose loop replaces the per-pair one
  const Rigid* prior = nullptr;
  JointRun* joint = nullptr;
};

// Argument checks of both entry points that need no cloud (the clouds are checked per pair by
// the callers, before any device work).
void check_pairs_params(const Ctx& c, int n_pairs, bool pointers_given, const sicp_register_params* rp) {
  SICP_REQUIRE(n_pairs >= 1 && n_pairs <= 65535, SICP_ERR_BAD_ARG, "n_pairs must be in [1, 65535]");
  SICP_REQUIRE(pointers_given && rp, SICP_ERR_BAD_ARG, "NULL argument");
  SICP_REQUIRE(rp->correspondences >= 1 && rp->correspondences <= 4096, SICP_ERR_BAD_ARG,
               "the batched engine runs one block per pair: correspondences must be in [1, 4096]");
  const sicp_run_params& p = rp->run;
  SICP_REQUIRE(p.max_iterations >= 1 && p.max_iterations <= 4096, SICP_ERR_BAD_ARG,
               "max_iterations must be in [1, 4096]");
  bool any_finite = false;
  for (int j = 0; j < 6; ++j) {
    SICP_REQUIRE(p.lsq.obs_weight[j] >= 0, SICP_ERR_BAD_ARG,
                 "All elements of rbp_observation_weights must be >= 0.");
    any_finite = any_finite || std::isfinite(p.lsq.obs_weight[j]);
    SICP_REQUIRE(c.variant == SICP_VARIANT_PYTHON || p.lsq.obs_weight[j] == 0.0, SICP_ERR_BAD_ARG,
                 "the linearised variants have no observed or fixed parameters");
  }
  SICP_REQUIRE(any_finite, SICP_ERR_BAD_ARG, "At least one element in rbp_observation_weights must be finite.");
  check_mov_neighbors(c, *rp);
}

void begin_pairs(PairsRun& r, int n_pairs, const sicp_register_params* rp, const double* observed) {
  r.n_pairs = n_pairs;
  r.rp = rp;
  r.observed = observed;
  r.overlap = rp->max_overlap_distance > 0 && std::isfinite(rp->max_overlap_distance);
  r.mo.assign((size_t)n_pairs + 1, 0);
  r.mov_slot.assign((size_t)n_pairs, -1);
}

void check_movable(const sicp_register_params& rp, int i, int64_t n_mov) {
  SICP_REQUIRE(n_mov >= rp.mov_neighbors, SICP_ERR_BAD_ARG,
               "mov_neighbors exceeds the number of points in the movable cloud of pair " + std::to_string(i));
}

// pair i's movable cloud (checked and counted) and its share of the per-query arrays
void add_movable(PairsRun& r, int i, int64_t n_mov) {
  check_movable(*r.rp, i, n_mov);
  r.max_n_mov = std::max<long long>(r.max_n_mov, n_mov);
  r.mo[(size_t)i + 1] = r.mo[(size_t)i] + n_mov;
}

// The movable-only clouds xyz[j], j in ids, cross PCIe into the store Batch::xyz at off[j] on the
// copy stream (behind the event the caller recorded on the context's stream after the last use of
// the buffers) and join PairsRun::mov_clouds; ev_copy marks their arrival.
void upload_movable(Ctx& c, Batch& b, PairsRun& r, const std::vector<int>& ids, const double* const* xyz,
                    const int64_t* n, const std::vector<long long>& off) {
  for (int j : ids) {
    double* dst = b.xyz.p + 3 * off[(size_t)j];
    SICP_CUDA(cudaMemcpyAsync(dst, xyz[j], sizeof(double) * 3 * (size_t)n[j], cudaMemcpyDefault, c.copy_stream));
    r.mov_clouds.push_back(HostCloud{dst, n[j], off[(size_t)j]});
  }
  SICP_CUDA(cudaEventRecord(c.ev_copy, c.copy_stream));
}

// Per-pair buffers and start states: every pair starts from its prior, observed row i (x0 =
// observed, as SimpleICP.run does) or the common x0; the overlap filter runs under that transform
// (H0, simpleicp.py:158-170).
void alloc_pair_buffers(Ctx& c, Batch& b, PairsRun& r) {
  cudaStream_t st = c.stream;
  const int n_pairs = r.n_pairs;
  const sicp_run_params& p = r.rp->run;
  const long long Kmax = r.Kmax;
  const size_t nq = (size_t)n_pairs * (size_t)Kmax;
  b.n_pairs = n_pairs;
  b.Kmax = Kmax;
  b.pairs.reserve(n_pairs);
  b.sel_idx.reserve(nq);
  b.nn_idx.reserve(nq);
  b.q_xyz.reserve(3 * nq);
  b.dist.reserve(nq);
  b.m_xyz.reserve(3 * nq);
  b.q_nrm.reserve(nq);
  b.bin_cap = bin_cap_for(Kmax);
  b.binstore.reserve((size_t)n_pairs * LH_BINS * (size_t)b.bin_cap);
  b.nn_pos.reserve(nq);
  b.keep.reserve(nq);
  b.state.reserve(n_pairs);
  b.lin_hist.reserve((size_t)n_pairs * (LH_BINS + 2));
  b.rec.reserve((size_t)n_pairs * (size_t)p.max_iterations);
  b.partials.reserve((size_t)n_pairs * 96 + 16);
  b.phase_t.reserve((size_t)n_pairs * 32);
  b.flags.reserve(2 * (size_t)n_pairs);
  b.results.reserve(n_pairs);
  pinned_reserve(b.flags_host, b.flags_cap, 2 * (size_t)n_pairs);
  pinned_reserve(b.results_host, b.results_cap, (size_t)n_pairs);
  SICP_CUDA(cudaMemsetAsync(b.lin_hist.p, 0, sizeof(unsigned int) * (size_t)n_pairs * (LH_BINS + 2), st));
  SICP_CUDA(cudaMemsetAsync(b.rec.p, 0, sizeof(sicp_iter_record) * (size_t)n_pairs * (size_t)p.max_iterations, st));
  SICP_CUDA(cudaMemsetAsync(b.nn_pos.p, 0xff, sizeof(uint32_t) * nq, st));
  SICP_CUDA(cudaMemsetAsync(b.keep.p, 0, nq, st));
  r.hs.assign((size_t)n_pairs, DevState{});
  for (int i = 0; i < n_pairs; ++i) {
    DevState& h = r.hs[(size_t)i];
    std::memset(&h, 0, sizeof(h));
    for (int j = 0; j < 6; ++j) h.x[j] = r.observed ? r.observed[6 * i + j] : p.lsq.x0[j];
    h.T = r.prior ? r.prior[i] : rigid_from_x(h.x);
    h.Tinv = rigid_inverse(h.T);
    h.T_res = h.T;
    h.H_rep = h.T;
  }
  SICP_CUDA(cudaMemcpyAsync(b.state.p, r.hs.data(), sizeof(DevState) * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
  r.pd.assign((size_t)n_pairs, PairDev{});
  for (auto& d : r.pd) std::memset(&d, 0, sizeof(d));
}

// Survivor lists of the overlap filter: bounds[i] .. bounds[i + 1] is pair i's slice.  A pair
// without a survivor is parked like a pair without enough correspondences (every later kernel
// returns at once) and reported as SICP_ERR_NO_OVERLAP.
void take_survivors(Ctx& c, Batch& b, PairsRun& r, const uint32_t* bounds) {
  bool parked = false;
  for (int i = 0; i < r.n_pairs; ++i) {
    PairDev& d = r.pd[(size_t)i];
    d.list_off = bounds[i];
    d.list_len = (long long)bounds[i + 1] - (long long)bounds[i];
    d.K = std::min<long long>(r.rp->correspondences, d.list_len);
    if (d.list_len == 0) {
      r.no_overlap[(size_t)i] = 1;
      r.hs[(size_t)i].stop = 2;
      parked = true;
    }
  }
  if (parked)
    SICP_CUDA(cudaMemcpyAsync(b.state.p, r.hs.data(), sizeof(DevState) * (size_t)r.n_pairs, cudaMemcpyHostToDevice,
                              c.stream));
}

// Overlap filter of sicp_register_batch and sicp_register_pairs: bounded search of every fixed
// point of every pair (coordinates in fix_xyz), one exclusive scan over the keep flags of the whole
// batch, ordered scatter of the flag positions, and ONE read-back of the pair boundaries.
void batch_filter(Ctx& c, Batch& b, PairsRun& r, const double* fix_xyz, long long max_n_fix) {
  CompactScratch& s = c.compact;
  const long long nf = b.total_fix;
  s.flag.reserve(nf);
  s.scan.reserve(nf + 1);
  b.ovl_list.reserve(std::max<long long>(nf, 1));
  // r2 as sicp_register computes it
  batch_overlap_launch(c, b, fix_xyz, max_n_fix, r.rp->max_overlap_distance * r.rp->max_overlap_distance);
  scan_u32(c, s.flag.p, nf, s.scan.p, s.sums);
  compact_scatter(c, s.flag.p, nf, s.scan.p, b.ovl_list.p, nullptr, nullptr, nullptr);
  std::vector<long long> fo((size_t)r.n_pairs + 1, nf);
  for (int i = 0; i < r.n_pairs; ++i) fo[(size_t)i] = r.pd[(size_t)i].flag_off;
  take_survivors(c, b, r, compact_bounds(c, s.scan.p, fo));
}

}  // namespace

// The box that holds every map point able to pass scan i's overlap filter.  A map point p passes
// when the squared distance from q = Tinv p (rounded) to some movable point m of the scan, rounded,
// is below r2 = r * r (rounded).  Every movable point lies in the box B of the scan's movable grid,
// [o, o + dims h].  In exact arithmetic, |T^-1 p - m| < r gives |p - T m| < r, and T m lies in the
// convex hull of the eight mapped corners of B, hence in their axis-aligned box grown by r.  What
// rounding adds is bounded by a few ulps of the largest magnitude M involved (map and scan
// coordinates, the translation): q and the mapped corners each carry a few ulps of M, Tinv is the
// inverse of T up to a few ulps (R^T is exact, R is orthogonal to ~1e-15), and the rounded d^2 and
// r2 move the radius by a few relative ulps.  Together that is below 1e-13 (M + r); the box is
// grown by r + 1e-12 (M + r), ten times more (5e-6 m at UTM coordinates).  The cells are the map
// grid's own cell_coord of the box faces: floor((v - o) / h) is monotone in v, so every point in the
// box lies in a cell between those of its faces, and the kernel tests each candidate against the
// box itself.  The proof covers two callers: sicp_register_to_map (map grid, scan i's movable grid,
// its prior) and sicp_overlap_graph's direction cull (a's grid as the map, b's grid as the scan,
// T_ab), whose count runs the same search under the same bound.
static MapCull map_cull_box(const GridView& map, const GridView& g, const Rigid& T, double r) {
  MapCull cu;
  std::memset(&cu, 0, sizeof(cu));
  const double lo_s[3] = {g.ox, g.oy, g.oz}, hi_s[3] = {g.ox + g.nx * g.h, g.oy + g.ny * g.h, g.oz + g.nz * g.h};
  const double o[3] = {map.ox, map.oy, map.oz};
  const int dims[3] = {map.nx, map.ny, map.nz};
  double mag = std::max(std::fabs(T.t[0]), std::max(std::fabs(T.t[1]), std::fabs(T.t[2])));
  for (int a = 0; a < 3; ++a) {
    cu.lo[a] = kInf;
    cu.hi[a] = -kInf;
    mag = std::max(mag, std::max(std::fabs(o[a]), std::fabs(o[a] + dims[a] * map.h)));
    mag = std::max(mag, std::max(std::fabs(lo_s[a]), std::fabs(hi_s[a])));
  }
  for (int k = 0; k < 8; ++k) {
    double v[3];
    rigid_apply(T, (k & 1) ? hi_s[0] : lo_s[0], (k & 2) ? hi_s[1] : lo_s[1], (k & 4) ? hi_s[2] : lo_s[2], v[0], v[1], v[2]);
    for (int a = 0; a < 3; ++a) {
      cu.lo[a] = std::min(cu.lo[a], v[a]);
      cu.hi[a] = std::max(cu.hi[a], v[a]);
      mag = std::max(mag, std::fabs(v[a]));
    }
  }
  const double grow = r + 1e-12 * (mag + r);
  for (int a = 0; a < 3; ++a) {
    cu.lo[a] -= grow;
    cu.hi[a] += grow;
    // no map point lies below the map's box minimum o or beyond o + dims h
    if (!(cu.hi[a] >= o[a]) || !(cu.lo[a] <= o[a] + (dims[a] + 1) * map.h)) return cu;  // rows = 0
    auto cell = [&](double v) {
      const double f = std::floor((v - o[a]) * map.inv_h);  // cell_coord's arithmetic, then its clamp
      return f < 0.0 ? 0 : (f > dims[a] - 1 ? dims[a] - 1 : (int)f);
    };
    cu.c0[a] = cell(cu.lo[a]);
    cu.c1[a] = cell(cu.hi[a]);
  }
  cu.rows = (long long)(cu.c1[1] - cu.c0[1] + 1) * (cu.c1[2] - cu.c0[2] + 1);
  return cu;
}

// Culled overlap filter of sicp_register_to_map: a bit per (scan, map point) set by the searches
// of the candidates in each scan's box, popcounts of the mask words, one exclusive scan over them,
// ONE read-back of the scans' boundaries (and the search count), then the ordered compaction into
// the survivor lists: ascending map indices per scan, as select_n_points needs them.
static void map_filter(Ctx& c, Batch& b, MapStore& m, PairsRun& r) {
  cudaStream_t st = c.stream;
  const int n = r.n_pairs;
  const double rr = r.rp->max_overlap_distance;
  std::vector<MapCull> cu((size_t)n);
  long long max_rows = 0, hint = 0;
  for (int i = 0; i < n; ++i) {
    cu[(size_t)i] = map_cull_box(m.view, r.pd[(size_t)i].gmov, r.hs[(size_t)i].T, rr);
    max_rows = std::max(max_rows, cu[(size_t)i].rows);
    hint += (long long)(cu[(size_t)i].rows * (cu[(size_t)i].c1[0] - cu[(size_t)i].c0[0] + 1) * c.grid_target_occ);
  }
  const long long words = (m.n + 31) / 32, nw = words * n;
  CompactScratch& s = c.compact;
  m.culls.reserve(n);
  m.bits.reserve(nw);
  s.flag.reserve(nw);
  s.scan.reserve(nw + 1);
  m.n_searched.reserve(1);
  SICP_CUDA(cudaMemcpyAsync(m.culls.p, cu.data(), sizeof(MapCull) * (size_t)n, cudaMemcpyHostToDevice, st));
  SICP_CUDA(cudaMemsetAsync(m.bits.p, 0, sizeof(uint32_t) * (size_t)nw, st));
  SICP_CUDA(cudaMemsetAsync(m.n_searched.p, 0, sizeof(unsigned long long), st));
  if (max_rows > 0) map_overlap_launch(c, b, m, m.culls.p, max_rows, rr * rr, hint);  // r2 as sicp_register computes it
  map_bits_popc_launch(c, m.bits.p, nw, s.flag.p);
  scan_u32(c, s.flag.p, nw, s.scan.p, s.sums);
  // n + 1 boundaries, then the count
  pinned_reserve(s.host, s.host_cap, (size_t)n + 1);
  uint32_t* bounds = s.host;
  unsigned long long* searched = reinterpret_cast<unsigned long long*>(c.scal_host);
  SICP_CUDA(cudaMemcpy2DAsync(bounds, sizeof(uint32_t), s.scan.p, sizeof(uint32_t) * (size_t)words,
                              sizeof(uint32_t), (size_t)n + 1, cudaMemcpyDeviceToHost, st));
  SICP_CUDA(cudaMemcpyAsync(searched, m.n_searched.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  SICP_CUDA(cudaStreamSynchronize(st));
  c.tm.overlap_candidates = (int64_t)*searched;
  b.ovl_list.reserve(std::max<long long>(bounds[n], 1));
  map_bits_scatter_launch(c, m.bits.p, nw, words, s.scan.p, b.ovl_list.p);
  take_survivors(c, b, r, bounds);
}

// What sicp_register_joint knows of its problem on the host: the edges, every cloud's pose and
// role, and (after the loop) the final poses.
struct JointRun {
  int n_clouds = 0, n_edges = 0, F = 0;
  const int32_t* fix_id = nullptr;
  const int32_t* mov_id = nullptr;
  std::vector<char> fixed;      // per cloud: pose held
  std::vector<Rigid> pose;      // per cloud, world <- cloud
  std::vector<Rigid> prior;     // per edge: T_a^-1 T_b
  std::vector<int> free_of, free_ids;
  // the pose priors the call reads (DESIGN.md §6.12): per cloud, a prior with six non-zero weights
  // (an anchor like a fixed cloud); the priors in free-cloud order, and per free cloud its prior or -1
  std::vector<char> full_prior;
  std::vector<JointPrior> poses;
  std::vector<int> prior_of;
  // the relative observations the call reads (DESIGN.md §6.13), in call order
  std::vector<JointRel> rels;
};

// Every read relative observation k, ascending, in the list of each block of the joint matrix it
// touches: the diagonal blocks of its free ends and, with both ends free, their lower off-diagonal
// block; block(p, q), p >= q, gives (and creates, as an empty edge list) the block's index.
template <class Block>
static std::vector<std::vector<int>> joint_rel_lists(const JointRun& j, Block block) {
  std::vector<std::vector<int>> rl;
  auto add = [&](int bi, int k) {
    if (bi >= (int)rl.size()) rl.resize((size_t)bi + 1);
    rl[(size_t)bi].push_back(k);
  };
  for (int k = 0; k < (int)j.rels.size(); ++k) {
    const int fa = j.rels[(size_t)k].fa, fb = j.rels[(size_t)k].fb;
    if (fa >= 0) add(block(fa, fa), k);
    if (fb >= 0) add(block(fb, fb), k);
    if (fa >= 0 && fb >= 0) add(block(std::max(fa, fb), std::min(fa, fb)), k);
  }
  return rl;
}

// lists appended to ids as offsets (lists.size() + 1), then entries; returns where each starts
static std::pair<size_t, size_t> append_lists(std::vector<int>& ids, const std::vector<std::vector<int>>& lists) {
  const size_t o = ids.size();
  int at = 0;
  for (const auto& l : lists) {
    ids.push_back(at);
    at += (int)l.size();
  }
  ids.push_back(at);
  const size_t k = ids.size();
  for (const auto& l : lists) ids.insert(ids.end(), l.begin(), l.end());
  return {o, k};
}

// Union-find of the clouds over the edges with use[e] != 0; SICP_REQUIRE fails with `code` when a
// cloud some edge references shares its component with no fixed cloud and no free cloud whose pose
// prior has six non-zero weights.
static void check_anchored(const JointRun& j, const std::vector<char>& use, int code, const char* msg) {
  std::vector<int> up((size_t)j.n_clouds);
  for (int i = 0; i < j.n_clouds; ++i) up[(size_t)i] = i;
  auto root = [&](int i) {
    while (up[(size_t)i] != i) i = up[(size_t)i] = up[(size_t)up[(size_t)i]];
    return i;
  };
  for (int e = 0; e < j.n_edges; ++e)
    if (use[(size_t)e]) up[(size_t)root(j.fix_id[e])] = root(j.mov_id[e]);
  std::vector<char> anchored((size_t)j.n_clouds, 0);
  for (const JointRel& o : j.rels)  // an observation with six non-zero weights joins its clouds
    if (o.w[0] > 0.0 && o.w[1] > 0.0 && o.w[2] > 0.0 && o.w[3] > 0.0 && o.w[4] > 0.0 && o.w[5] > 0.0)
      up[(size_t)root(o.ca)] = root(o.cb);
  for (int i = 0; i < j.n_clouds; ++i)
    if (j.fixed[(size_t)i] || j.full_prior[(size_t)i]) anchored[(size_t)root(i)] = 1;
  for (int e = 0; e < j.n_edges; ++e)
    for (int k = 0; k < 2; ++k) {
      const int cl = k ? j.mov_id[e] : j.fix_id[e];
      SICP_REQUIRE(anchored[(size_t)root(cl)], code, std::string(msg) + " (cloud " + std::to_string(cl) + ")");
    }
}

// The sparse solve's plan (joint_plan.h) over the free-free pairs of the edges with use[e] != 0 and
// of the relative observations; SICP_ERR_BAD_ARG when its panels would exceed JOINT_SPARSE_MAX_BYTES.
static JointPlan joint_sparse_plan(const JointRun& j, const std::vector<char>& use) {
  std::vector<std::pair<int, int>> pairs;
  for (int e = 0; e < j.n_edges; ++e) {
    const int fa = j.free_of[(size_t)j.fix_id[e]], fb = j.free_of[(size_t)j.mov_id[e]];
    if (use[(size_t)e] && fa >= 0 && fb >= 0) pairs.emplace_back(fa, fb);
  }
  for (const JointRel& o : j.rels)
    if (o.fa >= 0 && o.fb >= 0) pairs.emplace_back(o.fa, o.fb);
  JointPlan pl = make_joint_plan(j.F, pairs);
  SICP_REQUIRE(pl.factor_bytes() <= JOINT_SPARSE_MAX_BYTES, SICP_ERR_BAD_ARG,
               "joint_solver 1: the factor of this edge graph needs " + std::to_string(pl.factor_bytes()) +
                   " bytes, more than the limit of " + std::to_string(JOINT_SPARSE_MAX_BYTES));
  return pl;
}

// What k_joint_sparse_solve reads of the plan, appended to ids (offsets into it in o): the
// supernodes, structs, updates, maps, levels, the order, and every panel block's list of live edges
// in ascending order (2 e + (1: the block's cloud is the edge's a) on a diagonal block); with
// relative observations also each list's observations (rel: offsets, then entries).
struct SparseIds {
  size_t sn, st, up, map, lv_off, lv, perm, blk, lst_off, lst_edge;
  std::pair<size_t, size_t> rel;
};
static SparseIds joint_sparse_ids(const JointRun& j, const std::vector<char>& live, const JointPlan& pl,
                                  std::vector<int>& ids) {
  // the lists of the blocks the live edges touch, keyed by (free cloud, free cloud), smaller first
  std::unordered_map<long long, int> key_of;
  std::vector<std::vector<int>> lists;
  auto add = [&](int p, int q, int v) {
    const long long key = (long long)std::min(p, q) * j.F + std::max(p, q);
    auto it = key_of.emplace(key, (int)lists.size()).first;
    if (it->second == (int)lists.size()) lists.emplace_back();
    lists[(size_t)it->second].push_back(v);
  };
  for (int e = 0; e < j.n_edges; ++e) {
    if (!live[(size_t)e]) continue;
    const int fa = j.free_of[(size_t)j.fix_id[e]], fb = j.free_of[(size_t)j.mov_id[e]];
    if (fa >= 0) add(fa, fa, 2 * e + 1);
    if (fb >= 0) add(fb, fb, 2 * e);
    if (fa >= 0 && fb >= 0) add(fa, fb, 2 * e);
  }
  std::vector<std::vector<int>> rel = joint_rel_lists(j, [&](int p, int q) {
    auto it = key_of.emplace((long long)std::min(p, q) * j.F + std::max(p, q), (int)lists.size()).first;
    if (it->second == (int)lists.size()) lists.emplace_back();
    return it->second;
  });
  rel.resize(lists.size());
  static_assert(sizeof(JointSuper) == 8 * sizeof(int), "JointSuper travels as 8 ints");
  SparseIds o{};
  o.sn = ids.size();
  int table = 0;
  for (int s = 0; s < pl.n_super; ++s) {
    const int v[8] = {pl.first[(size_t)s], pl.ns(s), pl.nt(s), pl.st_off[(size_t)s], pl.up_off[(size_t)s],
                      pl.up_off[(size_t)s + 1], table, 0};  // JointSuper
    ids.insert(ids.end(), v, v + 8);
    table += (pl.ns(s) + pl.nt(s)) * pl.ns(s);
  }
  o.st = ids.size();
  ids.insert(ids.end(), pl.st.begin(), pl.st.end());
  o.up = ids.size();
  for (size_t u = 0; u < pl.up.size(); ++u) {
    const int v[4] = {pl.up[u], pl.up_i0[u], pl.up_nj[u], pl.up_map[u]};
    ids.insert(ids.end(), v, v + 4);
  }
  o.map = ids.size();
  ids.insert(ids.end(), pl.map.begin(), pl.map.end());
  o.lv_off = ids.size();
  ids.insert(ids.end(), pl.lv_off.begin(), pl.lv_off.end());
  o.lv = ids.size();
  ids.insert(ids.end(), pl.lv.begin(), pl.lv.end());
  o.perm = ids.size();
  ids.insert(ids.end(), pl.perm.begin(), pl.perm.end());
  o.blk = ids.size();
  for (int s = 0; s < pl.n_super; ++s) {
    const int ns = pl.ns(s), f0 = pl.first[(size_t)s];
    for (int ri = 0; ri < ns + pl.nt(s); ++ri) {
      const int pr = ri < ns ? f0 + ri : pl.st[(size_t)(pl.st_off[(size_t)s] + ri - ns)];
      for (int cj = 0; cj < ns; ++cj) {
        const int pc = f0 + cj;
        int l = -1;
        if (pr >= pc) {
          const int a = pl.perm[(size_t)pr], b = pl.perm[(size_t)pc];
          auto it = key_of.find((long long)std::min(a, b) * j.F + std::max(a, b));
          if (it != key_of.end()) l = it->second;
        }
        ids.push_back(l);
      }
    }
  }
  std::tie(o.lst_off, o.lst_edge) = append_lists(ids, lists);
  if (!j.rels.empty()) o.rel = append_lists(ids, rel);
  return o;
}

// The loop of sicp_register_joint, in place of run_pairs' per-pair loop: per iteration the match of
// every edge, k_joint_reject and k_joint_solve or, under option "joint_solver" 1,
// k_joint_sparse_solve (joint.cu), and the read of the stop flag every
// host_sync_every iterations.  The edges without overlap (parked by the filter) take no part.
static void joint_loop(Ctx& c, Batch& b, PairsRun& r) {
  JointRun& j = *r.joint;
  cudaStream_t st = c.stream;
  const int n_edges = r.n_pairs;
  std::vector<char> live((size_t)n_edges);
  for (int e = 0; e < n_edges; ++e) live[(size_t)e] = !r.no_overlap[(size_t)e];
  check_anchored(j, live, SICP_ERR_NO_OVERLAP, "a free cloud has no path to a fixed cloud over edges with overlap");
  // the common centre: the box centre of the first live edge's movable cloud, in the world (of the
  // last edge when none is live: then priors hold every free cloud)
  int e0 = 0;
  while (e0 + 1 < n_edges && !live[(size_t)e0]) ++e0;
  double cw[3];
  const double* cm = r.pd[(size_t)e0].cm;
  rigid_apply(j.pose[(size_t)j.mov_id[e0]], cm[0], cm[1], cm[2], cw[0], cw[1], cw[2]);
  // the lower blocks every live edge touches, its edges in ascending order (dense), or the plan
  const int F = j.F;
  const bool sparse = c.joint_solver == 1;
  JointPlan plan;
  if (sparse) plan = joint_sparse_plan(j, live);
  std::vector<std::vector<int>> lists;
  std::vector<int> blk_of(sparse ? 0 : (size_t)F * F, -1);
  auto add = [&](int p, int q, int v) {
    int& bi = blk_of[(size_t)p * F + q];
    if (bi < 0) {
      bi = (int)lists.size();
      lists.emplace_back();
    }
    lists[(size_t)bi].push_back(v);
  };
  for (int e = 0; e < n_edges && !sparse; ++e) {
    if (!live[(size_t)e]) continue;
    const int fa = j.free_of[(size_t)j.fix_id[e]], fb = j.free_of[(size_t)j.mov_id[e]];
    if (fa >= 0) add(fa, fa, 2 * e + 1);
    if (fb >= 0) add(fb, fb, 2 * e);
    if (fa >= 0 && fb >= 0) add(std::max(fa, fb), std::min(fa, fb), 2 * e);
  }
  // the relative observations' blocks, after the edges' (a block only they touch has no edges)
  std::vector<std::vector<int>> rel;
  if (!sparse) {
    rel = joint_rel_lists(j, [&](int p, int q) {
      int& bi = blk_of[(size_t)p * F + q];
      if (bi < 0) {
        bi = (int)lists.size();
        lists.emplace_back();
      }
      return bi;
    });
    rel.resize(lists.size());
  }
  std::vector<int> ids;
  ids.insert(ids.end(), j.fix_id, j.fix_id + n_edges);
  ids.insert(ids.end(), j.mov_id, j.mov_id + n_edges);
  ids.insert(ids.end(), j.free_of.begin(), j.free_of.end());
  ids.insert(ids.end(), j.free_ids.begin(), j.free_ids.end());
  ids.insert(ids.end(), blk_of.begin(), blk_of.end());
  const auto [o_off, o_edge] = append_lists(ids, lists);
  const SparseIds so = sparse ? joint_sparse_ids(j, live, plan, ids) : SparseIds{};
  const int n_prior = (int)j.poses.size();
  const size_t o_prior = ids.size();
  if (n_prior > 0) ids.insert(ids.end(), j.prior_of.begin(), j.prior_of.end());
  const int n_rel = (int)j.rels.size();
  const std::pair<size_t, size_t> o_rel = sparse ? so.rel : n_rel > 0 ? append_lists(ids, rel) : so.rel;

  JointStore& js = b.joint;
  const int npad = (6 * F + 1 + 31) / 32 * 32;
  js.n_clouds = j.n_clouds;
  js.n_edges = n_edges;
  js.F = F;
  js.npad = npad;
  for (int k = 0; k < 3; ++k) js.cw[k] = cw[k];
  js.role.assign((size_t)j.n_clouds, 0);
  for (int e = 0; e < n_edges; ++e)
    for (int cl : {j.fix_id[e], j.mov_id[e]}) js.role[(size_t)cl] = j.free_of[(size_t)cl] >= 0 ? 2 : 1;
  js.cov_done = false;
  js.sparse = sparse;
  js.n_prior = n_prior;
  if (n_prior > 0) {
    js.prior.reserve(n_prior);
    SICP_CUDA(cudaMemcpyAsync(js.prior.p, j.poses.data(), sizeof(JointPrior) * (size_t)n_prior,
                              cudaMemcpyHostToDevice, st));
  }
  js.n_rel = n_rel;
  if (n_rel > 0) {
    js.rel.reserve(n_rel);
    SICP_CUDA(cudaMemcpyAsync(js.rel.p, j.rels.data(), sizeof(JointRel) * (size_t)n_rel, cudaMemcpyHostToDevice, st));
    if (!sparse) js.rel_y.reserve(6 * (size_t)F);
  }
  js.edges.reserve(n_edges);
  js.flags.reserve(1);
  js.pose.reserve(j.n_clouds);
  js.ids.reserve(ids.size());
  if (!sparse) js.A.reserve((size_t)npad * npad);
  js.bar.reserve(2);
  if (sparse) {
    js.sp_panel.reserve(plan.panel.size());
    js.sp_L.reserve((size_t)plan.panel.back());
    js.sp_x.reserve(15 * (size_t)F);
    js.sp_flags.reserve(1 + (size_t)c.num_sms);
    SICP_CUDA(cudaMemcpyAsync(js.sp_panel.p, plan.panel.data(), sizeof(long long) * plan.panel.size(),
                              cudaMemcpyHostToDevice, st));
    SICP_CUDA(cudaMemsetAsync(js.sp_flags.p, 0, sizeof(int), st));
    std::vector<double> dc(3 * (size_t)F);
    for (int f = 0; f < F; ++f)
      for (int k = 0; k < 3; ++k) dc[3 * (size_t)f + k] = j.pose[(size_t)j.free_ids[(size_t)f]].t[k] - cw[k];
    SICP_CUDA(cudaMemcpyAsync(js.sp_x.p + 12 * (size_t)F, dc.data(), sizeof(double) * dc.size(),
                              cudaMemcpyHostToDevice, st));
  }
  if (!js.flags_host) SICP_CUDA(cudaMallocHost(&js.flags_host, sizeof(JointFlags)));
  SICP_CUDA(cudaMemsetAsync(js.edges.p, 0, sizeof(JointEdge) * (size_t)n_edges, st));
  SICP_CUDA(cudaMemsetAsync(js.flags.p, 0, sizeof(JointFlags), st));
  SICP_CUDA(cudaMemsetAsync(js.bar.p, 0, 2 * sizeof(unsigned int), st));
  SICP_CUDA(cudaMemcpyAsync(js.pose.p, j.pose.data(), sizeof(Rigid) * j.pose.size(), cudaMemcpyHostToDevice, st));
  SICP_CUDA(cudaMemcpyAsync(js.ids.p, ids.data(), sizeof(int) * ids.size(), cudaMemcpyHostToDevice, st));

  const sicp_run_params& p = r.rp->run;
  JointArgs a{};
  a.pairs = b.pairs.p;
  a.state = b.state.p;
  a.edges = js.edges.p;
  a.flags = js.flags.p;
  a.dist = b.dist.p;
  a.q_nrm = b.q_nrm.p;
  a.m_xyz = b.m_xyz.p;
  a.keep = b.keep.p;
  a.rec = b.rec.p;
  a.rec_stride = p.max_iterations;
  a.pose = js.pose.p;
  a.fix_id = js.ids.p;
  a.mov_id = js.ids.p + n_edges;
  a.free_of = js.ids.p + 2 * n_edges;
  a.free_ids = a.free_of + j.n_clouds;
  a.blk_of = a.free_ids + F;
  a.blk_off = js.ids.p + o_off;
  a.blk_edge = js.ids.p + o_edge;
  a.F = F;
  a.n_edges = n_edges;
  a.npad = npad;
  a.A = js.A.p;
  a.bar = js.bar.p;
  for (int k = 0; k < 3; ++k) a.cw[k] = cw[k];
  a.min_planarity = p.min_planarity;
  a.min_change = p.min_change;
  if (n_prior > 0) {
    a.prior = js.prior.p;
    a.prior_of = js.ids.p + o_prior;
    a.n_prior = n_prior;
  }
  JointRelArgs ra{};
  if (n_rel > 0) {
    ra.rel = js.rel.p;
    ra.off = js.ids.p + o_rel.first;
    ra.k = js.ids.p + o_rel.second;
    ra.y = sparse ? nullptr : js.rel_y.p;
    ra.n = n_rel;
  }
  JointSparseArgs sa{};
  if (sparse) {
    sa.j = a;
    sa.r = ra;
    sa.sn = reinterpret_cast<const JointSuper*>(js.ids.p + so.sn);
    sa.panel = js.sp_panel.p;
    sa.st = js.ids.p + so.st;
    sa.up = js.ids.p + so.up;
    sa.map = js.ids.p + so.map;
    sa.lv_off = js.ids.p + so.lv_off;
    sa.lv = js.ids.p + so.lv;
    sa.perm = js.ids.p + so.perm;
    sa.blk = js.ids.p + so.blk;
    sa.lst_off = js.ids.p + so.lst_off;
    sa.lst_edge = js.ids.p + so.lst_edge;
    sa.depth = plan.depth;
    sa.L = js.sp_L.p;
    sa.x = js.sp_x.p;
    sa.xf = js.sp_x.p + 6 * (size_t)F;
    sa.dc = js.sp_x.p + 12 * (size_t)F;
    sa.bad = js.sp_flags.p;
    sa.conv = js.sp_flags.p + 1;
    js.sp_args = sa;
    js.sp_plan = std::move(plan);
  }

  // device events around the three stages of the iterations queued since the last host read (match,
  // reject + blocks, solve + update: sicp_timings), read at each host read.  The host reads at
  // iteration 1 and then every `every` iterations, so every + 1 sets suffice; they are created once
  // per call and destroyed on every way out.
  struct Events {
    std::vector<cudaEvent_t> ev;
    ~Events() {
      for (cudaEvent_t e : ev)
        if (e) cudaEventDestroy(e);
    }
  } evs;
  const int every = std::max(1, c.host_sync_every);
  evs.ev.assign(4 * (size_t)(every + 1), nullptr);
  for (cudaEvent_t& e : evs.ev) SICP_CUDA(cudaEventCreate(&e));
  int queued = 0;
  double t3[3] = {0, 0, 0};
  int next_sync = 1;
  for (int it = 0; it < p.max_iterations; ++it) {
    a.it = it;
    a.last = it + 1 == p.max_iterations;
    cudaEvent_t* e = evs.ev.data() + 4 * queued++;
    SICP_CUDA(cudaEventRecord(e[0], st));
    batch_match_launch(c, b, c.warm_start && it > 0);
    SICP_CUDA(cudaEventRecord(e[1], st));
    joint_reject_launch(c, a, n_edges);
    if (n_prior > 0) joint_prior_launch(c, a, sparse ? sa.dc : nullptr);
    if (n_rel > 0) joint_relative_launch(c, a, ra, sparse ? sa.dc : nullptr);
    SICP_CUDA(cudaEventRecord(e[2], st));
    if (sparse) {
      sa.j.it = it;
      sa.j.last = a.last;
      joint_sparse_solve_launch(c, sa);
    } else {
      joint_solve_launch(c, a, ra);
    }
    SICP_CUDA(cudaEventRecord(e[3], st));
    if (it >= next_sync || a.last) {
      next_sync = it + every;
      SICP_CUDA(cudaMemcpyAsync(js.flags_host, js.flags.p, sizeof(JointFlags), cudaMemcpyDeviceToHost, st));
      SICP_CUDA(cudaStreamSynchronize(st));
      for (int q = 0; q < queued; ++q)
        for (int k = 0; k < 3; ++k) {
          float ms = 0;
          SICP_CUDA(cudaEventElapsedTime(&ms, evs.ev[4 * (size_t)q + k], evs.ev[4 * (size_t)q + k + 1]));
          t3[k] += ms;
        }
      queued = 0;
      if (js.flags_host->done) break;
    }
  }
  c.tm.match_ms = t3[0];
  c.tm.reject_solve_ms = t3[1];
  c.tm.transform_ms = t3[2];
  SICP_REQUIRE(!js.flags_host->singular, SICP_ERR_SINGULAR,
               "the joint normal matrix is not positive definite (a free cloud is not constrained in all six "
               "degrees of freedom)");
  SICP_CUDA(cudaMemcpy(j.pose.data(), js.pose.p, sizeof(Rigid) * j.pose.size(), cudaMemcpyDeviceToHost));
}

// Everything after the fixed side: descriptors, [select + normals], the grids of the movable-only
// clouds, [overlap filter, select + normals], movable normals, the loop and the results.  fix_xyz
// holds the fixed coordinates the descriptors' fix_off index; map (or null) is the resident map of
// sicp_register_to_map, whose filter is the culled one.
static void run_pairs(Ctx& c, Batch& b, PairsRun& r, const double* fix_xyz, MapStore* map, long long max_n_fix,
                      sicp_pair_result* out, int64_t* n_selected) {
  cudaStream_t st = c.stream;
  const int n_pairs = r.n_pairs;
  const sicp_register_params* rp = r.rp;
  const sicp_run_params& p = rp->run;
  for (int i = 0; i < n_pairs; ++i) {
    PairDev& d = r.pd[(size_t)i];
    d.n_mov = r.mo[(size_t)i + 1] - r.mo[(size_t)i];
    d.K = std::min<long long>(rp->correspondences, d.n_fix);
    d.q_off = (long long)i * r.Kmax;
    for (int j = 0; j < 6; ++j) d.obs[j] = r.observed ? r.observed[6 * i + j] : p.lsq.observed[j];
  }
  const int round_away = c.variant != SICP_VARIANT_PYTHON;
  auto select_and_normals = [&]() {
    batch_select_gather_launch(c, b, fix_xyz, r.overlap, round_away);
    StageTimer t(c, &c.tm.normals_ms);
    normals_launch(c, &b, false, rp->neighbors);
    t.stop();
  };
  // without the filter the selection needs only the fixed side: it runs while the movable clouds
  // are still in flight; with it, the selection follows the filter, which needs the movable grids
  if (!r.overlap) {
    SICP_CUDA(cudaMemcpyAsync(b.pairs.p, r.pd.data(), sizeof(PairDev) * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
    select_and_normals();
  }

  // ---- movable side: the grids of the movable-only clouds, once they have arrived
  c.tm.grid_mov_ms = 0;
  if (!r.mov_clouds.empty()) {
    SICP_CUDA(cudaStreamWaitEvent(st, c.ev_copy, 0));
    std::vector<GridView> views;
    std::vector<double> centres;
    {
      StageTimer t(c, &c.tm.grid_mov_ms);
      grid_build(c, b.gmov, r.mov_clouds, batch_policy(c), views, centres);
      t.stop();
    }
    for (int i = 0; i < n_pairs; ++i) {
      const int s = r.mov_slot[(size_t)i];
      if (s < 0) continue;
      r.pd[(size_t)i].gmov = views[(size_t)s];
      for (int a = 0; a < 3; ++a) r.pd[(size_t)i].cm[a] = centres[(size_t)s * 3 + a];
    }
  }
  r.no_overlap.assign((size_t)n_pairs, 0);
  c.tm.overlap_ms = 0;
  if (r.overlap) {
    SICP_CUDA(cudaMemcpyAsync(b.pairs.p, r.pd.data(), sizeof(PairDev) * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
    StageTimer t(c, &c.tm.overlap_ms);
    if (map) map_filter(c, b, *map, r);
    else batch_filter(c, b, r, fix_xyz, max_n_fix);
    t.stop();
  }
  SICP_CUDA(cudaMemcpyAsync(b.pairs.p, r.pd.data(), sizeof(PairDev) * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
  if (r.overlap) select_and_normals();
  // pc_mov.estimate_normals(mov_neighbors) of every movable cloud, once, in its own grid
  b.mov_attr = rp->mov_neighbors > 0;
  b.mov_cos_max = b.mov_attr ? mov_cos_max_of(rp->max_angle_rad) : -1.0;
  c.tm.mov_normals_ms = 0;
  if (b.mov_attr) {
    b.q_nrm_eff.reserve((size_t)n_pairs * (size_t)r.Kmax);
    if (r.mov_first.empty() || r.mov_first.size() == (size_t)n_pairs) {
      b.mov_desc = b.pairs.p;
      b.n_mov_desc = n_pairs;
    } else {
      std::vector<PairDev> desc;
      for (int i : r.mov_first) desc.push_back(r.pd[(size_t)i]);
      b.mov_pairs.reserve(desc.size());
      SICP_CUDA(cudaMemcpyAsync(b.mov_pairs.p, desc.data(), sizeof(PairDev) * desc.size(), cudaMemcpyHostToDevice, st));
      b.mov_desc = b.mov_pairs.p;
      b.n_mov_desc = (int)desc.size();
    }
    StageTimer t(c, &c.tm.mov_normals_ms);
    b.max_n_mov = r.max_n_mov;
    normals_launch(c, &b, true, rp->mov_neighbors);
    t.stop();
  }

  // ---- the loop: two launches per iteration for the whole batch
  cudaEvent_t e0, e1;
  SICP_CUDA(cudaEventCreate(&e0));
  SICP_CUDA(cudaEventCreate(&e1));
  SICP_CUDA(cudaEventRecord(e0, st));
  const int every = std::max(1, c.host_sync_every);
  int next_sync = 1;
  if (r.joint) joint_loop(c, b, r);
  for (int it = 0; !r.joint && it < p.max_iterations; ++it) {
    batch_match_launch(c, b, c.warm_start && it > 0);
    batch_rs_launch(c, b, p, it, it + 1 == p.max_iterations);
    if (it >= next_sync || it + 1 == p.max_iterations) {
      next_sync = it + every;
      k_gather_flags<<<(n_pairs + 127) / 128, 128, 0, st>>>(b.state.p, n_pairs, b.flags.p);
      SICP_CUDA(cudaMemcpyAsync(b.flags_host, b.flags.p, sizeof(int) * 2 * (size_t)n_pairs, cudaMemcpyDeviceToHost, st));
      SICP_CUDA(cudaStreamSynchronize(st));
      bool running = false;
      for (int i = 0; i < n_pairs; ++i) {
        const int stop = b.flags_host[2 * i], done = b.flags_host[2 * i + 1];
        // a pair without a stop flag that is not keeping up ran out of correspondences (< 6): it
        // stays where it is; everybody else decides
        if (stop == 0 && done == it + 1) running = true;
      }
      if (!running) break;
    }
  }
  SICP_CUDA(cudaEventRecord(e1, st));
  batch_finish_launch(c, b, p.max_iterations);
  SICP_CUDA(cudaMemcpyAsync(b.results_host, b.results.p, sizeof(sicp_pair_result) * (size_t)n_pairs,
                            cudaMemcpyDeviceToHost, st));
  SICP_CUDA(cudaStreamSynchronize(st));
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  if (!r.joint) c.tm.reject_solve_ms = ms;
  std::memcpy(out, b.results_host, sizeof(sicp_pair_result) * (size_t)n_pairs);
  for (int i = 0; i < n_pairs; ++i) {
    if (r.no_overlap[(size_t)i]) out[i].status = SICP_ERR_NO_OVERLAP;
    if (n_selected) n_selected[i] = r.pd[(size_t)i].K;
  }
  // what sicp_get_batch_outputs needs of this call (host bookkeeping only)
  b.out_n_pairs = n_pairs;
  b.out_max_iterations = p.max_iterations;
  b.out_n_mov.resize((size_t)n_pairs);
  b.out_n_kept.resize((size_t)n_pairs);
  b.out_status.resize((size_t)n_pairs);
  b.out_iterations.resize((size_t)n_pairs);
  b.out_mean_std.resize(2 * (size_t)n_pairs);
  for (int i = 0; i < n_pairs; ++i) {
    b.out_n_mov[(size_t)i] = r.pd[(size_t)i].n_mov;
    b.out_n_kept[(size_t)i] = out[i].n_kept;
    b.out_status[(size_t)i] = out[i].status;
    b.out_iterations[(size_t)i] = out[i].iterations;
    b.out_mean_std[2 * (size_t)i] = out[i].mean_res;
    b.out_mean_std[2 * (size_t)i + 1] = out[i].std_res;
  }
  b.out_valid = true;
  b.out_joint = r.joint != nullptr;
}

// The selected inversion's device inputs after a sparse call (DESIGN.md §6.14), checked before any
// launch: pos and the parked edges (both clouds free, their pair outside the pattern of L) into
// js.sel_ids, Z and y' into js.Z (the factor's size), the blocks of k_joint_sel_parked in *blocks.
static JointSelArgs joint_sel_args(Ctx& c, JointStore& js, int* blocks) {
  const JointPlan& pl = js.sp_plan;
  const int F = js.F;
  SICP_REQUIRE(pl.depth <= JOINT_SEL_MAX_PATH, SICP_ERR_BAD_ARG,
               "selected covariances: the elimination tree of this edge graph is " + std::to_string(pl.depth) +
                   " levels deep, more than " + std::to_string(JOINT_SEL_MAX_PATH));
  auto owner = [&](int p) { return (int)(std::upper_bound(pl.first.begin(), pl.first.end(), p) - pl.first.begin()) - 1; };
  auto path_len = [&](int p) {  // the unknowns of the supernodes from p's to its root
    long long n = 0;
    for (int k = owner(p); k >= 0; k = pl.parent[(size_t)k]) n += 6 * pl.ns(k);
    return n;
  };
  // the edges' clouds and the free index of every cloud, from the head of the call's ids
  std::vector<int> h_ids(2 * (size_t)js.n_edges + js.n_clouds);
  SICP_CUDA(cudaMemcpy(h_ids.data(), js.ids.p, sizeof(int) * h_ids.size(), cudaMemcpyDeviceToHost));
  const int *fix_id = h_ids.data(), *mov_id = fix_id + js.n_edges, *free_of = mov_id + js.n_edges;
  std::vector<int> ids(pl.pos.begin(), pl.pos.end());
  long long need = 0;
  for (int e = 0; e < js.n_edges; ++e) {
    const int fa = free_of[fix_id[e]], fb = free_of[mov_id[e]];
    if (fa < 0 || fb < 0) continue;
    const int pa = pl.pos[(size_t)fa], pb = pl.pos[(size_t)fb], lo = std::min(pa, pb), hi = std::max(pa, pb);
    const int k = owner(lo);
    if (hi < pl.first[(size_t)k + 1] ||
        std::binary_search(pl.st.begin() + pl.st_off[(size_t)k], pl.st.begin() + pl.st_off[(size_t)k + 1], hi))
      continue;
    ids.push_back(e);
    need = std::max(need, 6 * (path_len(pa) + path_len(pb)));
  }
  const int n_parked = (int)ids.size() - F;
  const long long zsize = pl.panel.back() - 6ll * F;
  *blocks = n_parked > 0 ? (int)std::min<long long>({(long long)n_parked, (long long)c.num_sms, zsize / need}) : 0;
  SICP_REQUIRE(n_parked == 0 || *blocks > 0, SICP_ERR_BAD_ARG,
               "selected covariances: an edge outside the factor's pattern needs more scratch than the factor holds");
  js.Z.reserve((size_t)pl.panel.back());
  js.sel_ids.reserve(ids.size());
  SICP_CUDA(cudaMemcpyAsync(js.sel_ids.p, ids.data(), sizeof(int) * ids.size(), cudaMemcpyHostToDevice, c.stream));
  JointSelArgs g{};
  g.s = js.sp_args;
  g.Z = js.Z.p;
  g.y = js.Z.p + zsize;
  g.pos = js.sel_ids.p;
  g.parked = js.sel_ids.p + F;
  g.n_parked = n_parked;
  g.scratch = need;
  return g;
}

// sicp_get_joint_covariances (selected false) and sicp_get_joint_selected_covariances (true): the
// first request after a sicp_register_joint runs joint_cov_launch (a dense call) or joint_sel_launch
// (a sparse one) on what its final iteration left and keeps the result on the host; every later one
// copies it.
static void get_joint_covariances(Ctx& c, int n_clouds, double* cloud_cov, int n_edges, double* edge_cov,
                                  double* s0, bool selected) {
  SICP_REQUIRE(c.batch && c.batch->out_valid && c.batch->out_joint, SICP_ERR_STATE,
               "no joint covariances: the last batched call on this context was not a successful "
               "sicp_register_joint, or a later call cleared its outputs");
  Batch& b = *c.batch;
  JointStore& js = b.joint;
  SICP_REQUIRE(selected || !js.sparse, SICP_ERR_STATE,
               "covariances need joint_solver 0 (sicp_get_joint_selected_covariances serves both solvers)");
  SICP_REQUIRE(n_clouds == js.n_clouds && n_edges == js.n_edges, SICP_ERR_BAD_ARG,
               "n_clouds and n_edges must equal the last sicp_register_joint's (" + std::to_string(js.n_clouds) +
                   ", " + std::to_string(js.n_edges) + ")");
  if (!js.cov_done) {
    const int F = js.F, ne = js.n_edges;
    JointSelArgs g{};
    int parked_blocks = 0;
    if (js.sparse) g = joint_sel_args(c, js, &parked_blocks);
    else js.Z.reserve((size_t)js.npad * js.npad);
    js.cov.reserve((size_t)ne + 1 + 36 * ((size_t)F + ne));
    JointCovArgs a{};
    a.pairs = b.pairs.p;
    a.state = b.state.p;
    a.keep = b.keep.p;
    a.m_xyz = b.m_xyz.p;
    a.q_xyz = b.q_xyz.p;
    a.q_nrm = b.q_nrm.p;
    a.edges = js.edges.p;
    a.pose = js.pose.p;
    a.fix_id = js.ids.p;
    a.mov_id = js.ids.p + ne;
    a.free_of = js.ids.p + 2 * ne;
    a.free_ids = a.free_of + js.n_clouds;
    a.L = js.A.p;
    a.Z = js.Z.p;
    a.ss = js.cov.p;
    a.s0sq = a.ss + ne;
    a.cov_f = a.s0sq + 1;
    a.cov_e = a.cov_f + 36 * (size_t)F;
    a.bar = js.bar.p;
    a.F = F;
    a.n_edges = ne;
    a.npad = js.npad;
    for (int k = 0; k < 3; ++k) a.cw[k] = js.cw[k];
    a.prior = js.prior.p;
    a.n_prior = js.n_prior;
    a.rel = js.rel.p;
    a.rel_y = js.sparse ? g.y : js.rel_y.p;
    a.n_rel = js.n_rel;
    if (js.sparse) {
      g.c = a;
      joint_sel_launch(c, g, parked_blocks);
    } else {
      joint_cov_launch(c, a);
    }
    std::vector<double> h(1 + 36 * ((size_t)F + ne));
    SICP_CUDA(cudaMemcpyAsync(h.data(), a.s0sq, sizeof(double) * h.size(), cudaMemcpyDeviceToHost, c.stream));
    SICP_CUDA(cudaStreamSynchronize(c.stream));
    const double nan = std::nan(""), s0sq = h[0];
    js.s0 = std::sqrt(s0sq);
    // a fixed cloud some edge references: 0 (NaN with s0); one no edge references: NaN
    js.cov_cloud.assign(36 * (size_t)js.n_clouds, std::isnan(s0sq) ? nan : 0.0);
    for (int i = 0, f = 0; i < js.n_clouds; ++i) {
      double* dst = js.cov_cloud.data() + 36 * (size_t)i;
      if (js.role[(size_t)i] == 2) std::memcpy(dst, h.data() + 1 + 36 * (size_t)f++, sizeof(double) * 36);
      else if (js.role[(size_t)i] == 0) std::fill(dst, dst + 36, nan);
    }
    js.cov_edge.assign(h.begin() + 1 + 36 * (size_t)F, h.end());
    js.cov_done = true;
  }
  if (cloud_cov) std::memcpy(cloud_cov, js.cov_cloud.data(), sizeof(double) * js.cov_cloud.size());
  if (edge_cov) std::memcpy(edge_cov, js.cov_edge.data(), sizeof(double) * js.cov_edge.size());
  if (s0) *s0 = js.s0;
}

// sicp_get_batch_outputs: everything is read from the buffers the last run_pairs left behind.
// One launch transforms the requested clouds, one compacts the requested residual vectors, one
// copy brings the log and one the transforms; each requested pair's slice then goes to the
// caller's memory with its own copy (any memory kind, any alignment).
static void get_batch_outputs(Ctx& c, int n_pairs, double* const* mov_xyz_out, double* const* residuals,
                              sicp_iter_record* log, double* T) {
  SICP_REQUIRE(c.batch && c.batch->out_valid, SICP_ERR_STATE,
               "no batch outputs: no sicp_register_batch / sicp_register_to_map / sicp_register_pairs has "
               "succeeded since the last sicp_set_map");
  Batch& b = *c.batch;
  SICP_REQUIRE(n_pairs == b.out_n_pairs, SICP_ERR_BAD_ARG,
               "n_pairs must equal the last batched call's (" + std::to_string(b.out_n_pairs) + ")");
  cudaStream_t st = c.stream;
  const int n = n_pairs;
  const auto ok = [&](int i) { return b.out_status[(size_t)i] == SICP_OK; };
  const auto n_mov = [&](int i) { return b.out_n_mov[(size_t)i]; };
  // requested pairs: transforms first, then residual vectors, each with its output offset
  std::vector<int> ids;
  std::vector<long long> off;
  long long max_n_mov = 0, n_pts = 0, n_res = 0;
  if (mov_xyz_out)
    for (int i = 0; i < n; ++i)
      if (ok(i) && mov_xyz_out[i]) {
        ids.push_back(i);
        off.push_back(n_pts);
        n_pts += n_mov(i);
        max_n_mov = std::max(max_n_mov, n_mov(i));
      }
  const int n_xyz = (int)ids.size();
  if (residuals)
    for (int i = 0; i < n; ++i)
      if (ok(i) && residuals[i] && b.out_n_kept[(size_t)i] > 0) {
        ids.push_back(i);
        off.push_back(n_res);
        n_res += b.out_n_kept[(size_t)i];
      }
  const int n_rv = (int)ids.size() - n_xyz;
  if (!ids.empty()) {
    b.out_ids.reserve(ids.size());
    b.out_off.reserve(off.size());
    SICP_CUDA(cudaMemcpyAsync(b.out_ids.p, ids.data(), sizeof(int) * ids.size(), cudaMemcpyHostToDevice, st));
    SICP_CUDA(cudaMemcpyAsync(b.out_off.p, off.data(), sizeof(long long) * off.size(), cudaMemcpyHostToDevice, st));
  }
  if (n_xyz > 0) {
    b.xyz_out.reserve(3 * (size_t)n_pts);
    batch_transform_launch(c, b, b.out_ids.p, n_xyz, b.out_off.p, max_n_mov, b.xyz_out.p);
    for (int j = 0; j < n_xyz; ++j) {
      const int i = ids[(size_t)j];
      copy_any(c, mov_xyz_out[i], b.xyz_out.p + 3 * off[(size_t)j], sizeof(double) * 3 * (size_t)n_mov(i));
    }
  }
  if (n_rv > 0) {
    b.resid_out.reserve((size_t)n_res);
    batch_residuals_launch(c, b, b.out_ids.p + n_xyz, n_rv, b.out_off.p + n_xyz, b.resid_out.p);
    for (int j = 0; j < n_rv; ++j) {
      const int i = ids[(size_t)(n_xyz + j)];
      copy_any(c, residuals[i], b.resid_out.p + off[(size_t)(n_xyz + j)], sizeof(double) * (size_t)b.out_n_kept[(size_t)i]);
    }
  }
  const size_t it_max = (size_t)b.out_max_iterations;
  if (log) {
    pinned_reserve(b.rec_host, b.rec_cap, (size_t)n * it_max);
    SICP_CUDA(cudaMemcpyAsync(b.rec_host, b.rec.p, sizeof(sicp_iter_record) * (size_t)n * it_max,
                              cudaMemcpyDeviceToHost, st));
  }
  if (T) {
    pinned_reserve(b.T_host, b.T_cap, (size_t)n);
    SICP_CUDA(cudaMemcpy2DAsync(b.T_host, sizeof(Rigid), reinterpret_cast<const char*>(b.state.p) + offsetof(DevState, T),
                                sizeof(DevState), sizeof(Rigid), (size_t)n, cudaMemcpyDeviceToHost, st));
  }
  SICP_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    if (!ok(i)) continue;
    if (log) {
      const size_t done = std::min<size_t>((size_t)b.out_iterations[(size_t)i], it_max);
      sicp_iter_record* dst = log + (size_t)i * it_max;
      std::memcpy(dst, b.rec_host + (size_t)i * it_max, sizeof(sicp_iter_record) * done);
      std::memset(dst + done, 0, sizeof(sicp_iter_record) * (it_max - done));
      // the last row carries the exact two-pass statistics, as sicp_register's log does
      if (done > 0) {
        dst[done - 1].mean_res = b.out_mean_std[2 * (size_t)i];
        dst[done - 1].std_res = b.out_mean_std[2 * (size_t)i + 1];
      }
    }
    if (T) H_from_rigid(b.T_host[i], T + 16 * (size_t)i);
  }
}

static void set_map(Ctx& c, const double* map_xyz, int64_t n_map) {
  if (c.batch) c.batch->out_valid = false;
  if (map_xyz == nullptr || n_map == 0) {
    delete c.map;
    c.map = nullptr;
    return;
  }
  SICP_REQUIRE(n_map > 0 && n_map < (1ll << 32), SICP_ERR_BAD_ARG, "n_map must be in [1, 2^32 - 1]");
  if (!c.map) c.map = new MapStore();
  MapStore& m = *c.map;
  m.n = 0;  // no map until the new one is complete
  m.xyz.reserve(3 * (size_t)n_map);
  {
    StageTimer t(c, &c.tm.upload_ms);
    upload_to_device(c, m.xyz.p, map_xyz, sizeof(double) * 3 * (size_t)n_map);
    t.stop();
  }
  std::vector<GridView> views;
  std::vector<double> centres;
  {
    StageTimer t(c, &c.tm.grid_fix_ms);
    grid_build(c, m.grid, {HostCloud{m.xyz.p, n_map, 0}}, batch_policy(c), views, centres);
    t.stop();
  }
  m.view = views[0];
  m.n = n_map;
}

static void register_to_map(Ctx& c, int n_scans, const double* const* mov_xyz, const int64_t* n_mov,
                            const sicp_register_params* rp, const double* observed, sicp_pair_result* out,
                            int64_t* n_selected) {
  if (c.batch) c.batch->out_valid = false;
  check_pairs_params(c, n_scans, mov_xyz && n_mov && out, rp);
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  MapStore& m = *c.map;
  SICP_REQUIRE(m.n >= rp->neighbors, SICP_ERR_BAD_ARG, "the map needs at least `neighbors` points");
  SICP_REQUIRE((long long)n_scans * m.n < (1ll << 32), SICP_ERR_BAD_ARG,
               "n_scans x n_map must be below 2^32 (32-bit survivor offsets): use fewer scans per call");
  PairsRun r;
  begin_pairs(r, n_scans, rp, observed);
  for (int i = 0; i < n_scans; ++i) {
    SICP_REQUIRE(mov_xyz[i], SICP_ERR_BAD_ARG, "cloud pointer is NULL");
    SICP_REQUIRE(n_mov[i] >= 1, SICP_ERR_BAD_ARG, "every movable cloud needs at least one point");
    add_movable(r, i, n_mov[i]);
  }
  if (!c.batch) c.batch = new Batch();
  Batch& b = *c.batch;
  r.Kmax = (std::min<long long>(rp->correspondences, m.n) + 1) & ~1ll;
  b.total_mov = r.mo[(size_t)n_scans];
  c.tm.overlap_candidates = 0;
  b.xyz.reserve(3 * (size_t)b.total_mov);
  SICP_CUDA(cudaEventRecord(c.ev_user, c.stream));
  SICP_CUDA(cudaStreamWaitEvent(c.copy_stream, c.ev_user, 0));  // buffers of an earlier call are free
  std::vector<int> scans((size_t)n_scans);
  for (int i = 0; i < n_scans; ++i) scans[(size_t)i] = i;
  upload_movable(c, b, r, scans, mov_xyz, n_mov, r.mo);
  alloc_pair_buffers(c, b, r);
  for (int i = 0; i < n_scans; ++i) {
    r.pd[(size_t)i].gfix = m.view;
    r.pd[(size_t)i].n_fix = m.n;
    r.pd[(size_t)i].fix_off = r.pd[(size_t)i].flag_off = 0;
    r.pd[(size_t)i].mov_off = r.mo[(size_t)i];
    r.mov_slot[(size_t)i] = i;
  }
  run_pairs(c, b, r, m.xyz.p, &m, m.n, out, n_selected);
}

// sicp_register_pairs: pair i is (cloud fix_id[i], cloud mov_id[i]).  Every referenced cloud is
// uploaded once into the store Batch::xyz and gridded once: in Batch::gfix if it is fixed in some
// pair (that grid is also its movable grid), else in Batch::gmov by run_pairs (a grid depends only
// on its own cloud).  The movable normals run once per distinct movable cloud.  Each pair has its
// own keep flags (flag_off) and its own output slices, so pairs that share a cloud never write
// into a shared slice.
static void register_pairs(Ctx& c, int n_clouds, const double* const* xyz, const int64_t* n, int n_pairs,
                           const int32_t* fix_id, const int32_t* mov_id, const sicp_register_params* rp,
                           const double* observed, sicp_pair_result* out, int64_t* n_selected,
                           JointRun* joint = nullptr) {
  if (c.batch) c.batch->out_valid = false;
  check_pairs_params(c, n_pairs, xyz && n && fix_id && mov_id && out, rp);
  SICP_REQUIRE(n_clouds >= 1, SICP_ERR_BAD_ARG, "n_clouds must be >= 1");
  // role[j]: bit 0 = fixed in some pair, bit 1 = movable in some pair; 0 = not read
  std::vector<int> role((size_t)n_clouds, 0);
  for (int i = 0; i < n_pairs; ++i) {
    SICP_REQUIRE(fix_id[i] >= 0 && fix_id[i] < n_clouds && mov_id[i] >= 0 && mov_id[i] < n_clouds,
                 SICP_ERR_BAD_ARG, "pair " + std::to_string(i) + ": cloud ids must be in [0, n_clouds)");
    role[(size_t)fix_id[i]] |= 1;
    role[(size_t)mov_id[i]] |= 2;
  }
  // the store, the overlap flags and their prefix sums are indexed with 32-bit offsets
  constexpr long long k32 = 1ll << 32;
  long long total = 0;
  for (int j = 0; j < n_clouds; ++j) {
    if (!role[(size_t)j]) continue;
    SICP_REQUIRE(xyz[j], SICP_ERR_BAD_ARG, "cloud pointer is NULL");
    SICP_REQUIRE(n[j] >= 1 && (!(role[(size_t)j] & 1) || n[j] >= rp->neighbors), SICP_ERR_BAD_ARG,
                 "every fixed cloud needs at least `neighbors` points, every movable cloud one");
    SICP_REQUIRE(n[j] < k32 - total, SICP_ERR_BAD_ARG, "the points of the referenced clouds must be below 2^32");
    total += n[j];
  }
  // the store holds the movable-only clouds, then the clouds in both roles, then the fixed-only
  // ones: the movable clouds are its prefix [0, total_mov), the fixed-role ones its suffix from
  // fix0; slot[j] is cloud j's place in mov_only or in fixed
  std::vector<long long> off((size_t)n_clouds, -1);
  std::vector<int> mov_only, fixed, slot((size_t)n_clouds, -1);
  long long at = 0, fix0 = 0, total_mov = 0;
  for (int rl : {2, 3, 1}) {
    if (rl == 3) fix0 = at;
    if (rl == 1) total_mov = at;
    for (int j = 0; j < n_clouds; ++j) {
      if (role[(size_t)j] != rl) continue;
      off[(size_t)j] = at;
      at += n[j];
      std::vector<int>& list = rl == 2 ? mov_only : fixed;
      slot[(size_t)j] = (int)list.size();
      list.push_back(j);
    }
  }
  PairsRun r;
  begin_pairs(r, n_pairs, rp, observed);
  if (joint) {
    r.joint = joint;
    r.prior = joint->prior.data();
  }
  std::vector<long long> fo((size_t)n_pairs + 1, 0);  // the pairs' flag offsets
  std::vector<char> seen((size_t)n_clouds, 0);
  long long Kmax = 0, max_n_fix = 0;
  for (int i = 0; i < n_pairs; ++i) {
    const long long nf = n[fix_id[i]];
    add_movable(r, i, n[mov_id[i]]);  // mov_neighbors <= the movable cloud's points
    fo[(size_t)i + 1] = fo[(size_t)i] + nf;
    SICP_REQUIRE(fo[(size_t)i + 1] < k32, SICP_ERR_BAD_ARG,
                 "the fixed points of all pairs must be below 2^32 (32-bit overlap flags and offsets)");
    Kmax = std::max<long long>(Kmax, std::min<long long>(rp->correspondences, nf));
    max_n_fix = std::max(max_n_fix, nf);
    if (!seen[(size_t)mov_id[i]]) {
      seen[(size_t)mov_id[i]] = 1;
      r.mov_first.push_back(i);
    }
  }
  if (!c.batch) c.batch = new Batch();
  Batch& b = *c.batch;
  r.Kmax = (Kmax + 1) & ~1ll;  // even: every pair's slice of the per-query arrays starts 16-byte aligned
  b.total_fix = fo[(size_t)n_pairs];
  b.total_mov = total_mov;

  // ---- uploads: the fixed-role clouds on the context's stream, the movable-only ones behind them
  // on the copy stream, where they go on arriving while the fixed side computes
  b.xyz.reserve(3 * (size_t)total);
  SICP_CUDA(cudaStreamWaitEvent(c.stream, c.ev_copy, 0));  // copies into the store a failed call left in flight
  SICP_CUDA(cudaEventRecord(c.ev_user, c.stream));
  SICP_CUDA(cudaStreamWaitEvent(c.copy_stream, c.ev_user, 0));  // buffers of an earlier call are free
  {
    StageTimer t(c, &c.tm.upload_ms);
    for (int j : fixed)
      upload_to_device(c, b.xyz.p + 3 * off[(size_t)j], xyz[j], sizeof(double) * 3 * (size_t)n[j]);
    upload_movable(c, b, r, mov_only, xyz, n, off);
    alloc_pair_buffers(c, b, r);  // queued while the clouds cross PCIe
    t.stop();  // the fixed-role clouds have arrived
  }

  // ---- the grids of the fixed-role clouds (the movable-only clouds are still in flight)
  std::vector<HostCloud> clouds;
  for (int j : fixed) clouds.push_back(HostCloud{b.xyz.p + 3 * off[(size_t)j], n[j], off[(size_t)j] - fix0});
  std::vector<GridView> views;
  std::vector<double> centres;
  {
    StageTimer t(c, &c.tm.grid_fix_ms);
    grid_build(c, b.gfix, clouds, batch_policy(c), views, centres);
    t.stop();
  }
  for (int i = 0; i < n_pairs; ++i) {
    PairDev& d = r.pd[(size_t)i];
    const int f = slot[(size_t)fix_id[i]], m = slot[(size_t)mov_id[i]];
    d.gfix = views[(size_t)f];
    d.n_fix = n[fix_id[i]];
    d.fix_off = off[(size_t)fix_id[i]];
    d.flag_off = fo[(size_t)i];
    d.mov_off = off[(size_t)mov_id[i]];
    if (role[(size_t)mov_id[i]] == 2) {
      r.mov_slot[(size_t)i] = m;
      continue;
    }
    d.gmov = views[(size_t)m];
    for (int a = 0; a < 3; ++a) d.cm[a] = centres[(size_t)m * 3 + a];
  }
  run_pairs(c, b, r, b.xyz.p, nullptr, max_n_fix, out, n_selected);
}

// The variant of the context for the length of one call.
struct VariantScope {
  Ctx& c;
  int saved;
  VariantScope(Ctx& c_, int v) : c(c_), saved(c_.variant) { c.variant = v; }
  ~VariantScope() { c.variant = saved; }
};

// The pose priors of sicp_register_joint_priors (DESIGN.md §6.12), checked and kept in j: a prior is
// read for a free cloud with a non-zero weight; its pose must then be finite and rigid (to 1e-6, as
// sicp_overlap_graph's poses).  Every weight must be finite and >= 0.
static void check_joint_priors(JointRun& j, const double* prior_H, const double* prior_w) {
  j.full_prior.assign((size_t)j.n_clouds, 0);
  SICP_REQUIRE((prior_H == nullptr) == (prior_w == nullptr), SICP_ERR_BAD_ARG,
               "prior_H and prior_w must both be given or both be NULL");
  if (!prior_w) return;
  for (long long k = 0; k < 6ll * j.n_clouds; ++k)
    SICP_REQUIRE(std::isfinite(prior_w[k]) && prior_w[k] >= 0.0, SICP_ERR_BAD_ARG,
                 "prior_w[" + std::to_string(k / 6) + "] has a weight that is negative or not finite");
  j.prior_of.assign((size_t)j.F, -1);
  for (int f = 0; f < j.F; ++f) {
    const int i = j.free_ids[(size_t)f];
    const double* w = prior_w + 6 * (size_t)i;
    int nz = 0;
    for (int q = 0; q < 6; ++q) nz += w[q] != 0.0;
    if (nz == 0) continue;
    const double* h = prior_H + 16 * (size_t)i;
    for (int q = 0; q < 16; ++q)
      SICP_REQUIRE(std::isfinite(h[q]), SICP_ERR_BAD_ARG, "prior_H[" + std::to_string(i) + "] has non-finite entries");
    SICP_REQUIRE(h[12] == 0.0 && h[13] == 0.0 && h[14] == 0.0 && h[15] == 1.0, SICP_ERR_BAD_ARG,
                 "prior_H[" + std::to_string(i) + "] does not have the bottom row (0, 0, 0, 1)");
    for (int p = 0; p < 3; ++p)
      for (int q = 0; q < 3; ++q) {
        const double d = h[p] * h[q] + h[4 + p] * h[4 + q] + h[8 + p] * h[8 + q] - (p == q ? 1.0 : 0.0);
        SICP_REQUIRE(std::fabs(d) <= 1e-6, SICP_ERR_BAD_ARG,
                     "the rotation part of prior_H[" + std::to_string(i) + "] is not orthonormal (to 1e-6)");
      }
    JointPrior pr{};
    pr.P = rigid_from_H(h);
    for (int q = 0; q < 6; ++q) pr.w[q] = w[q];
    pr.f = f;
    j.prior_of[(size_t)f] = (int)j.poses.size();
    j.poses.push_back(pr);
    j.full_prior[(size_t)i] = nz == 6;
  }
}

// The relative observations of sicp_register_joint_relative (DESIGN.md §6.13), checked and kept in
// j: observation k is read when a weight is non-zero and an end is free; its Z must then be finite and
// rigid (to 1e-6).  Every observation must join two different clouds that some edge references, and
// every weight must be finite and >= 0.
static void check_joint_relative(JointRun& j, int n_rel, const int32_t* rel_a, const int32_t* rel_b,
                                 const double* rel_H, const double* rel_w) {
  SICP_REQUIRE(n_rel >= 0 && n_rel <= 65535, SICP_ERR_BAD_ARG, "n_rel must be in [0, 65535]");
  if (n_rel == 0) return;
  SICP_REQUIRE(rel_a && rel_b && rel_H && rel_w, SICP_ERR_BAD_ARG,
               "rel_a, rel_b, rel_H and rel_w must not be NULL when n_rel > 0");
  std::vector<char> used((size_t)j.n_clouds, 0);
  for (int e = 0; e < j.n_edges; ++e) used[(size_t)j.fix_id[e]] = used[(size_t)j.mov_id[e]] = 1;
  for (int k = 0; k < n_rel; ++k) {
    const std::string at = "relative observation " + std::to_string(k);
    const int a = rel_a[k], b = rel_b[k];
    SICP_REQUIRE(a >= 0 && a < j.n_clouds && b >= 0 && b < j.n_clouds, SICP_ERR_BAD_ARG,
                 at + ": cloud ids must be in [0, n_clouds)");
    SICP_REQUIRE(a != b, SICP_ERR_BAD_ARG, at + " joins a cloud to itself");
    SICP_REQUIRE(used[(size_t)a] && used[(size_t)b], SICP_ERR_BAD_ARG,
                 at + ": both clouds must be referenced by an edge");
    const double* w = rel_w + 6 * (size_t)k;
    int nz = 0;
    for (int q = 0; q < 6; ++q) {
      SICP_REQUIRE(std::isfinite(w[q]) && w[q] >= 0.0, SICP_ERR_BAD_ARG,
                   at + " has a weight that is negative or not finite");
      nz += w[q] != 0.0;
    }
    if (nz == 0 || (j.fixed[(size_t)a] && j.fixed[(size_t)b])) continue;
    const double* h = rel_H + 16 * (size_t)k;
    for (int q = 0; q < 16; ++q)
      SICP_REQUIRE(std::isfinite(h[q]), SICP_ERR_BAD_ARG, "rel_H[" + std::to_string(k) + "] has non-finite entries");
    SICP_REQUIRE(h[12] == 0.0 && h[13] == 0.0 && h[14] == 0.0 && h[15] == 1.0, SICP_ERR_BAD_ARG,
                 "rel_H[" + std::to_string(k) + "] does not have the bottom row (0, 0, 0, 1)");
    for (int p = 0; p < 3; ++p)
      for (int q = 0; q < 3; ++q) {
        const double d = h[p] * h[q] + h[4 + p] * h[4 + q] + h[8 + p] * h[8 + q] - (p == q ? 1.0 : 0.0);
        SICP_REQUIRE(std::fabs(d) <= 1e-6, SICP_ERR_BAD_ARG,
                     "the rotation part of rel_H[" + std::to_string(k) + "] is not orthonormal (to 1e-6)");
      }
    JointRel o{};
    o.Z = rigid_from_H(h);
    for (int q = 0; q < 6; ++q) o.w[q] = w[q];
    o.ca = a;
    o.cb = b;
    o.fa = j.free_of[(size_t)a];
    o.fb = j.free_of[(size_t)b];
    j.rels.push_back(o);
  }
}

// sicp_register_joint: sicp_register_pairs' stages under the linearised rules, edge e = pair
// (fix_id[e], mov_id[e]) starting from T_a^-1 T_b, with joint_loop in place of the per-pair loop.
static void register_joint(Ctx& c, int n_clouds, const double* const* xyz, const int64_t* n, int n_edges,
                           const int32_t* fix_id, const int32_t* mov_id, const int32_t* is_fixed, const double* H0,
                           const double* prior_H, const double* prior_w, int n_rel, const int32_t* rel_a,
                           const int32_t* rel_b, const double* rel_H, const double* rel_w,
                           const sicp_register_params* rp, double* H_out, sicp_pair_result* out,
                           int64_t* n_selected) {
  if (c.batch) c.batch->out_valid = false;
  VariantScope linearised(c, SICP_VARIANT_LINEARIZED);
  check_pairs_params(c, n_edges, xyz && n && fix_id && mov_id && is_fixed && H_out && out, rp);
  SICP_REQUIRE(rp->mov_neighbors == 0, SICP_ERR_BAD_ARG, "the joint registration has no movable-side normals");
  SICP_REQUIRE(n_clouds >= 1, SICP_ERR_BAD_ARG, "n_clouds must be >= 1");
  JointRun j;
  j.n_clouds = n_clouds;
  j.n_edges = n_edges;
  j.fix_id = fix_id;
  j.mov_id = mov_id;
  std::vector<char> used((size_t)n_clouds, 0);
  for (int e = 0; e < n_edges; ++e) {
    SICP_REQUIRE(fix_id[e] >= 0 && fix_id[e] < n_clouds && mov_id[e] >= 0 && mov_id[e] < n_clouds,
                 SICP_ERR_BAD_ARG, "edge " + std::to_string(e) + ": cloud ids must be in [0, n_clouds)");
    SICP_REQUIRE(fix_id[e] != mov_id[e], SICP_ERR_BAD_ARG, "edge " + std::to_string(e) + " is a self edge");
    used[(size_t)fix_id[e]] = used[(size_t)mov_id[e]] = 1;
  }
  if (H0)
    for (long long k = 0; k < 16ll * n_clouds; ++k)
      SICP_REQUIRE(std::isfinite(H0[k]), SICP_ERR_BAD_ARG, "H0 has non-finite entries");
  j.fixed.assign((size_t)n_clouds, 0);
  j.free_of.assign((size_t)n_clouds, -1);
  j.pose.resize((size_t)n_clouds);
  const double I[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  for (int i = 0; i < n_clouds; ++i) {
    j.fixed[(size_t)i] = is_fixed[i] != 0;
    j.pose[(size_t)i] = rigid_from_H(H0 ? H0 + 16 * (size_t)i : I);
    if (used[(size_t)i] && !j.fixed[(size_t)i]) {
      j.free_of[(size_t)i] = (int)j.free_ids.size();
      j.free_ids.push_back(i);
    }
  }
  j.F = (int)j.free_ids.size();
  check_joint_priors(j, prior_H, prior_w);
  check_joint_relative(j, n_rel, rel_a, rel_b, rel_H, rel_w);
  if (c.joint_solver == 1)
    SICP_REQUIRE(j.F >= 1 && j.F <= JOINT_SPARSE_MAX_FREE, SICP_ERR_BAD_ARG,
                 "the edges must reference between 1 and " + std::to_string(JOINT_SPARSE_MAX_FREE) +
                     " free clouds under joint_solver 1 (got " + std::to_string(j.F) + ")");
  else
    SICP_REQUIRE(j.F >= 1 && j.F <= JOINT_MAX_FREE, SICP_ERR_BAD_ARG,
                 "the edges must reference between 1 and 256 free clouds (got " + std::to_string(j.F) + ")");
  const std::vector<char> every((size_t)n_edges, 1);
  check_anchored(j, every, SICP_ERR_BAD_ARG, "a free cloud is in a component of the edge graph without a fixed cloud");
  // the sparse factor's size over every edge, before any upload (joint_loop checks it again over the
  // edges that keep their overlap, whose plan it runs)
  if (c.joint_solver == 1) joint_sparse_plan(j, every);
  j.prior.resize((size_t)n_edges);
  for (int e = 0; e < n_edges; ++e)
    j.prior[(size_t)e] = rigid_compose(rigid_inverse(j.pose[(size_t)fix_id[e]]), j.pose[(size_t)mov_id[e]]);
  register_pairs(c, n_clouds, xyz, n, n_edges, fix_id, mov_id, rp, nullptr, out, n_selected, &j);
  for (int i = 0; i < n_clouds; ++i) {
    double* dst = H_out + 16 * (size_t)i;
    if (j.free_of[(size_t)i] >= 0) H_from_rigid(j.pose[(size_t)i], dst);
    else std::memcpy(dst, H0 ? H0 + 16 * (size_t)i : I, sizeof(double) * 16);
  }
}

// sicp_register_batch: sicp_register_pairs over its 2 n_pairs clouds, pair i = (cloud 2i, cloud
// 2i + 1).  Its own checks come first, in the order and with the messages they have always had.
static void batch_to_pairs(Ctx& c, int n_pairs, const double* const* fix_xyz, const int64_t* n_fix,
                           const double* const* mov_xyz, const int64_t* n_mov, const sicp_register_params* rp,
                           const double* observed, sicp_pair_result* out, int64_t* n_selected) {
  if (c.batch) c.batch->out_valid = false;
  check_pairs_params(c, n_pairs, fix_xyz && n_fix && mov_xyz && n_mov && out, rp);
  std::vector<const double*> xyz(2 * (size_t)n_pairs);
  std::vector<int64_t> n(2 * (size_t)n_pairs);
  std::vector<int32_t> fix_id((size_t)n_pairs), mov_id((size_t)n_pairs);
  for (int i = 0; i < n_pairs; ++i) {
    SICP_REQUIRE(fix_xyz[i] && mov_xyz[i], SICP_ERR_BAD_ARG, "cloud pointer is NULL");
    SICP_REQUIRE(n_fix[i] >= rp->neighbors && n_mov[i] >= 1, SICP_ERR_BAD_ARG,
                 "every fixed cloud needs at least `neighbors` points, every movable cloud one");
    check_movable(*rp, i, n_mov[i]);
    xyz[2 * (size_t)i] = fix_xyz[i];
    xyz[2 * (size_t)i + 1] = mov_xyz[i];
    n[2 * (size_t)i] = n_fix[i];
    n[2 * (size_t)i + 1] = n_mov[i];
    fix_id[(size_t)i] = 2 * i;
    mov_id[(size_t)i] = 2 * i + 1;
  }
  register_pairs(c, 2 * n_pairs, xyz.data(), n.data(), n_pairs, fix_id.data(), mov_id.data(), rp, observed, out,
                 n_selected);
}

// The clouds of sicp_map_insert and sicp_map_distances, checked before any device work: their
// offsets in the concatenation, n_clouds + 1 of them, the count saturated at 2^40 (both callers'
// limits are below 2^32).
static std::vector<long long> check_clouds(int n_clouds, const double* const* xyz, const int64_t* n, const double* H) {
  SICP_REQUIRE(n_clouds >= 1, SICP_ERR_BAD_ARG, "n_clouds must be >= 1");
  SICP_REQUIRE(xyz && n, SICP_ERR_BAD_ARG, "NULL argument");
  constexpr long long kMany = 1ll << 40;
  std::vector<long long> off((size_t)n_clouds + 1, 0);
  for (int i = 0; i < n_clouds; ++i) {
    SICP_REQUIRE(n[i] >= 0, SICP_ERR_BAD_ARG, "cloud " + std::to_string(i) + " has a negative point count");
    SICP_REQUIRE(n[i] == 0 || xyz[i], SICP_ERR_BAD_ARG, "cloud pointer is NULL");
    off[(size_t)i + 1] = std::min<long long>(off[(size_t)i] + std::min<long long>(n[i], kMany), kMany);
  }
  if (H)
    for (int j = 0; j < 16 * n_clouds; ++j)
      SICP_REQUIRE(std::isfinite(H[j]), SICP_ERR_BAD_ARG, "H has non-finite entries");
  return off;
}

// The clouds uploaded into MapStore::ins_xyz (off from check_clouds, nt = off[n_clouds] > 0 points)
// and moved there by k_insert_stage, which also writes the finite flags into Ctx::compact.flag
// (its scan is reserved too: the compactions of both callers take nt flags).
static void stage_clouds(Ctx& c, MapStore& m, int n_clouds, const double* const* xyz, const int64_t* n,
                         const double* H, const std::vector<long long>& off) {
  cudaStream_t st = c.stream;
  const long long nt = off[(size_t)n_clouds];
  m.ins_xyz.reserve(3 * (size_t)nt);
  for (int i = 0; i < n_clouds; ++i)
    if (n[i] > 0) upload_to_device(c, m.ins_xyz.p + 3 * off[(size_t)i], xyz[i], sizeof(double) * 3 * (size_t)n[i]);
  const std::vector<uint32_t> off32(off.begin(), off.end());
  m.ins_off.reserve((size_t)n_clouds + 1);
  SICP_CUDA(cudaMemcpyAsync(m.ins_off.p, off32.data(), sizeof(uint32_t) * off32.size(), cudaMemcpyHostToDevice, st));
  const Rigid* T = nullptr;
  if (H) {
    std::vector<Rigid> hT((size_t)n_clouds);
    for (int i = 0; i < n_clouds; ++i) hT[(size_t)i] = rigid_from_H(H + 16 * (size_t)i);  // as sicp_transform
    m.ins_T.reserve((size_t)n_clouds);
    SICP_CUDA(cudaMemcpyAsync(m.ins_T.p, hT.data(), sizeof(Rigid) * hT.size(), cudaMemcpyHostToDevice, st));
    T = m.ins_T.p;
  }
  c.compact.flag.reserve((size_t)nt);
  c.compact.scan.reserve((size_t)nt + 1);
  k_insert_stage<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(m.ins_xyz.p, nt, m.ins_off.p, n_clouds, T,
                                                               c.compact.flag.p);
  c.tm.kernel_launches += 1;
}

// The last step of every call that replaces the map (insert, crop, thin): the new map's n_new
// points are in MapStore::xyz_next; they get their grid from set_map's grid_build call, and only
// then are the two swapped in, so a failure leaves the map as it was, and the new map is the one
// set_map would make of the same points.  The old map's buffers are released after the swap: one
// map stays resident between calls.
static void swap_in_next_map(Ctx& c, MapStore& m, long long n_new) {
  std::vector<GridView> views;
  std::vector<double> centres;
  grid_build(c, m.grid_next, {HostCloud{m.xyz_next.p, n_new, 0}}, batch_policy(c), views, centres);  // as set_map
  SICP_CUDA(cudaStreamSynchronize(c.stream));
  m.xyz.swap(m.xyz_next);
  m.grid.swap(m.grid_next);
  m.view = views[0];
  m.n = n_new;
  m.xyz_next.release();
  m.grid_next.release();
}

// sicp_map_insert.  The clouds are staged into one buffer and moved there; their finite points
// are compacted in order and gridded as one cloud; k_map_insert_flags flags the points to add (a
// voxel key no map point has, first of its key among the new points); one scan + an ordered
// scatter append them after the map's points in a fresh buffer, which gets its grid from set_map's
// grid_build call.  Only then are the two swapped in, so a failure leaves the map as it was,
// and the grown map is the one set_map would make of the same points.  Peak device memory: the
// old and the new map (coordinates and grid) plus the staged clouds.
static void map_insert(Ctx& c, int n_clouds, const double* const* xyz, const int64_t* n, const double* H,
                       double voxel, int64_t* n_added) {
  if (c.batch) c.batch->out_valid = false;
  SICP_REQUIRE(std::isfinite(voxel) && voxel > 0, SICP_ERR_BAD_ARG, "voxel_size must be finite and > 0");
  const std::vector<long long> off = check_clouds(n_clouds, xyz, n, H);
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  MapStore& m = *c.map;
  const long long nt = off[(size_t)n_clouds];
  SICP_REQUIRE(m.n + nt < (1ll << 32), SICP_ERR_BAD_ARG,
               "n_map + the points of the clouds must be below 2^32 (the limit of sicp_set_map)");
  if (n_added) std::fill(n_added, n_added + n_clouds, 0);
  if (nt == 0) return;
  cudaStream_t st = c.stream;

  // ---- stage and move the clouds, flag and compact their finite points
  stage_clouds(c, m, n_clouds, xyz, n, H, off);
  CompactScratch& s = c.compact;
  scan_u32(c, s.flag.p, nt, s.scan.p, s.sums);
  const long long n_fin = compact_bounds(c, s.scan.p, {nt})[0];
  if (n_fin == 0) return;  // nothing finite, nothing added
  m.fin_xyz.reserve(3 * (size_t)n_fin);
  m.fin_idx.reserve((size_t)n_fin);
  compact_scatter(c, s.flag.p, nt, s.scan.p, m.fin_idx.p, m.ins_xyz.p, nullptr, m.fin_xyz.p);

  // ---- the points to add, and how many per cloud (one read-back)
  std::vector<GridView> views;
  std::vector<double> centres;
  grid_build(c, m.gnew, {HostCloud{m.fin_xyz.p, n_fin, 0}}, batch_policy(c), views, centres);
  SICP_CUDA(cudaMemsetAsync(s.flag.p, 0, sizeof(uint32_t) * (size_t)nt, st));
  map_insert_flags_launch(c, m.view, views[0], m.fin_xyz.p, m.fin_idx.p, n_fin, voxel, s.flag.p);
  scan_u32(c, s.flag.p, nt, s.scan.p, s.sums);
  const uint32_t* bounds = compact_bounds(c, s.scan.p, off);
  const long long added = bounds[n_clouds];
  if (added > 0) {
    // ---- the grown map in fresh buffers, then swapped in (DevBuf::reserve drops what it held)
    const long long n_new = m.n + added;
    m.xyz_next.reserve(3 * (size_t)n_new);
    SICP_CUDA(cudaMemcpyAsync(m.xyz_next.p, m.xyz.p, sizeof(double) * 3 * (size_t)m.n, cudaMemcpyDeviceToDevice, st));
    compact_scatter(c, s.flag.p, nt, s.scan.p, nullptr, m.ins_xyz.p, nullptr, m.xyz_next.p + 3 * m.n);
    swap_in_next_map(c, m, n_new);
  }
  if (n_added)
    for (int i = 0; i < n_clouds; ++i) n_added[i] = (int64_t)bounds[i + 1] - (int64_t)bounds[i];
}

static void get_map(Ctx& c, double* xyz, int64_t cap, int64_t* n) {
  SICP_REQUIRE(n, SICP_ERR_BAD_ARG, "n is NULL");
  SICP_REQUIRE(cap >= 0, SICP_ERR_BAD_ARG, "cap must be >= 0");
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  const MapStore& m = *c.map;
  *n = m.n;
  if (xyz && cap > 0) {
    copy_any(c, xyz, m.xyz.p, sizeof(double) * 3 * (size_t)std::min<long long>(m.n, cap));
    SICP_CUDA(cudaStreamSynchronize(c.stream));
  }
}

// The end of sicp_map_crop and sicp_map_thin: the map points whose keep flag (Ctx::compact.flag,
// one per map point) is set become the new map, in map order.  One scan and one read-back of the
// kept count; when every point is kept nothing else happens (the map and its grid stay as they
// are); otherwise the kept points are compacted into xyz_next and swap_in_next_map makes them the
// map.  A map is never empty: keeping no point is SICP_ERR_NO_OVERLAP with the map unchanged.
// Returns the points removed.
static long long keep_flagged(Ctx& c, MapStore& m) {
  CompactScratch& s = c.compact;
  const long long n = m.n;
  scan_u32(c, s.flag.p, n, s.scan.p, s.sums);
  const long long kept = compact_bounds(c, s.scan.p, {n})[0];
  SICP_REQUIRE(kept > 0, SICP_ERR_NO_OVERLAP, "no map point would be kept (a map is never empty): the map is unchanged");
  if (kept == n) return 0;
  m.xyz_next.reserve(3 * (size_t)kept);
  compact_scatter(c, s.flag.p, n, s.scan.p, nullptr, m.xyz.p, nullptr, m.xyz_next.p);
  swap_in_next_map(c, m, kept);
  return n - kept;
}

// sicp_map_crop: keep the map points within radius of at least one centre (k_map_crop_flags).
static void map_crop(Ctx& c, int n_centers, const double* centers, double radius, int64_t* n_removed) {
  if (c.batch) c.batch->out_valid = false;
  SICP_REQUIRE(n_centers >= 1, SICP_ERR_BAD_ARG, "n_centers must be >= 1");
  SICP_REQUIRE(centers, SICP_ERR_BAD_ARG, "centers is NULL");
  for (long long i = 0; i < 3ll * n_centers; ++i)
    SICP_REQUIRE(std::isfinite(centers[i]), SICP_ERR_BAD_ARG, "centers has non-finite coordinates");
  SICP_REQUIRE(std::isfinite(radius) && radius > 0, SICP_ERR_BAD_ARG, "radius must be finite and > 0");
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  MapStore& m = *c.map;
  if (n_removed) *n_removed = 0;
  cudaStream_t st = c.stream;
  m.crop_c.reserve(3 * (size_t)n_centers);
  SICP_CUDA(cudaMemcpyAsync(m.crop_c.p, centers, sizeof(double) * 3 * (size_t)n_centers, cudaMemcpyHostToDevice, st));
  c.compact.flag.reserve((size_t)m.n);
  c.compact.scan.reserve((size_t)m.n + 1);
  // r2 = fl(radius^2), as sicp_select_in_range and sicp_map_distances compute it
  k_map_crop_flags<<<(unsigned)((m.n + 255) / 256), 256, 0, st>>>(m.xyz.p, m.n, m.crop_c.p, n_centers,
                                                                  radius * radius, c.compact.flag.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
  const long long removed = keep_flagged(c, m);
  if (n_removed) *n_removed = removed;
}

// sicp_map_thin: keep the first map point of every voxel key (k_map_thin_flags, nn.cu).
static void map_thin(Ctx& c, double voxel, int64_t* n_removed) {
  if (c.batch) c.batch->out_valid = false;
  SICP_REQUIRE(std::isfinite(voxel) && voxel > 0, SICP_ERR_BAD_ARG, "voxel_size must be finite and > 0");
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  MapStore& m = *c.map;
  if (n_removed) *n_removed = 0;
  c.compact.flag.reserve((size_t)m.n);
  c.compact.scan.reserve((size_t)m.n + 1);
  map_thin_flags_launch(c, m.view, m.xyz.p, m.n, voxel, c.compact.flag.p);
  const long long removed = keep_flagged(c, m);
  if (n_removed) *n_removed = removed;
}

// sicp_map_carve: remove the map points that at least min_passes rays of the clouds pass.  The
// clouds are staged and moved as sicp_map_distances' are; k_map_carve (nn.cu) walks every ray
// through the map grid and counts the passes per map point; they go to the caller, and the map
// points with fewer than min_passes are kept through keep_flagged, as by a crop.
static void map_carve(Ctx& c, int n_clouds, const double* const* xyz, const int64_t* n, const double* H,
                      const double* origins, double radius, double margin, int32_t min_passes, uint32_t* passes,
                      int64_t* n_removed) {
  if (c.batch) c.batch->out_valid = false;
  const std::vector<long long> off = check_clouds(n_clouds, xyz, n, H);
  SICP_REQUIRE(origins || H, SICP_ERR_BAD_ARG, "origins and H are both NULL: a ray needs its origin");
  std::vector<double> o(3 * (size_t)n_clouds);
  for (int i = 0; i < n_clouds; ++i)
    for (int a = 0; a < 3; ++a)  // H's translation column, taken as it is
      o[3 * (size_t)i + a] = origins ? origins[3 * (size_t)i + a] : H[16 * (size_t)i + 4 * a + 3];
  for (double v : o) SICP_REQUIRE(std::isfinite(v), SICP_ERR_BAD_ARG, "origins has non-finite coordinates");
  SICP_REQUIRE(std::isfinite(radius) && radius > 0, SICP_ERR_BAD_ARG, "radius must be finite and > 0");
  SICP_REQUIRE(std::isfinite(margin) && margin >= 0, SICP_ERR_BAD_ARG, "margin must be finite and >= 0");
  SICP_REQUIRE(min_passes >= 1, SICP_ERR_BAD_ARG, "min_passes must be >= 1");
  const long long nt = off[(size_t)n_clouds];
  SICP_REQUIRE(nt < (1ll << 32), SICP_ERR_BAD_ARG, "the points of the clouds must be below 2^32 (32-bit offsets)");
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  MapStore& m = *c.map;
  if (n_removed) *n_removed = 0;
  cudaStream_t st = c.stream;
  // the staging's finite flags, then the keep flags of the map, share the compaction's scratch
  c.compact.flag.reserve((size_t)std::max(nt, m.n));
  c.compact.scan.reserve((size_t)std::max(nt, m.n) + 1);
  m.carve_passes.reserve((size_t)m.n);
  SICP_CUDA(cudaMemsetAsync(m.carve_passes.p, 0, sizeof(uint32_t) * (size_t)m.n, st));
  if (nt > 0) {
    stage_clouds(c, m, n_clouds, xyz, n, H, off);
    m.carve_o.reserve(o.size());
    SICP_CUDA(cudaMemcpyAsync(m.carve_o.p, o.data(), sizeof(double) * o.size(), cudaMemcpyHostToDevice, st));
    // r2 = fl(radius^2), as sicp_map_crop computes it
    map_carve_launch(c, m.view, m.ins_xyz.p, nt, m.ins_off.p, n_clouds, m.carve_o.p, radius, radius * radius, margin,
                     m.carve_passes.p);
  }
  if (passes) copy_any(c, passes, m.carve_passes.p, sizeof(uint32_t) * (size_t)m.n);
  k_carve_keep<<<(unsigned)((m.n + 255) / 256), 256, 0, st>>>(m.carve_passes.p, m.n, (uint32_t)min_passes,
                                                              c.compact.flag.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
  // keep_flagged reads its count back (a stream synchronise), so passes is complete when it
  // returns, also when it throws SICP_ERR_NO_OVERLAP
  const long long removed = keep_flagged(c, m);
  if (n_removed) *n_removed = removed;
}

// sicp_map_distances.  The clouds are staged and moved as sicp_map_insert's are; k_map_nearest
// finds each point's nearest map point within the bound (nn.cu); one scan over the within flags
// gives the per-cloud counts (one read-back) and the places of the within points, whose matched
// map points are gathered and get the normal estimate of sicp_estimate_normals in the map grid;
// k_dist_plane then writes the plane distances.  Every output is written to MapStore buffers and
// copied per cloud to the caller's arrays.  Nothing else of the context changes: the map, the
// batch outputs and the one-pair state stay as they are.
static void map_distances(Ctx& c, int n_clouds, const double* const* xyz, const int64_t* n, const double* H,
                          double max_distance, int k, int64_t* const* idx, double* const* dist2,
                          double* const* plane_dist, float* const* planarity, int64_t* n_within) {
  SICP_REQUIRE(std::isfinite(max_distance) && max_distance > 0, SICP_ERR_BAD_ARG,
               "max_distance must be finite and > 0");
  SICP_REQUIRE(k == 0 || (k >= 2 && k <= 64), SICP_ERR_BAD_ARG,
               "neighbors must be 0 or between 2 and 64 (got " + std::to_string(k) + ")");
  SICP_REQUIRE(k > 0 || (!plane_dist && !planarity), SICP_ERR_BAD_ARG,
               "plane_dist and planarity need the map's normals: neighbors must be > 0");
  const std::vector<long long> off = check_clouds(n_clouds, xyz, n, H);
  SICP_REQUIRE(c.map && c.map->n > 0, SICP_ERR_STATE, "no map: call sicp_set_map first");
  MapStore& m = *c.map;
  SICP_REQUIRE(k <= m.n, SICP_ERR_BAD_ARG, "neighbors exceeds the number of map points");
  const long long nt = off[(size_t)n_clouds];
  SICP_REQUIRE(nt < (1ll << 32), SICP_ERR_BAD_ARG, "the points of the clouds must be below 2^32 (32-bit offsets)");
  if (n_within) std::fill(n_within, n_within + n_clouds, 0);
  if (nt == 0) return;
  cudaStream_t st = c.stream;
  const unsigned blocks = (unsigned)((nt + 255) / 256);

  // ---- nearest map point of every staged point, within flags and their per-cloud counts
  stage_clouds(c, m, n_clouds, xyz, n, H, off);
  CompactScratch& s = c.compact;
  m.dst_idx.reserve((size_t)nt);
  m.dst_d2.reserve((size_t)nt);
  map_nearest_launch(c, m.view, m.ins_xyz.p, nt, max_distance * max_distance, m.dst_idx.p, m.dst_d2.p, s.flag.p);
  scan_u32(c, s.flag.p, nt, s.scan.p, s.sums);
  const uint32_t* bounds = compact_bounds(c, s.scan.p, off);
  const long long n_in = bounds[n_clouds];

  // ---- normals of the matched map points and the plane distances
  if (k > 0) {
    m.dst_plane.reserve((size_t)nt);
    m.dst_pl.reserve((size_t)nt);
    if (n_in > 0) {
      m.dst_mxyz.reserve(3 * (size_t)n_in);
      m.dst_nrm.reserve((size_t)n_in);
      compact_scatter(c, s.flag.p, nt, s.scan.p, nullptr, m.xyz.p, m.dst_idx.p, m.dst_mxyz.p);
      map_normals_launch(c, m.view, m.dst_mxyz.p, n_in, k, m.dst_nrm.p, m.dst_pos);
    }
    k_dist_plane<<<blocks, 256, 0, st>>>(m.ins_xyz.p, nt, s.flag.p, s.scan.p, m.dst_mxyz.p, m.dst_nrm.p,
                                         m.dst_plane.p, m.dst_pl.p);
    SICP_CUDA(cudaGetLastError());
    c.tm.kernel_launches += 1;
  }

  // ---- each requested cloud's slice to the caller (any memory kind)
  for (int i = 0; i < n_clouds; ++i) {
    const size_t s = (size_t)off[(size_t)i], cnt = (size_t)n[i];
    if (idx && idx[i]) copy_any(c, idx[i], m.dst_idx.p + s, sizeof(long long) * cnt);
    if (dist2 && dist2[i]) copy_any(c, dist2[i], m.dst_d2.p + s, sizeof(double) * cnt);
    if (plane_dist && plane_dist[i]) copy_any(c, plane_dist[i], m.dst_plane.p + s, sizeof(double) * cnt);
    if (planarity && planarity[i]) copy_any(c, planarity[i], m.dst_pl.p + s, sizeof(float) * cnt);
  }
  SICP_CUDA(cudaStreamSynchronize(st));
  if (n_within)
    for (int i = 0; i < n_clouds; ++i) n_within[i] = (int64_t)bounds[i + 1] - (int64_t)bounds[i];
}

// sicp_overlap_graph (DESIGN.md §6.10).  Every non-empty cloud is staged once and gridded once
// under the batch cell policy, as sicp_register_pairs does it.  Two culls on the host leave the
// directions whose count can be nonzero:
//  - pair cull: the world box of each cloud's grid box under its pose, grown by half the bound
//    (plus the rounding margin of map_cull_box); a sort-and-sweep along the axis with the widest
//    spread of box centres gives the pairs whose grown boxes meet.  Two clouds whose grown boxes
//    are disjoint hold no points within r of each other: both counts are 0.
//  - direction cull: map_cull_box(a's grid, b's grid, T_ab, r) bounds the points of a that can
//    pass; rows == 0 means count_ab = 0 with no search.
// k_overlap_count (nn.cu) then runs the overlap filter's search for the sampled points of a in the
// box, 65535 directions per launch, and one read-back brings the two counters of every candidate.
// With poses that are not rigid to the last bits (the call accepts |R^T R - I| <= 1e-6), the
// inverse of T_ab is off by up to about 3 eps times the coordinates' magnitude M; both culls grow
// by 16 eps (M + r) more for that.
static void overlap_graph(Ctx& c, int n_clouds, const double* const* xyz, const int64_t* n, const double* H,
                          double r, int64_t stride, int32_t* pair_a, int32_t* pair_b, int64_t* count_ab,
                          int64_t* count_ba, int64_t cap, int64_t* n_pairs) {
  SICP_REQUIRE(n_pairs, SICP_ERR_BAD_ARG, "n_pairs is NULL");
  const std::vector<long long> off = check_clouds(n_clouds, xyz, n, H);
  double eps = 0.0;  // the largest entry of |R^T R - I| over the poses
  for (int i = 0; H && i < n_clouds; ++i) {
    const double* h = H + 16 * (size_t)i;
    SICP_REQUIRE(h[12] == 0.0 && h[13] == 0.0 && h[14] == 0.0 && h[15] == 1.0, SICP_ERR_BAD_ARG,
                 "H[" + std::to_string(i) + "] does not have the bottom row (0, 0, 0, 1)");
    for (int p = 0; p < 3; ++p)
      for (int q = 0; q < 3; ++q) {
        const double d = h[p] * h[q] + h[4 + p] * h[4 + q] + h[8 + p] * h[8 + q] - (p == q ? 1.0 : 0.0);
        SICP_REQUIRE(std::fabs(d) <= 1e-6, SICP_ERR_BAD_ARG,
                     "the rotation part of H[" + std::to_string(i) + "] is not orthonormal (to 1e-6)");
        eps = std::max(eps, std::fabs(d));
      }
  }
  SICP_REQUIRE(std::isfinite(r) && r > 0, SICP_ERR_BAD_ARG, "max_distance must be finite and > 0");
  SICP_REQUIRE(stride >= 1, SICP_ERR_BAD_ARG, "stride must be >= 1");
  SICP_REQUIRE(cap >= 0, SICP_ERR_BAD_ARG, "cap must be >= 0");
  SICP_REQUIRE(off[(size_t)n_clouds] < (1ll << 32), SICP_ERR_BAD_ARG,
               "the points of the clouds must be below 2^32 (32-bit offsets)");
  *n_pairs = 0;
  c.tm.upload_ms = c.tm.grid_fix_ms = c.tm.overlap_ms = 0;
  std::vector<int> ids;  // the non-empty clouds; k-th grid = cloud ids[k]
  for (int i = 0; i < n_clouds; ++i)
    if (n[i] > 0) ids.push_back(i);
  if (ids.size() < 2) return;
  if (!c.ovl) c.ovl = new OverlapStore();
  OverlapStore& o = *c.ovl;
  cudaStream_t st = c.stream;
  const int K = (int)ids.size();

  // ---- every non-empty cloud once, and its grid
  o.xyz.reserve(3 * (size_t)off[(size_t)n_clouds]);
  {
    StageTimer t(c, &c.tm.upload_ms);
    for (int i : ids) upload_to_device(c, o.xyz.p + 3 * off[(size_t)i], xyz[i], sizeof(double) * 3 * (size_t)n[i]);
    t.stop();
  }
  std::vector<HostCloud> clouds;
  for (int i : ids) clouds.push_back(HostCloud{o.xyz.p + 3 * off[(size_t)i], n[i], off[(size_t)i]});
  std::vector<GridView> views;
  std::vector<double> centres;
  {
    StageTimer t(c, &c.tm.grid_fix_ms);
    grid_build(c, o.grid, clouds, batch_policy(c), views, centres);
    t.stop();
  }
  StageTimer timer(c, &c.tm.overlap_ms);

  // ---- pair cull: world boxes, grown, swept along one axis
  Rigid I;
  std::memset(&I, 0, sizeof(I));
  I.r[0] = I.r[4] = I.r[8] = 1.0;
  std::vector<Rigid> T((size_t)K, I);
  if (H)
    for (int k = 0; k < K; ++k) T[(size_t)k] = rigid_from_H(H + 16 * (size_t)ids[(size_t)k]);
  std::vector<double> wlo(3 * (size_t)K, kInf), whi(3 * (size_t)K, -kInf);
  double mag = 0.0;
  for (int k = 0; k < K; ++k) {
    const GridView& g = views[(size_t)k];
    const double lo[3] = {g.ox, g.oy, g.oz}, hi[3] = {g.ox + g.nx * g.h, g.oy + g.ny * g.h, g.oz + g.nz * g.h};
    for (int a = 0; a < 3; ++a)
      mag = std::max(mag, std::max(std::max(std::fabs(lo[a]), std::fabs(hi[a])), std::fabs(T[(size_t)k].t[a])));
    for (int q = 0; q < 8; ++q) {
      double v[3];
      rigid_apply(T[(size_t)k], (q & 1) ? hi[0] : lo[0], (q & 2) ? hi[1] : lo[1], (q & 4) ? hi[2] : lo[2], v[0], v[1],
                  v[2]);
      for (int a = 0; a < 3; ++a) {
        wlo[3 * (size_t)k + a] = std::min(wlo[3 * (size_t)k + a], v[a]);
        whi[3 * (size_t)k + a] = std::max(whi[3 * (size_t)k + a], v[a]);
        mag = std::max(mag, std::fabs(v[a]));
      }
    }
  }
  const double r_cull = r + 16.0 * eps * (mag + r);  // the bound the culls are proven for
  const double half = 0.5 * (r_cull + 1e-12 * (mag + r_cull));
  for (double& v : wlo) v -= half;
  for (double& v : whi) v += half;
  int ax = 0;
  double best_spread = -1.0;
  for (int a = 0; a < 3; ++a) {
    double cmin = kInf, cmax = -kInf;
    for (int k = 0; k < K; ++k) {
      const double cen = 0.5 * (wlo[3 * (size_t)k + a] + whi[3 * (size_t)k + a]);
      cmin = std::min(cmin, cen);
      cmax = std::max(cmax, cen);
    }
    if (cmax - cmin > best_spread) {
      best_spread = cmax - cmin;
      ax = a;
    }
  }
  std::vector<int> order((size_t)K);
  for (int k = 0; k < K; ++k) order[(size_t)k] = k;
  std::sort(order.begin(), order.end(), [&](int p, int q) { return wlo[3 * (size_t)p + ax] < wlo[3 * (size_t)q + ax]; });
  std::vector<std::pair<int, int>> cand;  // (k, l), k < l: grid slots, ascending like the cloud ids
  std::vector<int> active;
  for (int k : order) {
    size_t keep = 0;
    for (int l : active) {
      if (whi[3 * (size_t)l + ax] < wlo[3 * (size_t)k + ax]) continue;  // ends before every later box starts
      active[keep++] = l;
      bool meet = true;
      for (int a = 0; a < 3; ++a)
        meet = meet && wlo[3 * (size_t)k + a] <= whi[3 * (size_t)l + a] && wlo[3 * (size_t)l + a] <= whi[3 * (size_t)k + a];
      if (meet) cand.emplace_back(std::min(k, l), std::max(k, l));
    }
    active.resize(keep);
    active.push_back(k);
  }
  std::sort(cand.begin(), cand.end());
  const long long n_cand = (long long)cand.size();

  // ---- direction cull and count, 65535 directions per launch
  o.views.reserve(K);
  SICP_CUDA(cudaMemcpyAsync(o.views.p, views.data(), sizeof(GridView) * (size_t)K, cudaMemcpyHostToDevice, st));
  o.counts.reserve(std::max<long long>(2 * n_cand, 1));
  SICP_CUDA(cudaMemsetAsync(o.counts.p, 0, sizeof(uint32_t) * (size_t)std::max<long long>(2 * n_cand, 1), st));
  constexpr int kChunk = 65535;  // blockIdx.y is the direction
  const size_t ds = sizeof(DevState) * kChunk;
  o.dirs.reserve(ds + sizeof(OverlapDir) * kChunk);
  std::vector<DevState> hs;
  std::vector<OverlapDir> hd;
  long long max_rows = 0, n_q = 0;
  auto flush = [&]() {
    if (hd.empty()) return;
    const int nd = (int)hd.size();
    // the previous launch has read its directions before this copy lands (stream order); a
    // pageable source is staged by the runtime before the call returns
    SICP_CUDA(cudaMemcpyAsync(o.dirs.p, hs.data(), sizeof(DevState) * (size_t)nd, cudaMemcpyHostToDevice, st));
    SICP_CUDA(cudaMemcpyAsync(o.dirs.p + ds, hd.data(), sizeof(OverlapDir) * (size_t)nd, cudaMemcpyHostToDevice, st));
    // r2 as sicp_select_in_range computes it
    overlap_count_launch(c, o.views.p, reinterpret_cast<const DevState*>(o.dirs.p),
                         reinterpret_cast<const OverlapDir*>(o.dirs.p + ds), nd, max_rows, stride, r * r, o.counts.p,
                         n_q);
    hs.clear();
    hd.clear();
    max_rows = n_q = 0;
  };
  for (long long p = 0; p < n_cand; ++p) {
    const int k = cand[(size_t)p].first, l = cand[(size_t)p].second;
    for (int side = 0; side < 2; ++side) {
      const int a = side ? l : k, b = side ? k : l;
      // T_ab = T_a^-1 T_b as sicp_register_joint forms its priors; exactly I without poses
      const Rigid Tab = H ? rigid_compose(rigid_inverse(T[(size_t)a]), T[(size_t)b]) : I;
      OverlapDir d;
      std::memset(&d, 0, sizeof(d));
      d.cu = map_cull_box(views[(size_t)a], views[(size_t)b], Tab, r_cull);
      if (d.cu.rows == 0) continue;
      d.a = a;
      d.b = b;
      d.slot = (int)(2 * p + side);
      DevState s;
      std::memset(&s, 0, sizeof(s));
      s.T = Tab;
      s.Tinv = rigid_inverse(Tab);
      hs.push_back(s);
      hd.push_back(d);
      max_rows = std::max(max_rows, d.cu.rows);
      n_q += (long long)(d.cu.rows * (d.cu.c1[0] - d.cu.c0[0] + 1) * c.grid_target_occ) / stride;
      if ((int)hd.size() == kChunk) flush();
    }
  }
  flush();

  // ---- one read-back: the rows with a nonzero total, in candidate order (ascending (a, b))
  pinned_reserve(o.counts_host, o.counts_cap, (size_t)std::max<long long>(2 * n_cand, 1));
  SICP_CUDA(cudaMemcpyAsync(o.counts_host, o.counts.p, sizeof(uint32_t) * 2 * (size_t)n_cand, cudaMemcpyDeviceToHost, st));
  SICP_CUDA(cudaStreamSynchronize(st));
  timer.stop();
  long long total = 0;
  for (long long p = 0; p < n_cand; ++p) {
    const uint32_t cab = o.counts_host[2 * p], cba = o.counts_host[2 * p + 1];
    if (cab == 0 && cba == 0) continue;
    if (total < cap) {
      if (pair_a) pair_a[total] = ids[(size_t)cand[(size_t)p].first];
      if (pair_b) pair_b[total] = ids[(size_t)cand[(size_t)p].second];
      if (count_ab) count_ab[total] = cab;
      if (count_ba) count_ba[total] = cba;
    }
    ++total;
  }
  *n_pairs = total;
}

}  // namespace sicp

using namespace sicp;

extern "C" int32_t sicp_register_batch(sicp_ctx* ctx, int32_t n_pairs, const double* const* fix_xyz,
                                       const int64_t* n_fix, const double* const* mov_xyz,
                                       const int64_t* n_mov, const sicp_register_params* p,
                                       const double* observed, sicp_pair_result* out, int64_t* n_selected) {
  API_BEGIN(ctx)
  batch_to_pairs(c, n_pairs, fix_xyz, n_fix, mov_xyz, n_mov, p, observed, out, n_selected);
  API_END
}

extern "C" int32_t sicp_set_map(sicp_ctx* ctx, const double* map_xyz, int64_t n_map) {
  API_BEGIN(ctx)
  set_map(c, map_xyz, n_map);
  API_END
}

extern "C" int32_t sicp_register_to_map(sicp_ctx* ctx, int32_t n_scans, const double* const* mov_xyz,
                                        const int64_t* n_mov, const sicp_register_params* p,
                                        const double* observed, sicp_pair_result* out, int64_t* n_selected) {
  API_BEGIN(ctx)
  register_to_map(c, n_scans, mov_xyz, n_mov, p, observed, out, n_selected);
  API_END
}

extern "C" int32_t sicp_register_pairs(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz, const int64_t* n,
                                       int32_t n_pairs, const int32_t* fix_id, const int32_t* mov_id,
                                       const sicp_register_params* p, const double* observed, sicp_pair_result* out,
                                       int64_t* n_selected) {
  API_BEGIN(ctx)
  register_pairs(c, n_clouds, xyz, n, n_pairs, fix_id, mov_id, p, observed, out, n_selected);
  API_END
}

extern "C" int32_t sicp_register_joint_relative(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz,
                                                const int64_t* n, int32_t n_edges, const int32_t* fix_id,
                                                const int32_t* mov_id, const int32_t* is_fixed, const double* H0,
                                                const double* prior_H, const double* prior_w, int32_t n_rel,
                                                const int32_t* rel_a, const int32_t* rel_b, const double* rel_H,
                                                const double* rel_w, const sicp_register_params* p, double* H_out,
                                                sicp_pair_result* out, int64_t* n_selected) {
  API_BEGIN(ctx)
  register_joint(c, n_clouds, xyz, n, n_edges, fix_id, mov_id, is_fixed, H0, prior_H, prior_w, n_rel, rel_a, rel_b,
                 rel_H, rel_w, p, H_out, out, n_selected);
  API_END
}

extern "C" int32_t sicp_register_joint_priors(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz,
                                              const int64_t* n, int32_t n_edges, const int32_t* fix_id,
                                              const int32_t* mov_id, const int32_t* is_fixed, const double* H0,
                                              const double* prior_H, const double* prior_w,
                                              const sicp_register_params* p, double* H_out, sicp_pair_result* out,
                                              int64_t* n_selected) {
  return sicp_register_joint_relative(ctx, n_clouds, xyz, n, n_edges, fix_id, mov_id, is_fixed, H0, prior_H, prior_w, 0,
                                      nullptr, nullptr, nullptr, nullptr, p, H_out, out, n_selected);
}

extern "C" int32_t sicp_register_joint(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz, const int64_t* n,
                                       int32_t n_edges, const int32_t* fix_id, const int32_t* mov_id,
                                       const int32_t* is_fixed, const double* H0, const sicp_register_params* p,
                                       double* H_out, sicp_pair_result* out, int64_t* n_selected) {
  return sicp_register_joint_priors(ctx, n_clouds, xyz, n, n_edges, fix_id, mov_id, is_fixed, H0, nullptr, nullptr,
                                    p, H_out, out, n_selected);
}

extern "C" int32_t sicp_map_insert(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz, const int64_t* n,
                                   const double* H, double voxel_size, int64_t* n_added) {
  API_BEGIN(ctx)
  map_insert(c, n_clouds, xyz, n, H, voxel_size, n_added);
  API_END
}

extern "C" int32_t sicp_get_map(sicp_ctx* ctx, double* xyz, int64_t cap, int64_t* n) {
  API_BEGIN(ctx)
  get_map(c, xyz, cap, n);
  API_END
}

extern "C" int32_t sicp_map_crop(sicp_ctx* ctx, int32_t n_centers, const double* centers, double radius,
                                 int64_t* n_removed) {
  API_BEGIN(ctx)
  map_crop(c, n_centers, centers, radius, n_removed);
  API_END
}

extern "C" int32_t sicp_map_thin(sicp_ctx* ctx, double voxel_size, int64_t* n_removed) {
  API_BEGIN(ctx)
  map_thin(c, voxel_size, n_removed);
  API_END
}

extern "C" int32_t sicp_map_carve(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz, const int64_t* n,
                                  const double* H, const double* origins, double radius, double margin,
                                  int32_t min_passes, uint32_t* passes, int64_t* n_removed) {
  API_BEGIN(ctx)
  map_carve(c, n_clouds, xyz, n, H, origins, radius, margin, min_passes, passes, n_removed);
  API_END
}

extern "C" int32_t sicp_map_distances(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz, const int64_t* n,
                                      const double* H, double max_distance, int32_t neighbors, int64_t* const* idx,
                                      double* const* dist2, double* const* plane_dist, float* const* planarity,
                                      int64_t* n_within) {
  API_BEGIN(ctx)
  map_distances(c, n_clouds, xyz, n, H, max_distance, neighbors, idx, dist2, plane_dist, planarity, n_within);
  API_END
}

extern "C" int32_t sicp_overlap_graph(sicp_ctx* ctx, int32_t n_clouds, const double* const* xyz, const int64_t* n,
                                      const double* H, double max_distance, int64_t stride, int32_t* pair_a,
                                      int32_t* pair_b, int64_t* count_ab, int64_t* count_ba, int64_t cap,
                                      int64_t* n_pairs) {
  API_BEGIN(ctx)
  overlap_graph(c, n_clouds, xyz, n, H, max_distance, stride, pair_a, pair_b, count_ab, count_ba, cap, n_pairs);
  API_END
}

extern "C" int32_t sicp_get_batch_outputs(sicp_ctx* ctx, int32_t n_pairs, double* const* mov_xyz_out,
                                          double* const* residuals, sicp_iter_record* log, double* T) {
  API_BEGIN(ctx)
  get_batch_outputs(c, n_pairs, mov_xyz_out, residuals, log, T);
  API_END
}

extern "C" int32_t sicp_get_joint_covariances(sicp_ctx* ctx, int32_t n_clouds, double* cloud_cov, int32_t n_edges,
                                              double* edge_cov, double* s0) {
  API_BEGIN(ctx)
  get_joint_covariances(c, n_clouds, cloud_cov, n_edges, edge_cov, s0, false);
  API_END
}

extern "C" int32_t sicp_get_joint_selected_covariances(sicp_ctx* ctx, int32_t n_clouds, double* cloud_cov,
                                                       int32_t n_edges, double* edge_cov, double* s0) {
  API_BEGIN(ctx)
  get_joint_covariances(c, n_clouds, cloud_cov, n_edges, edge_cov, s0, true);
  API_END
}
