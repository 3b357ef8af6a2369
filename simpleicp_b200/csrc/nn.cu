// nn.cu — nearest-neighbour correspondence search (reference: CorrPts.match,
// python/simpleicp/corrpts.py:124-137 + 195-211, and PointCloud.select_in_range,
// python/simpleicp/pointcloud.py:149-171).
//
// The reference transforms the whole movable cloud by H, rebuilds a kd-tree and queries it with
// the selected fixed points.  Rigid maps preserve distances, so here the K queries are moved by
// H^-1 instead and searched in a STATIC structure over the original movable cloud; only the
// matched point is moved by H for the point-to-plane distance.
//
// Two exact engines:
//   grid  : uniform-grid search in float64, 3x3x3 block then shell-by-shell ring expansion until
//           the best distance is provably <= the distance to every unexplored cell.
//   brute : tiled exhaustive search.  float4 tiles of the (centred, float32) cloud are staged
//           into shared memory with 1-D TMA bulk copies (cp.async.bulk + mbarrier, 4-stage ring),
//           lanes split the tile, float32 distances act as a FILTER with a rigorous error margin,
//           every candidate that passes is re-evaluated in float64 from the original
//           coordinates, and the per-lane winners are combined with a warp-shuffle min-reduction.
// Ties are broken towards the lower original index in both.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <type_traits>

#include "ctx.cuh"

namespace sicp {

namespace {

// ------------------------------------------------------------------------------------------
// grid engine
// ------------------------------------------------------------------------------------------
// bpos follows the winner's position in the cell-sorted record array: the record holds the
// original coordinates, so whoever needs the matched point afterwards re-reads that (cache-hot)
// record instead of gathering mov_xyz[bidx] from a cold line.
__device__ __forceinline__ void consider(const Rec& r, uint32_t pos, double qx, double qy, double qz,
                                         double& best, long long& bidx, uint32_t& bpos) {
  const double dx = r.x - qx, dy = r.y - qy, dz = r.z - qz;
  const double d2 = dx * dx + dy * dy + dz * dz;
  if (d2 < best || (d2 == best && r.idx < bidx)) {
    best = d2;
    bidx = r.idx;
    bpos = pos;
  }
}

// Scan the records [s, e).  The search is latency-bound, so four 32-byte records (LDG.E.256
// each) are requested before the first one is used; the tail re-reads the last record instead
// of branching (a duplicate never changes the result: same distance, same index).
__device__ __forceinline__ void scan_range(const Rec* __restrict__ recs, uint32_t s, uint32_t e,
                                           double qx, double qy, double qz, double& best,
                                           long long& bidx, uint32_t& bpos) {
  for (uint32_t i = s; i < e; i += 4) {
    const uint32_t last = e - 1;
    const uint32_t i1 = min(i + 1, last), i2 = min(i + 2, last), i3 = min(i + 3, last);
    const Rec r0 = recs[i];
    const Rec r1 = recs[i1];
    const Rec r2 = recs[i2];
    const Rec r3 = recs[i3];
    consider(r0, i, qx, qy, qz, best, bidx, bpos);
    consider(r1, i1, qx, qy, qz, best, bidx, bpos);
    consider(r2, i2, qx, qy, qz, best, bidx, bpos);
    consider(r3, i3, qx, qy, qz, best, bidx, bpos);
  }
}

// consider() that also keeps sec, the smallest d2 among the visited records other than the
// winner (certificate of the warm-started match, below).  A record at the winner's position is
// not a second point: the warm-start record every lane starts from, and the last record that
// scan_range re-reads as padding, come back with the winner's position.  A record that loses
// (or is displaced) lost to a record earlier in the (d2, idx) order, so sec never holds the winner.
__device__ __forceinline__ void consider_sec(const Rec& r, uint32_t pos, double qx, double qy, double qz,
                                             double& best, long long& bidx, uint32_t& bpos, double& sec) {
  const double dx = r.x - qx, dy = r.y - qy, dz = r.z - qz;
  const double d2 = dx * dx + dy * dy + dz * dz;
  if (pos == bpos) return;
  if (d2 < best || (d2 == best && r.idx < bidx)) {
    sec = fmin(sec, best);
    best = d2;
    bidx = r.idx;
    bpos = pos;
  } else {
    sec = fmin(sec, d2);
  }
}

__device__ __forceinline__ void scan_range_sec(const Rec* __restrict__ recs, uint32_t s, uint32_t e,
                                               double qx, double qy, double qz, double& best,
                                               long long& bidx, uint32_t& bpos, double& sec) {
  for (uint32_t i = s; i < e; i += 4) {
    const uint32_t last = e - 1;
    const uint32_t i1 = min(i + 1, last), i2 = min(i + 2, last), i3 = min(i + 3, last);
    const Rec r0 = recs[i];
    const Rec r1 = recs[i1];
    const Rec r2 = recs[i2];
    const Rec r3 = recs[i3];
    consider_sec(r0, i, qx, qy, qz, best, bidx, bpos, sec);
    consider_sec(r1, i1, qx, qy, qz, best, bidx, bpos, sec);
    consider_sec(r2, i2, qx, qy, qz, best, bidx, bpos, sec);
    consider_sec(r3, i3, qx, qy, qz, best, bidx, bpos, sec);
  }
}

// Returns true when (best, bidx) is proven to be the nearest neighbour.
// cap2 >= 0: the caller only needs to know on which side of cap2 the squared nearest-neighbour
// distance lies (overlap filter, PointCloud.select_in_range): the search may stop as soon as any
// point closer than the bound is found, or once every unexplored cell is farther than the bound.
__device__ bool grid_nn(const GridView& g, double qx, double qy, double qz, int rmax, double cap2,
                        double& best, long long& bidx) {
  const int cx = cell_coord(qx, g.ox, g.inv_h, g.nx);
  const int cy = cell_coord(qy, g.oy, g.inv_h, g.ny);
  const int cz = cell_coord(qz, g.oz, g.inv_h, g.nz);
  best = kInf;
  bidx = -1;
  uint32_t bpos = 0;
  const uint32_t* __restrict__ cs = g.cell_start;
  for (int r = 1;; ++r) {
    const int x0 = cx - r, x1 = cx + r, y0 = cy - r, y1 = cy + r, z0 = cz - r, z1 = cz + r;
    const int xa = max(x0, 0), xb = min(x1, g.nx - 1);
    const int za = max(z0, 0), zb = min(z1, g.nz - 1);
    const int ya = max(y0, 0), yb = min(y1, g.ny - 1);
    for (int z = za; z <= zb; ++z) {
      for (int y = ya; y <= yb; ++y) {
        const long long row = ((long long)z * g.ny + y) * g.nx;
        const bool full = (r == 1) || z == z0 || z == z1 || y == y0 || y == y1;
        if (full) {
          scan_range(g.recs, cs[row + xa], cs[row + xb + 1], qx, qy, qz, best, bidx, bpos);
        } else {
          if (x0 >= 0) scan_range(g.recs, cs[row + x0], cs[row + x0 + 1], qx, qy, qz, best, bidx, bpos);
          if (x1 < g.nx) scan_range(g.recs, cs[row + x1], cs[row + x1 + 1], qx, qy, qz, best, bidx, bpos);
        }
      }
    }
    // distance from the query to the nearest face behind which unexplored cells remain
    double guard = kInf;
    if (x0 > 0) guard = fmin(guard, qx - (g.ox + x0 * g.h));
    if (x1 < g.nx - 1) guard = fmin(guard, (g.ox + (x1 + 1) * g.h) - qx);
    if (y0 > 0) guard = fmin(guard, qy - (g.oy + y0 * g.h));
    if (y1 < g.ny - 1) guard = fmin(guard, (g.oy + (y1 + 1) * g.h) - qy);
    if (z0 > 0) guard = fmin(guard, qz - (g.oz + z0 * g.h));
    if (z1 < g.nz - 1) guard = fmin(guard, (g.oz + (z1 + 1) * g.h) - qz);
    if (guard >= kInf) return true;  // the block covers the whole grid
    guard -= 1e-9 * g.h;             // cell assignment of points rounds at the 1e-13 level
    if (guard > 0.0 && best <= guard * guard) return true;
    if (cap2 >= 0.0 && (best < cap2 || (guard > 0.0 && guard * guard >= cap2))) return true;
    if (r >= rmax) return false;
  }
}

// signed point-to-plane distance exactly as the reference evaluates it (corrpts.py:198-209):
// (dx*nx + dy*ny) + dz*nz with the float32 normal promoted to float64, no fused multiply-add.
__device__ __forceinline__ double plane_distance(const Rigid& T, const double* __restrict__ mov_xyz,
                                                 long long j, double px, double py, double pz,
                                                 float4 nrm) {
  double tx, ty, tz;
  rigid_apply(T, mov_xyz[3 * j + 0], mov_xyz[3 * j + 1], mov_xyz[3 * j + 2], tx, ty, tz);
  const double dx = tx - px, dy = ty - py, dz = tz - pz;
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, (double)nrm.x), __dmul_rn(dy, (double)nrm.y)),
                   __dmul_rn(dz, (double)nrm.z));
}

__device__ __forceinline__ double plane_distance_rec(const Rigid& T, const Rec& m, double px, double py,
                                                     double pz, float4 nrm) {
  double tx, ty, tz;
  rigid_apply(T, m.x, m.y, m.z, tx, ty, tz);
  const double dx = tx - px, dy = ty - py, dz = tz - pz;
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, (double)nrm.x), __dmul_rn(dy, (double)nrm.y)),
                   __dmul_rn(dz, (double)nrm.z));
}

// Feed the predictor histogram of the reject kernel (reject_solve.cuh: lh_bin): one spread-out
// atomic per member of the statistics set instead of a separate pass over the distances later.
// The value the atomic returns is the correspondence's rank inside its bin: it doubles as the
// slot of a per-bin store of the members' order-preserving distance keys (f64_to_key), so that
// the reject/solve kernel reads the members of the few bins that hold its order statistics with
// one load each (no scan, no gather pass, no barrier, no index chase).
struct Pred {
  double med, mad, minpl;
  int valid;
};
__device__ __forceinline__ Pred load_pred(const DevState* st) {
  return Pred{st->pred_med, st->pred_mad, st->pred_minpl, st->pred_valid};
}
// Returns the slot (0 when the correspondence is not a member), for the diagnostics stamp that
// marks the atomic's return.
__device__ __forceinline__ unsigned int lin_hist_add(const Pred& p, unsigned int* lin_hist, float planarity, double d,
                                                     unsigned long long* binstore, int bin_cap, long long qi) {
  if (lin_hist != nullptr && p.valid && (double)planarity >= p.minpl) {
    const int b = lh_bin(d, p.med, p.mad);
    const unsigned int slot = atomicAdd(&lin_hist[b], 1u);
    if (binstore != nullptr && b < LH_BINS && slot < (unsigned int)bin_cap)
      binstore[(size_t)b * bin_cap + slot] = f64_to_key(d);
    return slot;
  }
  return 0u;
}
__device__ __forceinline__ void lin_hist_add(const DevState* st, unsigned int* lin_hist,
                                             float planarity, double d, unsigned long long* binstore,
                                             int bin_cap, long long qi) {
  lin_hist_add(load_pred(st), lin_hist, planarity, d, binstore, bin_cap, qi);
}

// Epilogue data of one correspondence for the fused reject/solve kernel: the matched movable
// point in caller coordinates (so the moment pass streams it instead of chasing nn_idx ->
// mov_xyz) and the histogram code.
struct CorrOut {
  unsigned long long* binstore;  // LH_BINS x bin_cap distance keys, may be null
  int bin_cap;
  double* m_xyz;           // K x 3, may be null
  // Warm start (may be null): position, in the cell-sorted record array, of the neighbour each
  // query found in the PREVIOUS iteration of this registration.  Its distance to the moved query
  // is a valid upper bound from the first instruction on, so most of the 27 cells of ring 1 are
  // pruned by their distance bound before their cell-table entries are even requested.  The
  // result is unchanged (any point is a valid bound; ties still go to the lower index).
  uint32_t* nn_pos;
  int warm;              // nn_pos holds positions of the previous iteration
  int sphere;            // finish a search inside the sphere of the first known point (option "sphere_scan")
  // Movable-side attributes (null = the reference's default run, pc_mov without normals):
  // mov_nrm[j] = (nx, ny, nz, planarity) of movable point j in ITS OWN frame, NaN where not
  // estimated.  q_eff[i] receives the fixed normal with an "effective planarity" that carries
  // both movable-side tests to the reject kernels (effective_planarity below).
  const float4* mov_nrm;
  float4* q_eff;
  double cos_max;        // cos of the largest accepted angle between the normals; < 0: no angle test
};
// CorrPts.reject_wrt_planarity's second branch (corrpts.py:157-162: a correspondence also needs
// planarity >= min_planarity on the MOVABLE side when pc_mov carries the column; NaN, i.e. "not
// estimated", fails the comparison) and the hook the reference leaves unimplemented
// (reject_wrt_to_angle_between_normals, corrpts.py:190-193; called after the distance rejection,
// simpleicp.py:207).  Both are folded into one float per correspondence:
//   |w| = min(planarity_fix, planarity_mov)   (NaN if either is NaN): both planarity tests are
//         |w| >= min_planarity, and the median / MAD population is the set that passes them;
//   sign(w) = 1 if the angle between the fixed normal and the ROTATED movable normal exceeds the
//         limit (normals are axes: the angle is taken modulo their sign): such a correspondence
//         takes part in the median / MAD like in the reference's call order, and is dropped after it.
__device__ __forceinline__ float effective_planarity(const CorrOut& co, const Rigid& T, long long qi,
                                                     long long midx, const float4& nr) {
  if (co.mov_nrm == nullptr) return nr.w;
  const float4 m = co.mov_nrm[midx];
  float w = (m.w >= nr.w) ? nr.w : ((m.w < nr.w) ? m.w : __int_as_float(0x7fc00000));
  if (co.cos_max >= 0.0) {
    const double rx = T.r[0] * (double)m.x + T.r[1] * (double)m.y + T.r[2] * (double)m.z;
    const double ry = T.r[3] * (double)m.x + T.r[4] * (double)m.y + T.r[5] * (double)m.z;
    const double rz = T.r[6] * (double)m.x + T.r[7] * (double)m.y + T.r[8] * (double)m.z;
    const double c = fabs(rx * (double)nr.x + ry * (double)nr.y + rz * (double)nr.z);
    if (!(c >= co.cos_max)) w = __int_as_float(__float_as_int(w) | 0x80000000);
  }
  co.q_eff[qi] = make_float4(nr.x, nr.y, nr.z, w);
  return fabsf(w);
}
// Certificate of the one-pair warm-started match (DESIGN §3.2, "certificate"): a search that
// finishes in the warm sphere scan proves that the record it found stays the strict nearest
// neighbour of every query within rho of the query it searched, c.  The next match of the same
// query skips its search while the moved query is provably inside that ball.  Part of the
// warm-start state: valid exactly where nn_pos is.
#ifndef SICP_CERT_SKIN
#define SICP_CERT_SKIN 0.125f  // skin of the sphere scan that writes a certificate, in cells
#endif
constexpr float kCertSkin = SICP_CERT_SKIN;
struct MatchCert {
  double* c;              // K x 3: the moved query of the search that wrote the certificate
  float* rho;             // K: radius of the certified ball, rounded down; <= 0: no certificate
  unsigned int* n_cert;   // queries of this launch answered from their certificate
  unsigned int* n_clear;  // the next launch's counter: zeroed here (ctx.cuh: cert_count)
  unsigned long long* stamps;  // diagnostics, may be null: 16 phase stamps (sicp_get_match_phase_times)
};

// %globaltimer once `dep` has arrived: the timer read is predicated on a test of dep, so it cannot
// issue before the loads dep is made of (a plain read would not wait for them).  0 in the
// (diagnostics-only) case dep == ~0u.
__device__ __forceinline__ unsigned long long global_timer_after(unsigned int dep) {
  unsigned long long t;
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0xffffffff;\n\tmov.u64 %0, 0;\n\t@p mov.u64 %0, %%globaltimer;\n\t}"
      : "=l"(t)
      : "r"(dep));
  return t;
}
// A load the compiler keeps where it is written: it is not merged with a plain load of the same
// address, and it stays ahead of the dependent-launch wait that follows it in the source (SASS:
// LDG.STRONG.GPU before ACQBULK).  ptxas moves weak loads, .nc ones included, below the wait.
__device__ __forceinline__ double ld_early(const double* p) {
  double v;
  asm volatile("ld.relaxed.gpu.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int dep_bits(double v) {
  return (unsigned int)__double2hiint(v) ^ (unsigned int)__double2loint(v);
}

__device__ __forceinline__ void store_matched(const CorrOut& co, long long qi, double x, double y, double z) {
  if (co.m_xyz) {
    co.m_xyz[3 * qi + 0] = x;
    co.m_xyz[3 * qi + 1] = y;
    co.m_xyz[3 * qi + 2] = z;
  }
}

__global__ void __launch_bounds__(128)
    k_match_grid(GridView g, const DevState* __restrict__ st, const double* __restrict__ q_xyz,
                 const float4* __restrict__ q_nrm, const double* __restrict__ mov_xyz, long long K,
                 int rmax, int with_distance, long long* __restrict__ nn_idx,
                 double* __restrict__ out, unsigned int* __restrict__ unresolved,
                 unsigned int* __restrict__ lin_hist, double cap2, CorrOut co) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= K || st->stop) return;
  const Rigid Tinv = st->Tinv;
  const double px = q_xyz[3 * i + 0], py = q_xyz[3 * i + 1], pz = q_xyz[3 * i + 2];
  double qx, qy, qz;
  rigid_apply(Tinv, px, py, pz, qx, qy, qz);
  double best;
  long long bidx;
  const bool ok = grid_nn(g, qx, qy, qz, rmax, cap2, best, bidx);
  if (!ok) {
    const unsigned int slot = atomicAdd(&unresolved[K], 1u);
    unresolved[slot] = (unsigned int)i;
    return;
  }
  nn_idx[i] = bidx;
  if (with_distance) {
    const float4 nr = q_nrm[i];
    const double d = plane_distance(st->T, mov_xyz, bidx, px, py, pz, nr);
    out[i] = d;
    lin_hist_add(st, lin_hist, effective_planarity(co, st->T, i, bidx, nr), d, co.binstore, co.bin_cap, i);
    store_matched(co, i, mov_xyz[3 * bidx + 0], mov_xyz[3 * bidx + 1], mov_xyz[3 * bidx + 2]);
  } else {
    out[i] = best;
  }
}

// Cooperative variant: MG lanes share one query.  In ring 1 every lane owns one of the 9 grid
// rows (x-contiguous cell triples), so the 9 dependent chains cell_start -> records run side by
// side instead of back to back; the winners are combined with a shuffle min-reduction inside the
// 16-lane group.  Later rings deal their (2r+1)^2 rows round-robin over the lanes.  The search is
// latency-bound (a handful of 32-byte L2 sectors per query), so what counts is how many of
// those loads are in flight — with one thread per query a K = 1000 search took 27 us.
// KEEP (overlap filter of a batch, with_distance = 0, unlimited rings): instead of nn_idx and the
// squared distance, keep[qi] = (d2 < cap2), the comparison of k_range_keep (capi.cu).
// CERT (one-pair match only): read and write the certificates of `cert` (MatchCert above);
// cert.rho is null when the launch keeps none (with_distance = 0).
// Returns true on the one lane of a group that answered its query from the certificate.
template <int MG, bool KEEP = false, bool CERT = false>
__device__ __forceinline__ bool match_coop_body(
    const GridView& g, const DevState* __restrict__ st, const double* __restrict__ q_xyz,
    const float4* __restrict__ q_nrm, const double* __restrict__ mov_xyz, long long K, int rmax,
    int with_distance, long long* __restrict__ nn_idx, double* __restrict__ out,
    unsigned int* __restrict__ unresolved, unsigned int* __restrict__ lin_hist, double cap2,
    const CorrOut& co, const long long gt, uint32_t* __restrict__ keep = nullptr,
    const MatchCert& cert = MatchCert{}) {
  const long long qi = gt / MG;
  const int sub = threadIdx.x & (MG - 1);
  // diagnostics: thread 0 of the first and of the last block stamps its phases
  unsigned long long* const stamp =
      (CERT && cert.stamps != nullptr && threadIdx.x == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1))
          ? cert.stamps + ((blockIdx.x == 0) ? 0 : 8)
          : nullptr;
  if (stamp) {
    stamp[0] = global_timer_ns();
    for (int i = 1; i < 7; ++i) stamp[i] = 0ull;  // a phase this launch does not reach reads -1
  }
  pdl_launch_dependents();
  if (qi >= K) return false;  // a whole group leaves together
  // The query's coordinates do not depend on the previous kernel: on their way before the wait.
  // The certified path takes its own copy through ld_early (below): a plain load is one value
  // with the search's copy, which lives through the whole search, so at the register bound the
  // compiler spilled it at once (waiting for the cold line before the wait) or sank the load
  // below the wait.  The search reads q_xyz again after the decision (an L1/L2 hit).
  double px, py, pz;
  if constexpr (!CERT) {
    px = q_xyz[3 * qi + 0];
    py = q_xyz[3 * qi + 1];
    pz = q_xyz[3 * qi + 2];
  }
  double epx = 0.0, epy = 0.0, epz = 0.0;
  if constexpr (CERT) {
    if (co.warm) {
      epx = ld_early(q_xyz + 3 * qi + 0);
      epy = ld_early(q_xyz + 3 * qi + 1);
      epz = ld_early(q_xyz + 3 * qi + 2);
    }
  }
  pdl_wait();
  if (stamp) stamp[1] = global_timer_ns();
  if constexpr (CERT) {
    if (gt == 0 && cert.n_clear) *cert.n_clear = 0u;
    // Fast path: |q - c| < rho (computed norm times 1 + 1e-12, an upper bound) proves that the
    // full search would return the record at nn_pos[qi] again, as the strict winner (DESIGN §3.2).
    // nn_idx, nn_pos, m_xyz and the certificate keep their values; only the epilogue runs.  A
    // non-finite q fails the comparison.  Every line the decision and the answer need
    // (certificate, matched point, normal, stop flag, Tinv) is requested in one round: the stop
    // flag is part of the decision instead of a branch before it, since the compiler sinks loads
    // below such a branch.  T and the predictor are read after the decision: the state's lines
    // are shared by every query, so that read hits L1 or L2.
    if (co.warm) {
      const double cx = cert.c[3 * qi + 0], cy = cert.c[3 * qi + 1], cz = cert.c[3 * qi + 2];
      const float rho = cert.rho[qi];
      const double mx = co.m_xyz[3 * qi + 0], my = co.m_xyz[3 * qi + 1], mz = co.m_xyz[3 * qi + 2];
      const int stop = st->stop;
      const Rigid Tinv = st->Tinv;
      const long long midx = co.mov_nrm ? nn_idx[qi] : -1;
      const float4 nr = q_nrm[qi];
      double qx, qy, qz;
      rigid_apply(Tinv, epx, epy, epz, qx, qy, qz);
      const double ex = qx - cx, ey = qy - cy, ez = qz - cz;
      if (stamp) stamp[2] = global_timer_after(dep_bits(ex + ey + ez) ^ __float_as_uint(rho));
      if (stop == 0 && sqrt(ex * ex + ey * ey + ez * ez) * (1.0 + 1e-12) < (double)rho) {
        if (sub != 0) return false;
        if (stamp) stamp[3] = global_timer_ns();
        const Rigid T = st->T;
        const Pred pred = load_pred(st);
        const Rec m{mx, my, mz, midx};
        const double d = plane_distance_rec(T, m, epx, epy, epz, nr);
        if (stamp) stamp[4] = global_timer_after(dep_bits(d));
        out[qi] = d;
        const unsigned int slot =
            lin_hist_add(pred, lin_hist, effective_planarity(co, T, qi, m.idx, nr), d, co.binstore, co.bin_cap, qi);
        if (stamp) stamp[5] = global_timer_after(slot ^ 0x80000000u);
        return true;
      }
    }
    px = q_xyz[3 * qi + 0];
    py = q_xyz[3 * qi + 1];
    pz = q_xyz[3 * qi + 2];
  }
  if (st->stop) return false;
  const unsigned int gmask = (MG == 32) ? 0xffffffffu : (((1u << MG) - 1u) << ((threadIdx.x & 31) & ~(MG - 1)));
  const Rigid Tinv = st->Tinv;
  double qx, qy, qz;
  rigid_apply(Tinv, px, py, pz, qx, qy, qz);
  const int cx = cell_coord(qx, g.ox, g.inv_h, g.nx);
  const int cy = cell_coord(qy, g.oy, g.inv_h, g.ny);
  const int cz = cell_coord(qz, g.oz, g.inv_h, g.nz);
  const uint32_t* __restrict__ cs = g.cell_start;
  // the normal is only needed at the very end: start its (cold) line on the way now
  if (with_distance && sub == 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(q_nrm + qi));
  double best = kInf;
  long long bidx = -1;
  uint32_t bpos = 0;
  bool resolved = false;
  if (co.warm) {
    const uint32_t p = co.nn_pos[qi];
    if ((long long)p < g.n_points) consider(g.recs[p], p, qx, qy, qz, best, bidx, bpos);
  }
  // Sphere scan: once ANY point is known (its squared distance is `best`), the nearest neighbour
  // lies inside the sphere of that radius around the query, i.e. in the cells of the box
  // [q - R, q + R] clipped to the grid; each x-row of the box is pruned by its distance to the
  // query and narrowed to the chord of the sphere.  With a good bound (the previous iteration's
  // neighbour) that is 1-4 rows of 1-2 cells instead of the 27 cells of ring 1; for a query
  // outside the cloud's box (partial overlap) it is the small cap of the sphere that reaches into
  // the grid instead of rings expanding through empty space.  rs = radius of the cube of cells
  // already scanned around the query's cell (0: none).  Returns false (nothing done) when the box
  // is too large to be worth it: the bound is poor, another ring will improve it.
  // The row bounds are evaluated in float, in CELL units, with margins that keep every bound on
  // the safe side (a row is only skipped / narrowed when it certainly holds nothing nearer than
  // `best`); the distances themselves stay float64.  (Per-row float64 bounds, a float64 sqrt, two
  // float64 floor conversions and an integer division were half of the first iteration's
  // instructions.)
  const float fqx = (float)((qx - g.ox) * g.inv_h), fqy = (float)((qy - g.oy) * g.inv_h),
              fqz = (float)((qz - g.oz) * g.inv_h);
  // float32 error of a cell coordinate (a query may lie far outside the grid) + cell faces vs the
  // floor() that assigned the points
  const float marg = 1e-3f + 4e-7f * fmaxf(fmaxf(fabsf(fqx), fabsf(fqy)),
                                           fmaxf(fabsf(fqz), (float)max(g.nx, max(g.ny, g.nz))));
  const double inv_h2 = g.inv_h * g.inv_h;
  // With a certificate to write (S true), the scan prunes with the skin: rows and chords are
  // bounded by (sqrt(best) + kCertSkin h)^2 instead of best, a superset of the same candidates
  // (the result does not change), it keeps sec (consider_sec) and sets rho.
  float rho = 0.0f;
  auto sphere_scan = [&](auto S, const int rs, const int max_rows) -> bool {
    constexpr bool SK = decltype(S)::value;
    // squared pruning radius in cells, rounded up; ties are still visited (1e-12)
    auto lim_of = [&](double b) -> float {
      if constexpr (SK) {
        const float r = __fadd_ru(__fsqrt_ru(__double2float_ru(b * (1.0 + 1e-12) * inv_h2)), kCertSkin);
        return __fmul_ru(r, r);
      } else {
        return __double2float_ru(b * (1.0 + 1e-12) * inv_h2);
      }
    };
    double sec = kInf;
    float Rc = sqrtf(__double2float_ru(best * inv_h2)) * (1.0f + 1e-6f) + marg;  // radius in cells, rounded up
    if constexpr (SK) Rc += kCertSkin;
    const int ya = min(max(__float2int_rd(fqy - Rc), 0), g.ny - 1), yb = min(max(__float2int_rd(fqy + Rc), 0), g.ny - 1);
    const int za = min(max(__float2int_rd(fqz - Rc), 0), g.nz - 1), zb = min(max(__float2int_rd(fqz + Rc), 0), g.nz - 1);
    const int nyb = yb - ya + 1;
    const long long rows = (long long)nyb * (zb - za + 1);
    if (rows > max_rows) return false;
    // (yr, zr) walk the box with stride MG, kept incrementally (no division per row)
    int zr = sub / nyb, yr = sub - zr * nyb;
    float limc = lim_of(best);
    double best_seen = best;
    for (int t = sub; t < (int)rows; t += MG, yr += MG) {
      while (yr >= nyb) {
        yr -= nyb;
        ++zr;
      }
      const int yy = ya + yr, zz = za + zr;
      if (best != best_seen) {
        best_seen = best;
        limc = lim_of(best);
      }
      const float by = fmaxf(fabsf(fqy - ((float)yy + 0.5f)) - 0.5f - marg, 0.0f);
      const float bz = fmaxf(fabsf(fqz - ((float)zz + 0.5f)) - 0.5f - marg, 0.0f);
      const float lb = (by * by + bz * bz) * (1.0f - 1e-6f);  // rounded down
      if (lb > limc) continue;
      const float xr = sqrtf(limc - lb) * (1.0f + 1e-6f) + marg;
      const int xs = max(__float2int_rd(fqx - xr), 0), xe = min(__float2int_rd(fqx + xr), g.nx - 1);
      if (xs > xe) continue;  // the chord lies outside the grid
      const uint32_t row = ((uint32_t)zz * (uint32_t)g.ny + (uint32_t)yy) * (uint32_t)g.nx;  // < 2^25 cells
      if (rs > 0 && abs(yy - cy) <= rs && abs(zz - cz) <= rs) {
        // cells cx - rs .. cx + rs of this row were scanned by the rings
        const int le = min(xe, cx - rs - 1), rb = max(xs, cx + rs + 1);
        if (xs <= le) scan_range(g.recs, cs[row + xs], cs[row + le + 1], qx, qy, qz, best, bidx, bpos);
        if (rb <= xe) scan_range(g.recs, cs[row + rb], cs[row + xe + 1], qx, qy, qz, best, bidx, bpos);
      } else if constexpr (SK) {  // rs = 0: the warm-start scan
        scan_range_sec(g.recs, cs[row + xs], cs[row + xe + 1], qx, qy, qz, best, bidx, bpos, sec);
      } else {
        scan_range(g.recs, cs[row + xs], cs[row + xe + 1], qx, qy, qz, best, bidx, bpos);
      }
    }
#pragma unroll
    for (int o = MG / 2; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(gmask, best, o, MG);
      const long long oi = __shfl_xor_sync(gmask, bidx, o, MG);
      const uint32_t op = __shfl_xor_sync(gmask, bpos, o, MG);
      if constexpr (SK) {
        // the pair's loser is a second point unless it is the winner's record (bidx >= 0 in
        // every lane: the scan starts from the warm-start record)
        const double osec = __shfl_xor_sync(gmask, sec, o, MG);
        const bool take = od < best || (od == best && oi < bidx);
        sec = fmin(sec, osec);
        if (op != bpos) sec = fmin(sec, take ? best : od);
        if (take) {
          best = od;
          bidx = oi;
          bpos = op;
        }
      } else if (od < best || (od == best && oi >= 0 && (bidx < 0 || oi < bidx))) {
        best = od;
        bidx = oi;
        bpos = op;
      }
    }
    if constexpr (SK) {
      // U >= |c - m| and L <= |c - j| for every other record j: sec bounds the visited ones (the
      // computed squared distances are within a few ulps), and every record the scan skipped lies
      // farther than sqrt(lim_of(best)) cells: each lane pruned with lim_of(its best) >=
      // lim_of(the group's best), rounded up, with the margins of the row bounds
      const double L = fmin(sqrt(sec) * (1.0 - 1e-14), sqrt((double)lim_of(best)) * g.h * (1.0 - 1e-6));
      const double U = sqrt(best) * (1.0 + 1e-14);
      rho = __double2float_rd((L - U) * 0.5 - 1e-12 * L);
    }
    return true;
  };
  const bool use_sphere = (cap2 < 0.0) && co.sphere;
  // Warm start: finish inside the sphere of the previous neighbour right away when that sphere
  // is small (the steady state: 1-4 rows).  After a large update of the transform (second
  // iteration of a registration) the old neighbour is a poor bound — several cells — while the
  // true one is almost surely in the query's own row: ring 1 first, it prunes with the bound it
  // has and leaves a much smaller sphere to the scan after it.
  if (use_sphere && best < kInf && sphere_scan(std::integral_constant<bool, CERT>{}, 0, 4 * MG)) resolved = true;
  for (int r = 1; !resolved; ++r) {
    const int x0 = cx - r, x1 = cx + r;
    const int xa = max(x0, 0), xb = min(x1, g.nx - 1);
    if (r == 1) {
      // Ring 1 in two steps.  (1) the query's own x-row, one cell per lane; (2) the eight
      // neighbouring rows, each skipped (or narrowed in x) when the distance from the query to
      // the row / cell already exceeds the best distance of step 1 — the nearest neighbour
      // is usually in the own row, so most of the 27 cells are never read.
      // (Requesting every cell-table entry step 2 might need before step 1's records — to shorten
      // the chain of dependent round trips — was measured 10 % SLOWER: the kernel is bound by
      // issue slots as much as by latency, and 8 extra loads per lane cost more than the round
      // trip they save.)
      constexpr int NR = (8 + MG - 1) / MG;  // rows per lane in step 2
      // distances from the query to the faces of its own cell (>= 0 up to rounding)
      const double fxl = fmax(qx - (g.ox + cx * g.h), 0.0), fxh = fmax((g.ox + (cx + 1) * g.h) - qx, 0.0);
      const double fyl = fmax(qy - (g.oy + cy * g.h), 0.0), fyh = fmax((g.oy + (cy + 1) * g.h) - qy, 0.0);
      const double fzl = fmax(qz - (g.oz + cz * g.h), 0.0), fzh = fmax((g.oz + (cz + 1) * g.h) - qz, 0.0);
#pragma unroll
      for (int t = sub; t < 3 || t == sub; t += MG) {  // one pass for MG >= 4, two for MG = 2
        const int x = cx - 1 + t;
        bool own = t < 3 && x >= 0 && x < g.nx;
        // with a warm-start bound the two side cells of the own row are usually out of reach
        const double bx = (t == 0) ? fxl : ((t == 2) ? fxh : 0.0);
        if (bx * bx > best * (1.0 + 1e-12)) own = false;
        const long long row0 = ((long long)cz * g.ny + cy) * g.nx;
        const uint32_t os = own ? cs[row0 + x] : 0u, oe = own ? cs[row0 + x + 1] : 0u;
        scan_range(g.recs, os, oe, qx, qy, qz, best, bidx, bpos);
        if (MG >= 3) break;
      }
#pragma unroll
      for (int o = MG / 2; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(gmask, best, o, MG);
        const long long oi = __shfl_xor_sync(gmask, bidx, o, MG);
        const uint32_t op = __shfl_xor_sync(gmask, bpos, o, MG);
        if (od < best || (od == best && oi >= 0 && (bidx < 0 || oi < bidx))) {
          best = od;
          bidx = oi;
          bpos = op;
        }
      }
      const double lim = best * (1.0 + 1e-12);  // strictly farther only: ties are still visited
      uint32_t rs[NR], re[NR];
#pragma unroll
      for (int u = 0; u < NR; ++u) {
        rs[u] = re[u] = 0;
        const int t = sub + u * MG;
        if (t >= 8) continue;
        const int tt = t + (t >= 4 ? 1 : 0);  // 0..8 without the centre (4)
        const int dz = tt / 3 - 1, dy = tt % 3 - 1;
        const int y = cy + dy, z = cz + dz;
        if (y < 0 || y >= g.ny || z < 0 || z >= g.nz) continue;
        const double by = (dy < 0) ? fyl : ((dy > 0) ? fyh : 0.0);
        const double bz = (dz < 0) ? fzl : ((dz > 0) ? fzh : 0.0);
        const double lb = by * by + bz * bz;
        if (lb > lim) continue;
        int xs = xa, xe = xb;
        if (x0 >= 0 && lb + fxl * fxl > lim) xs = cx;
        if (x1 < g.nx && lb + fxh * fxh > lim) xe = cx;
        const long long row = ((long long)z * g.ny + y) * g.nx;
        rs[u] = cs[row + xs];
        re[u] = cs[row + xe + 1];
      }
#pragma unroll
      for (int u = 0; u < NR; ++u) scan_range(g.recs, rs[u], re[u], qx, qy, qz, best, bidx, bpos);
    } else {
      const int side = 2 * r + 1, items = side * side;
      // (dy, dz) walk the (2r+1)^2 rows with stride MG; kept incrementally — two integer
      // divisions by the run-time `side` per row were a third of the instructions of this loop
      int dzr = sub / side, dyr = sub - dzr * side;
      for (int t = sub; t < items; t += MG, dyr += MG) {
        while (dyr >= side) {
          dyr -= side;
          ++dzr;
        }
        const int dz = dzr - r, dy = dyr - r;
        const int y = cy + dy, z = cz + dz;
        if (y < 0 || y >= g.ny || z < 0 || z >= g.nz) continue;
        const long long row = ((long long)z * g.ny + y) * g.nx;
        const bool full = dy == -r || dy == r || dz == -r || dz == r;
        if (full) {
          scan_range(g.recs, cs[row + xa], cs[row + xb + 1], qx, qy, qz, best, bidx, bpos);
        } else {
          if (x0 >= 0) scan_range(g.recs, cs[row + x0], cs[row + x0 + 1], qx, qy, qz, best, bidx, bpos);
          if (x1 < g.nx) scan_range(g.recs, cs[row + x1], cs[row + x1 + 1], qx, qy, qz, best, bidx, bpos);
        }
      }
    }
    // min-reduction of (d2, idx) over the 16 lanes of the group; every lane ends with the result
#pragma unroll
    for (int o = MG / 2; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(gmask, best, o, MG);
      const long long oi = __shfl_xor_sync(gmask, bidx, o, MG);
      const uint32_t op = __shfl_xor_sync(gmask, bpos, o, MG);
      if (od < best || (od == best && oi >= 0 && (bidx < 0 || oi < bidx))) {
        best = od;
        bidx = oi;
        bpos = op;
      }
    }
    const int y0 = cy - r, y1 = cy + r, z0 = cz - r, z1 = cz + r;
    double guard = kInf;
    if (x0 > 0) guard = fmin(guard, qx - (g.ox + x0 * g.h));
    if (x1 < g.nx - 1) guard = fmin(guard, (g.ox + (x1 + 1) * g.h) - qx);
    if (y0 > 0) guard = fmin(guard, qy - (g.oy + y0 * g.h));
    if (y1 < g.ny - 1) guard = fmin(guard, (g.oy + (y1 + 1) * g.h) - qy);
    if (z0 > 0) guard = fmin(guard, qz - (g.oz + z0 * g.h));
    if (z1 < g.nz - 1) guard = fmin(guard, (g.oz + (z1 + 1) * g.h) - qz);
    if (guard >= kInf) {
      resolved = true;
      break;
    }
    guard -= 1e-9 * g.h;
    if (guard > 0.0 && best <= guard * guard) {
      resolved = true;
      break;
    }
    if (cap2 >= 0.0 && (best < cap2 || (guard > 0.0 && guard * guard >= cap2))) {
      resolved = true;  // overlap filter: the side of the bound is decided (see grid_nn)
      break;
    }
    // Nothing within the 27 cells (first iteration of a registration: the clouds are still apart
    // by several cells, typically along the surface normal).  A cube grown ring by ring meets a
    // sheet-like surface with a whole FACE at once — hundreds of candidates at ring r, thousands
    // of cell-table reads before it.  Probe outwards along the three axes instead (six cells per
    // step): a surface at distance D crosses one of the axes within sqrt(3) D, the first point
    // found bounds the search, and the sphere scan below finishes it.
    if (use_sphere && r == 1 && best == kInf) {
      // The y and z probes read three x-neighbouring cells (one contiguous record range, the same
      // two cell-table loads): a sheet sampled at ~3 points per cell has holes, and a probe that
      // slips through one runs on until another axis meets the surface ten times farther out —
      // 5 % of the queries of the C3 pair, i.e. a third of the warps, with single-cell probes.
      // The lanes only vote per step; the (distance, index, position) reduction runs once, after
      // the step that found something.
      for (int s2 = 2; s2 <= 96; ++s2) {
        bool any_inside = false;
        for (int t = sub; t < 6; t += MG) {
          const int axis = t >> 1, off = (t & 1) ? s2 : -s2;
          const int x = cx + (axis == 0 ? off : 0), y = cy + (axis == 1 ? off : 0), z = cz + (axis == 2 ? off : 0);
          if (x < 0 || x >= g.nx || y < 0 || y >= g.ny || z < 0 || z >= g.nz) continue;
          any_inside = true;
          const long long row = ((long long)z * g.ny + y) * g.nx;
          const int xl = (axis == 0) ? x : max(x - 1, 0), xh = (axis == 0) ? x : min(x + 1, g.nx - 1);
          scan_range(g.recs, cs[row + xl], cs[row + xh + 1], qx, qy, qz, best, bidx, bpos);
        }
        const bool found = __any_sync(gmask, best < kInf);
        const bool inside = __any_sync(gmask, any_inside);
        if (found) {
#pragma unroll
          for (int o = MG / 2; o > 0; o >>= 1) {
            const double od = __shfl_xor_sync(gmask, best, o, MG);
            const long long oi = __shfl_xor_sync(gmask, bidx, o, MG);
            const uint32_t op = __shfl_xor_sync(gmask, bpos, o, MG);
            if (od < best || (od == best && oi >= 0 && (bidx < 0 || oi < bidx))) {
              best = od;
              bidx = oi;
              bpos = op;
            }
          }
          break;
        }
        if (!inside) break;
      }
    }
    // a point is known now: finish inside its sphere instead of growing the cube ring by ring
    // (best is uniform across the group after the reduction, so the whole group takes one branch)
    if (use_sphere && best < kInf && sphere_scan(std::false_type{}, r, 64 * MG)) {  // ~15 instructions per pruned row: cheaper than the next rings up to there
      resolved = true;
      break;
    }
    if (r >= rmax) break;
  }
  if (sub != 0) return false;
  if constexpr (KEEP) {
    // with cap2 the search stops once the side of the bound is decided (see grid_nn), so `best`
    // is then an upper bound below cap2 or a value at or above it: the comparison is exact
    keep[qi] = (best < cap2) ? 1u : 0u;  // strict: cKDTree distance_upper_bound semantics
    return false;
  }
  if (co.nn_pos) co.nn_pos[qi] = resolved ? bpos : 0xffffffffu;
  if constexpr (CERT) {
    if (cert.rho) {
      if (rho > 0.0f) {
        cert.c[3 * qi + 0] = qx;
        cert.c[3 * qi + 1] = qy;
        cert.c[3 * qi + 2] = qz;
      }
      cert.rho[qi] = rho;
    }
  }
  if (!resolved) {
    const unsigned int slot = atomicAdd(&unresolved[K], 1u);
    unresolved[slot] = (unsigned int)qi;
    return false;
  }
  nn_idx[qi] = bidx;
  if (with_distance) {
    const float4 nr = q_nrm[qi];
    // the winner's record was read a moment ago by a lane of this warp: same coordinates as
    // mov_xyz[bidx], but from L1/L2 instead of a cold line
    const Rec m = g.recs[bpos];
    const double d = plane_distance_rec(st->T, m, px, py, pz, nr);
    out[qi] = d;
    lin_hist_add(st, lin_hist, effective_planarity(co, st->T, qi, bidx, nr), d, co.binstore, co.bin_cap, qi);
    store_matched(co, qi, m.x, m.y, m.z);
  } else {
    out[qi] = best;
  }
  return false;
}

// 6 blocks per SM (80 registers): the certified steady state is a few dependent round trips per
// query, so its time is set by the number of waves; the compiler's own choice, 96, fits 5.
template <int MG>
__global__ void __launch_bounds__(128, 6)
    k_match_grid_coop(GridView g, const DevState* __restrict__ st, const double* __restrict__ q_xyz,
                      const float4* __restrict__ q_nrm, const double* __restrict__ mov_xyz,
                      long long K, int rmax, int with_distance, long long* __restrict__ nn_idx,
                      double* __restrict__ out, unsigned int* __restrict__ unresolved,
                      unsigned int* __restrict__ lin_hist, double cap2, CorrOut co, MatchCert cert) {
  const bool certified =
      match_coop_body<MG, false, true>(g, st, q_xyz, q_nrm, mov_xyz, K, rmax, with_distance, nn_idx, out, unresolved,
                                       lin_hist, cap2, co, blockIdx.x * (long long)blockDim.x + threadIdx.x, nullptr, cert);
  // One atomic per block on the certified counter instead of one per warp (a single address:
  // ~12 500 same-address atomics per launch at K = 100 000).  Every thread comes here, and a warp
  // that is done holds nothing while it waits: the block retires with its slowest warp either way.
  if (cert.n_cert) {
    const int n = __syncthreads_count(certified);
    if (threadIdx.x == 0 && n > 0) atomicAdd(cert.n_cert, (unsigned int)n);
  }
  if (cert.stamps && threadIdx.x == 0 && (blockIdx.x == 0 || blockIdx.x == gridDim.x - 1))
    cert.stamps[((blockIdx.x == 0) ? 0 : 8) + 6] = global_timer_ns();
}

// Batched form: blockIdx.y is the pair, everything else comes from its descriptor.  The ring
// expansion runs to completion (no brute-force hand-over inside a batch).
struct BatchMatchArgs {
  const PairDev* pairs;
  const DevState* state;
  const double* q_xyz;
  const float4* q_nrm;
  long long* nn_idx;
  double* dist;
  unsigned int* lin_hist;
  unsigned long long* binstore;
  int bin_cap;
  double* m_xyz;
  uint32_t* nn_pos;
  int warm;
  int sphere;
};
template <int MG>
__device__ __forceinline__ void match_batch_body(const BatchMatchArgs& a, const float4* mov_nrm, float4* q_eff,
                                                 double cos_max) {
  const PairDev pd = a.pairs[blockIdx.y];
  const long long gt = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (gt / MG >= pd.K) return;
  const long long q = pd.q_off;
  const CorrOut co{a.binstore + (size_t)blockIdx.y * LH_BINS * a.bin_cap, a.bin_cap, a.m_xyz + 3 * q, a.nn_pos + q, a.warm, a.sphere,
                   mov_nrm ? mov_nrm + pd.mov_off : nullptr, mov_nrm ? q_eff + q : nullptr, cos_max};
  match_coop_body<MG>(pd.gmov, a.state + blockIdx.y, a.q_xyz + 3 * q, a.q_nrm + q, nullptr, pd.K, 1 << 30, 1,
                      a.nn_idx + q, a.dist + q, nullptr, a.lin_hist + (size_t)blockIdx.y * (LH_BINS + 2), -1.0,
                      co, gt);
}
template <int MG>
__global__ void __launch_bounds__(128) k_match_batch(BatchMatchArgs a) {
  match_batch_body<MG>(a, nullptr, nullptr, -1.0);
}
// The form with movable-side attributes (mov_neighbors > 0), its own kernel so that the default
// batch keeps its code: mov_nrm = Batch::mov_nrm (total_mov), q_eff = Batch::q_nrm_eff.  Launched
// with 128 threads; 128 registers (instead of launch bounds) keep it free of spills (at 96 the
// 4-lane form spills).  Only the movable-attribute batches run it.
struct BatchMatchAttrArgs {
  BatchMatchArgs a;
  const float4* mov_nrm;
  float4* q_eff;
  double cos_max;
};
template <int MG>
__global__ void __maxnreg__(128) k_match_batch_attr(BatchMatchAttrArgs m) {
  match_batch_body<MG>(m.a, m.mov_nrm, m.q_eff, m.cos_max);
}

// Overlap filter of a batch (PointCloud.select_in_range, simpleicp.py:158-170): blockIdx.y is the
// pair, the queries are ALL its fixed points, read in place from the concatenated clouds, and the
// transform is the pair's DevState (its prior).  Bounded search with unlimited rings, one keep
// flag per fixed point of each pair, at the pair's own flag offset (pairs may share a fixed cloud).
template <int MG>
__global__ void __launch_bounds__(128)
    k_overlap_batch(const PairDev* __restrict__ pairs, const DevState* __restrict__ state,
                    const double* __restrict__ fix_xyz, double r2, uint32_t* __restrict__ keep) {
  const PairDev& pd = pairs[blockIdx.y];
  const long long n = pd.n_fix;
  const long long gt = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (gt / MG >= n) return;
  const CorrOut co{nullptr, 0, nullptr, nullptr, 0, 0, nullptr, nullptr, -1.0};
  match_coop_body<MG, true>(pd.gmov, state + blockIdx.y, fix_xyz + 3 * pd.fix_off, nullptr, nullptr, n, 1 << 30, 0,
                            nullptr, nullptr, nullptr, nullptr, r2, co, gt, keep + pd.flag_off);
}

// Culled overlap filter of sicp_register_to_map: blockIdx.y is the scan, blockIdx.x one x-row of
// the map grid inside the scan's MapCull cells, i.e. one contiguous range of cell-sorted map
// records.  The groups of MG lanes walk the row's records; a record inside the scan's box gets
// k_overlap_batch's bounded search (match_coop_body<MG, true> on the same coordinates, movable
// grid, prior and bound, so the flag is that of the batch filter bit for bit), and a survivor
// sets the bit of its map index in the scan's row of the mask (`words` words per scan).  Points
// outside the box cannot pass (batch.cu: map_cull_box), so they are skipped unsearched.
template <int MG>
__global__ void __launch_bounds__(128)
    k_map_overlap(const PairDev* __restrict__ pairs, const DevState* __restrict__ state,
                  const MapCull* __restrict__ culls, GridView map, double r2, long long words,
                  uint32_t* __restrict__ bits, unsigned long long* __restrict__ n_searched) {
  const MapCull& cu = culls[blockIdx.y];
  if ((long long)blockIdx.x >= cu.rows) return;
  const int ny = cu.c1[1] - cu.c0[1] + 1;
  const int y = cu.c0[1] + (int)(blockIdx.x % (unsigned)ny), z = cu.c0[2] + (int)(blockIdx.x / (unsigned)ny);
  const long long row = ((long long)z * map.ny + y) * map.nx;
  // the row's end is read from shared memory in every round: held in a register across the
  // inlined search it was spilled
  __shared__ uint32_t row_end;
  const uint32_t s = map.cell_start[row + cu.c0[0]];
  if (threadIdx.x == 0) row_end = map.cell_start[row + cu.c1[0] + 1];
  __syncthreads();
  const PairDev& pd = pairs[blockIdx.y];
  const CorrOut co{nullptr, 0, nullptr, nullptr, 0, 0, nullptr, nullptr, -1.0};
  const int sub = threadIdx.x & (MG - 1);
  uint32_t* __restrict__ mask = bits + (size_t)blockIdx.y * words;
  // the search's flag goes to a shared slot of the group (a local variable would live in memory)
  __shared__ uint32_t flags[128 / MG];
  uint32_t* flag = flags + threadIdx.x / MG;
  unsigned int searched = 0;
  for (uint32_t p = s + threadIdx.x / MG; p < *(volatile uint32_t*)&row_end; p += 128 / MG) {
    const Rec r = map.recs[p];  // the whole group reads the same record and takes the same branch
    if (r.x < cu.lo[0] || r.x > cu.hi[0] || r.y < cu.lo[1] || r.y > cu.hi[1] || r.z < cu.lo[2] || r.z > cu.hi[2])
      continue;
    const double q[3] = {r.x, r.y, r.z};
    match_coop_body<MG, true>(pd.gmov, state + blockIdx.y, q, nullptr, nullptr, 1, 1 << 30, 0, nullptr, nullptr,
                              nullptr, nullptr, r2, co, sub, flag);
    if (sub == 0) {  // the lane that wrote the flag
      ++searched;
      if (*flag) atomicOr(&mask[r.idx >> 5], 1u << (r.idx & 31));
    }
  }
  searched = __reduce_add_sync(0xffffffffu, searched);
  if ((threadIdx.x & 31) == 0 && searched) atomicAdd(n_searched, (unsigned long long)searched);
}

// Count of sicp_overlap_graph, k_map_overlap's walk for many directions: blockIdx.y is the
// direction (a, b), blockIdx.x one x-row of a's grid inside the direction's MapCull cells.  A
// record inside the box whose index is a multiple of `stride` gets k_overlap_batch's bounded
// search in b's grid under the direction's state (prior T_ab), so its flag is that of the pair's
// overlap filter bit for bit.  The survivors are counted per warp and added with one atomic per
// warp to the direction's 32-bit counter (a cloud has fewer than 2^32 points); integer sums, so
// the count does not depend on the order.
template <int MG>
__global__ void __launch_bounds__(128)
    k_overlap_count(const GridView* __restrict__ views, const DevState* __restrict__ state,
                    const OverlapDir* __restrict__ dirs, uint32_t stride, double r2, uint32_t* __restrict__ counts) {
  const OverlapDir& dr = dirs[blockIdx.y];
  const MapCull& cu = dr.cu;
  if ((long long)blockIdx.x >= cu.rows) return;
  const GridView& ga = views[dr.a];
  const int ny = cu.c1[1] - cu.c0[1] + 1;
  const int y = cu.c0[1] + (int)(blockIdx.x % (unsigned)ny), z = cu.c0[2] + (int)(blockIdx.x / (unsigned)ny);
  const long long row = ((long long)z * ga.ny + y) * ga.nx;
  // the row's end lives in shared memory, as in k_map_overlap
  __shared__ uint32_t row_end;
  const uint32_t s = ga.cell_start[row + cu.c0[0]];
  if (threadIdx.x == 0) row_end = ga.cell_start[row + cu.c1[0] + 1];
  __syncthreads();
  const Rec* __restrict__ recs = ga.recs;
  const CorrOut co{nullptr, 0, nullptr, nullptr, 0, 0, nullptr, nullptr, -1.0};
  const int sub = threadIdx.x & (MG - 1);
  __shared__ uint32_t flags[128 / MG];
  uint32_t* flag = flags + threadIdx.x / MG;
  unsigned int kept = 0;
  for (uint32_t p = s + threadIdx.x / MG; p < *(volatile uint32_t*)&row_end; p += 128 / MG) {
    const Rec r = recs[p];  // the whole group reads the same record and takes the same branch
    if (r.x < cu.lo[0] || r.x > cu.hi[0] || r.y < cu.lo[1] || r.y > cu.hi[1] || r.z < cu.lo[2] || r.z > cu.hi[2])
      continue;
    if (stride > 1 && (uint32_t)r.idx % stride != 0) continue;  // idx < 2^32 - 1
    const double q[3] = {r.x, r.y, r.z};
    match_coop_body<MG, true>(views[dr.b], state + blockIdx.y, q, nullptr, nullptr, 1, 1 << 30, 0, nullptr, nullptr,
                              nullptr, nullptr, r2, co, sub, flag);
    if (sub == 0) kept += *flag;  // the lane that wrote the flag
  }
  kept = __reduce_add_sync(0xffffffffu, kept);
  if ((threadIdx.x & 31) == 0 && kept) atomicAdd(&counts[dr.slot], kept);
}

__global__ void __launch_bounds__(256) k_map_popc(const uint32_t* __restrict__ bits, long long n, uint32_t* __restrict__ popc) {
  const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (w < n) popc[w] = (uint32_t)__popc(bits[w]);
}

// word w of scan w / per_scan holds map points 32 (w % per_scan) + b: its set bits go, in
// ascending order, to list[scan[w] ...]
__global__ void __launch_bounds__(256)
    k_map_scatter(const uint32_t* __restrict__ bits, long long n, long long per_scan,
                  const uint32_t* __restrict__ scan, uint32_t* __restrict__ list) {
  const long long w = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (w >= n) return;
  uint32_t v = bits[w];
  if (!v) return;
  uint32_t o = scan[w];
  const uint32_t base = (uint32_t)(w % per_scan) << 5;
  while (v) {
    const int b = __ffs(v) - 1;
    list[o++] = base + (uint32_t)b;
    v &= v - 1;
  }
}

// ---- sicp_map_insert: one new point per voxel the map does not occupy ----------------------
// key(p) = (floor(p.x / v), floor(p.y / v), floor(p.z / v)) with IEEE double division, compared
// as doubles.  Only records inside the box of p's voxel can share its key:
//   a point q with key k on an axis has fl(q / v) in [k, k + 1) (fl(q / v) = k when |k| >= 2^53,
//   where k + 1 rounds to k).  Division is correctly rounded, so q / v lies within u|k + 1| + u|k|
//   + 2^-1075 of [k, k + 1] (u = 2^-53; the last term covers a quotient in the subnormal range),
//   i.e. q lies in [k v, (k + 1) v] grown by u (|k| + |k + 1|) v + v 2^-1075.  The computed faces
//   lo = k v and hi = (k + 1) v are each within u of their value, plus 2^-1075 below the normal
//   range, and |lo| + |hi| >= (1 - 2u) v while both are finite.  So the box [lo, hi] grown by
//   4u (|lo| + |hi|) + 2^-1072 holds every such q; the kernel grows it by
//   g = 1e-12 (|lo| + |hi|) + 1e-300, over a thousand times more.  A face that overflows (or
//   inf - inf) opens that axis to the whole line.
// The cells are the grid's own cell_coord of the grown faces: a rounded product, a floor and a
// clamp are each monotone, and the builder binned every record with the same cell_coord, so a
// record inside the box lies in a cell between those of the faces (also when they clamp: a box
// beyond the grid only walks its edge cells, whose records then fail the key test).  In a cubic
// x-fastest grid each (y, z) row of that range is one contiguous range of records.
__device__ __forceinline__ bool voxel_taken(const GridView& g, const double lo[3], const double hi[3], double v,
                                            const double k[3], long long below) {
  const int x0 = cell_coord(lo[0], g.ox, g.inv_h, g.nx), x1 = cell_coord(hi[0], g.ox, g.inv_h, g.nx);
  const int y0 = cell_coord(lo[1], g.oy, g.inv_h, g.ny), y1 = cell_coord(hi[1], g.oy, g.inv_h, g.ny);
  const int z0 = cell_coord(lo[2], g.oz, g.inv_h, g.nz), z1 = cell_coord(hi[2], g.oz, g.inv_h, g.nz);
  for (int z = z0; z <= z1; ++z)
    for (int y = y0; y <= y1; ++y) {
      const long long row = ((long long)z * g.ny + y) * g.nx;
      const uint32_t e = g.cell_start[row + x1 + 1];
      for (uint32_t p = g.cell_start[row + x0]; p < e; ++p) {
        const Rec r = g.recs[p];
        if (r.idx >= below || r.x < lo[0] || r.x > hi[0] || r.y < lo[1] || r.y > hi[1] || r.z < lo[2] || r.z > hi[2])
          continue;
        if (floor(__ddiv_rn(r.x, v)) == k[0] && floor(__ddiv_rn(r.y, v)) == k[1] && floor(__ddiv_rn(r.z, v)) == k[2])
          return true;
      }
    }
  return false;
}

// The voxel key k of point p (three doubles) and the grown box [lo, hi] of its voxel, as above.
__device__ __forceinline__ void voxel_box(const double* __restrict__ p, double v, double k[3], double lo[3],
                                          double hi[3]) {
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    k[a] = floor(__ddiv_rn(p[a], v));
    const double l = k[a] * v, h = (k[a] + 1.0) * v;
    const double g = 1e-12 * (fabs(l) + fabs(h)) + 1e-300;
    lo[a] = l - g;
    hi[a] = h + g;
    if (!(lo[a] >= -DBL_MAX)) lo[a] = -kInf;  // overflow or NaN
    if (!(hi[a] <= DBL_MAX)) hi[a] = kInf;
  }
}

// One thread per finite new point f (fin_xyz, the compacted points gridded in `fresh`, Rec::idx =
// f): it is added unless a map record has its key or a fresh record with a smaller index does.
__global__ void __launch_bounds__(256)
    k_map_insert_flags(GridView map, GridView fresh, const double* __restrict__ fin_xyz,
                       const uint32_t* __restrict__ fin_idx, long long n_fin, double v, uint32_t* __restrict__ flag) {
  const long long f = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (f >= n_fin) return;
  double k[3], lo[3], hi[3];
  voxel_box(fin_xyz + 3 * f, v, k, lo, hi);
  if (voxel_taken(map, lo, hi, v, k, LLONG_MAX) || voxel_taken(fresh, lo, hi, v, k, f)) return;
  flag[fin_idx[f]] = 1u;
}

// ---- sicp_map_thin: one map point per voxel -------------------------------------------------
// One thread per map point j (xyz in map order, gridded in `map`, Rec::idx = j): keep[j] = 1 iff no
// map point with a smaller index has its key (the grid builder admits finite points only).
__global__ void __launch_bounds__(256)
    k_map_thin_flags(GridView map, const double* __restrict__ xyz, long long n, double v, uint32_t* __restrict__ keep) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= n) return;
  double k[3], lo[3], hi[3];
  voxel_box(xyz + 3 * j, v, k, lo, hi);
  keep[j] = voxel_taken(map, lo, hi, v, k, j) ? 0u : 1u;
}

// ---- sicp_map_carve: the map points the rays of clouds pass ---------------------------------
// Point j of xyz (cloud i = the last with off[i] <= j, finite after the move) is the ray (o, p)
// from o = origins[i].  For a map record m, with every operation rounded on its own:
//   d = p - o, u = m - o, L2 = (dx dx + dy dy) + dz dz, L = sqrt(L2),
//   s = ((ux dx + uy dy) + uz dz) / L, e2 = ((ux ux + uy uy) + uz uz) - s s,
//   m is passed iff L2 > 0, L2 finite, s > 0, s < L - margin and e2 < r2 (= fl(r r), host).
// Coverage.  Take the exact segment S from o to o + (L - margin) / L (p - o).  The computed u and
// d are within u_r |u| and u_r |d| of the exact ones (u_r = 2^-53); the three-term sums, the root
// and the division add a few u_r each, so s and e2 are within 8 u_r |u| and 8 u_r |u|^2 of the
// exact projection and squared line distance.  A passed m therefore lies within
// r + sqrt(8 u_r) |u| + 16 u_r (|u| + L) < r + 4e-8 (L + r) of S (|u| < L + r + tiny for a passed
// m).  The walk grows that tube to R = r + 1e-6 (L + r) + 1e-12 A, where A bounds the magnitude of
// every coordinate the walk computes (the endpoints' and the grid box's): each face, end and
// segment coordinate below is a few rounded operations on such numbers, so it moves by less than
// 1e-15 A + 1e-15 (L + r), far inside the slack, also at UTM-scale coordinates.
// Cells are the grid's own cell_coord of the grown faces, monotone and clamping as in voxel_taken,
// so a record whose coordinate lies between two faces lies in a cell between theirs.
//  1. Clip: every record lies in the grid's box, so the foot point of a passed m on S lies in that
//     box grown by R on every axis; S is clipped to it (t in [t0, t1] of o + t d).
//  2. Layers: on the major axis a of d (|d_a| largest), layer i holds the records with
//     cell_coord(m_a) = i, whose m_a lies in [g.o_a + i h, g.o_a + (i + 1) h] grown by 1e-12 A
//     (open below the first layer and above the last, where cell_coord clamps).  A passed m in
//     layer i has its foot point within R of that slab on axis a: the part of S there is one
//     t-interval, and its extent on the other two axes grown by R bounds m's cells there.
//  3. Each cell at most once per ray: layers partition axis a, and a layer's (b, c) box lists
//     each cell once, walked as contiguous x-rows like voxel_taken.  So passes counts rays.
// One thread per ray: on the probe of DESIGN §6.8 it was faster than groups of 4 or 8 lanes that
// split each row's records.
__global__ void __launch_bounds__(256)
    k_map_carve(GridView g, const double* __restrict__ xyz, long long n, const uint32_t* __restrict__ off,
                int n_clouds, const double* __restrict__ origins, double r, double r2, double margin,
                uint32_t* __restrict__ passes) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double p[3] = {xyz[3 * j + 0], xyz[3 * j + 1], xyz[3 * j + 2]};
  if (!(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]))) return;
  int lo = 0, hi = n_clouds;  // off[lo] <= j < off[hi], as k_insert_stage
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (off[mid] <= (unsigned long long)j) lo = mid;
    else hi = mid;
  }
  const double o[3] = {origins[3 * lo + 0], origins[3 * lo + 1], origins[3 * lo + 2]};
  const double d[3] = {__dsub_rn(p[0], o[0]), __dsub_rn(p[1], o[1]), __dsub_rn(p[2], o[2])};
  const double L2 = __dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2]));
  if (!(L2 > 0.0 && L2 <= DBL_MAX)) return;  // zero-length or overflowing ray
  const double L = __dsqrt_rn(L2);
  const double Lm = __dsub_rn(L, margin);
  if (!(Lm > 0.0)) return;  // s > 0 and s < L - margin cannot both hold

  const double gn[3] = {(double)g.nx, (double)g.ny, (double)g.nz}, go[3] = {g.ox, g.oy, g.oz};
  double A = 0.0;
#pragma unroll
  for (int a = 0; a < 3; ++a) A = fmax(A, fabs(o[a]) + fabs(p[a]) + fabs(go[a]) + gn[a] * g.h);
  const double slack = 1e-12 * A + 1e-300;
  const double R = r + 1e-6 * (L + r) + slack;
  // 1. clip S (t in [0, Lm / L]) to the grid's box grown by R
  double t0 = 0.0, t1 = fmin(1.0, Lm / L);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double blo = go[a] - R, bhi = go[a] + gn[a] * g.h + R;
    if (d[a] == 0.0) {
      if (o[a] < blo || o[a] > bhi) return;
    } else {
      const double ta = (blo - o[a]) / d[a], tb = (bhi - o[a]) / d[a];
      t0 = fmax(t0, fmin(ta, tb));
      t1 = fmin(t1, fmax(ta, tb));
    }
  }
  if (!(t0 <= t1)) return;  // the ray misses the grown box
  // 2. layers on the major axis (selected without indexing the arrays, which stay in registers)
  const int a = (fabs(d[1]) > fabs(d[0])) ? ((fabs(d[2]) > fabs(d[1])) ? 2 : 1) : ((fabs(d[2]) > fabs(d[0])) ? 2 : 0);
  const int gi[3] = {g.nx, g.ny, g.nz};
  const double oa = (a == 0) ? o[0] : ((a == 1) ? o[1] : o[2]);
  const double da = (a == 0) ? d[0] : ((a == 1) ? d[1] : d[2]);
  const double goa = (a == 0) ? go[0] : ((a == 1) ? go[1] : go[2]);
  const int na = (a == 0) ? gi[0] : ((a == 1) ? gi[1] : gi[2]);
  const double ida = 1.0 / da;
  const double sa0 = oa + t0 * da, sa1 = oa + t1 * da;
  const int i0 = cell_coord(fmin(sa0, sa1) - R, goa, g.inv_h, na);
  const int i1 = cell_coord(fmax(sa0, sa1) + R, goa, g.inv_h, na);
  for (int i = i0; i <= i1; ++i) {
    const double f0 = (i == 0) ? -kInf : goa + i * g.h - slack - R;
    const double f1 = (i == na - 1) ? kInf : goa + (i + 1) * g.h + slack + R;
    const double ta = (f0 - oa) * ida, tb = (f1 - oa) * ida;
    const double tl = fmax(t0, fmin(ta, tb)), th = fmin(t1, fmax(ta, tb));
    if (!(tl <= th)) continue;
    int cl[3], ch[3];  // the layer's cell box: [i, i] on axis a, the grown extent of S's part on the others
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double e0 = o[k] + tl * d[k], e1 = o[k] + th * d[k];
      cl[k] = (k == a) ? i : cell_coord(fmin(e0, e1) - R, go[k], g.inv_h, gi[k]);
      ch[k] = (k == a) ? i : cell_coord(fmax(e0, e1) + R, go[k], g.inv_h, gi[k]);
    }
    // 3. the layer's cells, as contiguous x-rows
    for (int z = cl[2]; z <= ch[2]; ++z)
      for (int y = cl[1]; y <= ch[1]; ++y) {
        const long long row = ((long long)z * g.ny + y) * g.nx;
        const uint32_t e = g.cell_start[row + ch[0] + 1];
        for (uint32_t q = g.cell_start[row + cl[0]]; q < e; ++q) {
          const Rec m = g.recs[q];
          const double ux = __dsub_rn(m.x, o[0]), uy = __dsub_rn(m.y, o[1]), uz = __dsub_rn(m.z, o[2]);
          const double s =
              __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(ux, d[0]), __dmul_rn(uy, d[1])), __dmul_rn(uz, d[2])), L);
          if (!(s > 0.0 && s < Lm)) continue;
          const double e2 = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), __dmul_rn(uz, uz)),
                                      __dmul_rn(s, s));
          if (e2 < r2) atomicAdd(&passes[m.idx], 1u);
        }
      }
  }
}

// ---- sicp_map_distances: the nearest map point of a point, within a bound --------------------
// MG lanes per point run grid_nn's ring expansion with the rows of each ring dealt over the lanes
// and reduced after the ring.  guard is the distance from the point to the nearest face behind
// which unexplored cells remain, less 1e-9 h (cell assignment rounds at the 1e-13 level), so every
// unexplored point lies farther than guard.  The search stops when
//   best <= guard^2   the best point is the nearest, ties included, or
//   guard^2 >= cap2   no unexplored point is within the bound: whether the nearest is within is
//                     decided by best alone (best < cap2 <= guard^2 is the first case).
// The first is grid_nn's rule; the second replaces its cap2 stop at the first point under the
// bound, which answers only yes or no.  A row is skipped when its distance to the point, less the
// same margin, exceeds min(best, cap2) (1e-12 relative slack): it holds nothing nearer than the
// lane's best, which bounds the group's, and nothing within the bound.
template <int MG>
__global__ void __launch_bounds__(128)
    k_map_nearest(GridView g, const double* __restrict__ xyz, long long n, double cap2, long long* __restrict__ idx,
                  double* __restrict__ d2, uint32_t* __restrict__ within) {
  const long long j = (blockIdx.x * (long long)blockDim.x + threadIdx.x) / MG;
  const int sub = threadIdx.x & (MG - 1);
  if (j >= n) return;  // a whole group leaves together
  const unsigned int gmask = ((1u << MG) - 1u) << ((threadIdx.x & 31) & ~(MG - 1));
  const double qx = xyz[3 * j + 0], qy = xyz[3 * j + 1], qz = xyz[3 * j + 2];
  if (!(isfinite(qx) && isfinite(qy) && isfinite(qz))) {
    if (sub == 0) {
      idx[j] = -1;
      d2[j] = __longlong_as_double(0x7ff8000000000000ll);
      within[j] = 0u;
    }
    return;
  }
  const int cx = cell_coord(qx, g.ox, g.inv_h, g.nx);
  const int cy = cell_coord(qy, g.oy, g.inv_h, g.ny);
  const int cz = cell_coord(qz, g.oz, g.inv_h, g.nz);
  const uint32_t* __restrict__ cs = g.cell_start;
  const double marg = 1e-9 * g.h;
  double best = kInf;
  long long bidx = -1;
  uint32_t bpos = 0;
  // r stays below the grid's largest dimension: once the ring's block covers the grid, guard is inf
  for (int r = 1;; ++r) {
    const int x0 = cx - r, x1 = cx + r, y0 = cy - r, y1 = cy + r, z0 = cz - r, z1 = cz + r;
    const int xa = max(x0, 0), xb = min(x1, g.nx - 1);
    // the ring's (y, z) rows clamped to the grid: at most ny nz < 2^25 of them
    const int ya = max(y0, 0), yb = min(y1, g.ny - 1), za = max(z0, 0), zb = min(z1, g.nz - 1);
    const int nyr = yb - ya + 1, items = nyr * (zb - za + 1);
    int zr = sub / nyr, yr = sub - zr * nyr;
    for (int t = sub; t < items; t += MG, yr += MG) {
      while (yr >= nyr) {
        yr -= nyr;
        ++zr;
      }
      const int y = ya + yr, z = za + zr;
      const double by = fmax(fmax((g.oy + y * g.h) - qy, qy - (g.oy + (y + 1) * g.h)) - marg, 0.0);
      const double bz = fmax(fmax((g.oz + z * g.h) - qz, qz - (g.oz + (z + 1) * g.h)) - marg, 0.0);
      if (by * by + bz * bz > fmin(best, cap2) * (1.0 + 1e-12)) continue;
      const long long row = ((long long)z * g.ny + y) * g.nx;
      if (r == 1 || y == y0 || y == y1 || z == z0 || z == z1) {
        scan_range(g.recs, cs[row + xa], cs[row + xb + 1], qx, qy, qz, best, bidx, bpos);
      } else {
        if (x0 >= 0) scan_range(g.recs, cs[row + x0], cs[row + x0 + 1], qx, qy, qz, best, bidx, bpos);
        if (x1 < g.nx) scan_range(g.recs, cs[row + x1], cs[row + x1 + 1], qx, qy, qz, best, bidx, bpos);
      }
    }
#pragma unroll
    for (int o = MG / 2; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(gmask, best, o, MG);
      const long long oi = __shfl_xor_sync(gmask, bidx, o, MG);
      if (od < best || (od == best && oi >= 0 && (bidx < 0 || oi < bidx))) {
        best = od;
        bidx = oi;
      }
    }
    double guard = kInf;
    if (x0 > 0) guard = fmin(guard, qx - (g.ox + x0 * g.h));
    if (x1 < g.nx - 1) guard = fmin(guard, (g.ox + (x1 + 1) * g.h) - qx);
    if (y0 > 0) guard = fmin(guard, qy - (g.oy + y0 * g.h));
    if (y1 < g.ny - 1) guard = fmin(guard, (g.oy + (y1 + 1) * g.h) - qy);
    if (z0 > 0) guard = fmin(guard, qz - (g.oz + z0 * g.h));
    if (z1 < g.nz - 1) guard = fmin(guard, (g.oz + (z1 + 1) * g.h) - qz);
    if (guard >= kInf) break;  // the block covers the whole grid
    guard -= marg;
    if (guard > 0.0 && (best <= guard * guard || guard * guard >= cap2)) break;
  }
  if (sub != 0) return;
  const bool in = best < cap2;  // strict: cKDTree distance_upper_bound semantics, as k_range_keep
  idx[j] = in ? bidx : -1;
  d2[j] = in ? best : kInf;
  within[j] = in ? 1u : 0u;
}

// ------------------------------------------------------------------------------------------
// brute-force engine (TMA staged)
// ------------------------------------------------------------------------------------------
constexpr int BF_TILE = kBfTile;  // float4 points per stage = 32 KB
constexpr int BF_STAGES = 3;    // 96 KB of shared memory in flight per block, two blocks per SM
constexpr int BF_THREADS = 256; // 8 warps
constexpr int BF_QPW = 8;       // queries per warp
constexpr int BF_QPB = BF_QPW * (BF_THREADS / 32);

struct BfPartial {
  double d2;
  long long idx;
};

// float32 filter margin.  Centred float32 coordinates carry a per-coordinate error
// eta <= 2^-23 (|a|_inf + R) * 1.5 (a = centred query, R = cloud half-extent); the float32
// squared distance then differs from the true one by at most e(d) = 4 eta sqrt(d) + 1e-6 d +
// 4 eta^2.  A point is re-evaluated in float64 iff d32 <= best32 + 2.5 e(best32), which the
// true nearest neighbour always satisfies.  The threshold is evaluated in float32 with its
// constants rounded up (cA = 10 eta, cC = 10 eta^2, 4e-6 >= 2.5e-6 + rounding).
__device__ __forceinline__ float bf_threshold(float best32, float cA, float cC) {
  return fmaf(cA, sqrtf(best32), fmaf(4.0e-6f, best32, best32)) + cC;
}

__global__ void __launch_bounds__(BF_THREADS, 2)
    k_bf_nn(const float4* __restrict__ mov_f4, const double* __restrict__ mov_xyz, long long n_mov,
            long long n_pad, double cx, double cy, double cz, double radius,
            const DevState* __restrict__ st,
            const double* __restrict__ q_xyz, const unsigned int* __restrict__ qlist,
            const unsigned int* __restrict__ qcount_ptr, long long q_total, int tiles_per_chunk,
            BfPartial* __restrict__ partials) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float4* tiles = reinterpret_cast<float4*>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)BF_STAGES * BF_TILE * sizeof(float4));
  uint64_t* empty = full + BF_STAGES;
  double* q64 = reinterpret_cast<double*>(empty + BF_STAGES);  // BF_QPB x 3

  const long long nq = qlist ? (long long)(*qcount_ptr) : q_total;
  const long long n_groups = (nq + BF_QPB - 1) / BF_QPB;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long n_tiles = n_pad / BF_TILE;
  const long long tile0 = (long long)blockIdx.y * tiles_per_chunk;
  const long long tile1 = min(tile0 + tiles_per_chunk, n_tiles);
  if (tile0 >= tile1 || n_groups == 0 || st->stop) return;
  const int my_tiles = (int)(tile1 - tile0);
  const Rigid Tinv = st->Tinv;

  if (threadIdx.x == 0) {
    for (int s = 0; s < BF_STAGES; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], BF_THREADS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  uint32_t it_base = 0;  // tiles consumed so far by this block (across query groups)
  for (long long grp = blockIdx.x; grp < n_groups; grp += gridDim.x) {
    // ---- queries of this warp: move into the movable frame, centre, round to float32
    float ax[BF_QPW], ay[BF_QPW], az[BF_QPW], best32[BF_QPW], thr[BF_QPW], cA[BF_QPW], cC[BF_QPW];
    double best64[BF_QPW];
    int bidx[BF_QPW];
#pragma unroll
    for (int k = 0; k < BF_QPW; ++k) {
      const long long qi = grp * BF_QPB + warp * BF_QPW + k;
      double mx = 0, my = 0, mz = 0;
      if (qi < nq) {
        const long long q = qlist ? (long long)qlist[qi] : qi;
        rigid_apply(Tinv, q_xyz[3 * q + 0], q_xyz[3 * q + 1], q_xyz[3 * q + 2], mx, my, mz);
      }
      if (lane == 0) {
        q64[(warp * BF_QPW + k) * 3 + 0] = mx;
        q64[(warp * BF_QPW + k) * 3 + 1] = my;
        q64[(warp * BF_QPW + k) * 3 + 2] = mz;
      }
      const double a0 = mx - cx, a1 = my - cy, a2 = mz - cz;
      ax[k] = (float)a0;
      ay[k] = (float)a1;
      az[k] = (float)a2;
      const double eta = 1.1920929e-7 * (fmax(fabs(a0), fmax(fabs(a1), fabs(a2))) + radius) * 1.5;
      cA[k] = nextafterf((float)(10.0 * eta), 3.0e38f);
      cC[k] = nextafterf((float)(10.0 * eta * eta), 3.0e38f);
      best32[k] = 3.0e38f;
      thr[k] = 3.0e38f;
      best64[k] = kInf;
      bidx[k] = -1;
    }
    __syncwarp();

    // ---- producer prologue: fill the ring
    if (threadIdx.x == 0) {
      for (int t = 0; t < min(BF_STAGES, my_tiles); ++t) {
        const uint32_t g_it = it_base + t;
        const int s = g_it % BF_STAGES;
        if (g_it >= BF_STAGES) mbar_wait(&empty[s], ((g_it / BF_STAGES) - 1) & 1);
        mbar_expect_tx(&full[s], BF_TILE * sizeof(float4));
        tma_load_1d(tiles + (size_t)s * BF_TILE, mov_f4 + (tile0 + t) * BF_TILE,
                    BF_TILE * sizeof(float4), &full[s]);
      }
    }

    for (int t = 0; t < my_tiles; ++t) {
      const uint32_t g_it = it_base + t;
      const int s = g_it % BF_STAGES;
      mbar_wait(&full[s], (g_it / BF_STAGES) & 1);
      const float4* __restrict__ tp = tiles + (size_t)s * BF_TILE;
      const long long base = (tile0 + t) * BF_TILE;
      unsigned int improved = 0;  // bit k: this lane lowered best32[k] in this tile
#pragma unroll 2
      for (int j = lane; j < BF_TILE; j += 32) {
        const float4 p = tp[j];  // conflict-free LDS.128
        float dk[BF_QPW];
        bool hit = false;
#pragma unroll
        for (int k = 0; k < BF_QPW; ++k) {
          const float dx = p.x - ax[k], dy = p.y - ay[k], dz = p.z - az[k];
          dk[k] = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
          hit = hit || (dk[k] <= thr[k]);
        }
        if (__builtin_expect(hit, 0)) {
          // rare: exact float64 re-evaluation from the original coordinates
          const long long gi = base + j;
          if (gi < n_mov) {
            const double gx = mov_xyz[3 * gi + 0], gy = mov_xyz[3 * gi + 1], gz = mov_xyz[3 * gi + 2];
#pragma unroll
            for (int k = 0; k < BF_QPW; ++k) {
              if (dk[k] <= thr[k]) {
                const double* qq = &q64[(warp * BF_QPW + k) * 3];
                const double ex = gx - qq[0], ey = gy - qq[1], ez = gz - qq[2];
                const double d64 = ex * ex + ey * ey + ez * ez;
                if (d64 < best64[k] || (d64 == best64[k] && (int)gi < bidx[k])) {
                  best64[k] = d64;
                  bidx[k] = (int)gi;
                }
                if (dk[k] < best32[k]) {
                  best32[k] = dk[k];
                  thr[k] = bf_threshold(dk[k], cA[k], cC[k]);
                  improved |= 1u << k;
                }
              }
            }
          }
        }
      }
      // share the float32 bound across the warp, but only for the queries some lane improved in
      // this tile (after the first tiles that is almost never)
      unsigned int any = improved;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) any |= __shfl_xor_sync(0xffffffffu, any, o);
      if (any) {
#pragma unroll
        for (int k = 0; k < BF_QPW; ++k) {
          if (any & (1u << k)) {
            float m = best32[k];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
            if (m < best32[k]) {
              best32[k] = m;
              thr[k] = bf_threshold(m, cA[k], cC[k]);
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      // producer: refill this stage with tile t + BF_STAGES once every warp has released it
      if (threadIdx.x == 0 && t + BF_STAGES < my_tiles) {
        mbar_wait(&empty[s], (g_it / BF_STAGES) & 1);
        mbar_expect_tx(&full[s], BF_TILE * sizeof(float4));
        tma_load_1d(tiles + (size_t)s * BF_TILE, mov_f4 + (tile0 + t + BF_STAGES) * BF_TILE,
                    BF_TILE * sizeof(float4), &full[s]);
      }
    }
    it_base += my_tiles;

    // ---- warp-shuffle lexicographic min-reduction of (d64, idx) over the lanes
#pragma unroll
    for (int k = 0; k < BF_QPW; ++k) {
      double d = best64[k];
      int ix = bidx[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, d, o);
        const int oi = __shfl_xor_sync(0xffffffffu, ix, o);
        if (od < d || (od == d && oi >= 0 && (ix < 0 || oi < ix))) {
          d = od;
          ix = oi;
        }
      }
      const long long qi = grp * BF_QPB + warp * BF_QPW + k;
      if (lane == 0 && qi < nq) {
        BfPartial pr;
        pr.d2 = d;
        pr.idx = ix;
        partials[(long long)blockIdx.y * q_total + qi] = pr;
      }
    }
    __syncthreads();  // q64 is reused by the next group
  }
}

__global__ void __launch_bounds__(128)
    k_bf_finalize(const BfPartial* __restrict__ partials, int n_chunks, long long q_total,
                  const unsigned int* __restrict__ qlist, const unsigned int* __restrict__ qcount_ptr,
                  const DevState* __restrict__ st, const double* __restrict__ q_xyz,
                  const float4* __restrict__ q_nrm,
                  const double* __restrict__ mov_xyz, int with_distance,
                  long long* __restrict__ nn_idx, double* __restrict__ out,
                  unsigned int* __restrict__ lin_hist, CorrOut co) {
  const long long nq = qlist ? (long long)(*qcount_ptr) : q_total;
  const long long qi = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (qi >= nq || st->stop) return;
  const Rigid T = st->T;
  double d = kInf;
  long long ix = -1;
  for (int c = 0; c < n_chunks; ++c) {
    const BfPartial p = partials[(long long)c * q_total + qi];
    if (p.idx >= 0 && (p.d2 < d || (p.d2 == d && p.idx < ix) || ix < 0)) {
      d = p.d2;
      ix = p.idx;
    }
  }
  const long long q = qlist ? (long long)qlist[qi] : qi;
  nn_idx[q] = ix;
  if (with_distance) {
    const float4 nr = q_nrm[q];
    const double dd = plane_distance(T, mov_xyz, ix, q_xyz[3 * q + 0], q_xyz[3 * q + 1], q_xyz[3 * q + 2], nr);
    out[q] = dd;
    lin_hist_add(st, lin_hist, effective_planarity(co, T, q, ix, nr), dd, co.binstore, co.bin_cap, q);
    store_matched(co, q, mov_xyz[3 * ix + 0], mov_xyz[3 * ix + 1], mov_xyz[3 * ix + 2]);
  } else {
    out[q] = d;
  }
}

__global__ void __launch_bounds__(256)
    k_gather_queries(const double* __restrict__ fix_xyz, const long long* __restrict__ sel,
                     long long K, double* __restrict__ q_xyz) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= K) return;
  const long long j = sel[i];
  q_xyz[3 * i + 0] = fix_xyz[3 * j + 0];
  q_xyz[3 * i + 1] = fix_xyz[3 * j + 1];
  q_xyz[3 * i + 2] = fix_xyz[3 * j + 2];
}

constexpr size_t kBfSmem =
    (size_t)BF_STAGES * BF_TILE * sizeof(float4) + 2 * BF_STAGES * sizeof(uint64_t) +
    (size_t)BF_QPB * 3 * sizeof(double);

}  // namespace

void gather_queries_launch(Ctx& c) {
  c.unresolved_clean = false;  // another K: the counter lives at another address
  c.q_xyz.reserve(3 * std::max<long long>(c.K, 1));
  k_gather_queries<<<(unsigned)((c.K + 255) / 256), 256, 0, c.stream>>>(c.fix_xyz.p, c.sel_idx.p,
                                                                       c.K, c.q_xyz.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

// Slots per histogram bin of the per-bin index store: a few times the mean count of a bin that
// matters (the statistics set spreads over ~2500 of the 4096 bins), so that a distribution which
// narrows several-fold between two iterations still fits; a bin that overflows just sends that
// iteration through the general kernel.
int bin_cap_for(long long K) {
  long long cap = 32;
  while (cap < K / 192 && cap < 2048) cap *= 2;
  return (int)cap;
}
static void reserve_binstore(Ctx& c) {
  c.bin_cap = bin_cap_for(c.K);
  c.binstore.reserve((size_t)LH_BINS * c.bin_cap);
}

// Brute-force pass over either the unresolved list (qlist != nullptr) or all K queries.
static void bf_launch(Ctx& c, bool with_distance, double* out, bool whole_set) {
  if (with_distance) {
    reserve_binstore(c);
    c.m_xyz.reserve(3 * std::max<long long>(c.K, 1));
  }
  // the attribute belongs to the (device-specific) function handle: once per context, not per process
  if (!c.bf_attr_set) {
    SICP_CUDA(cudaFuncSetAttribute(k_bf_nn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBfSmem));
    c.bf_attr_set = true;
  }
  const long long n_tiles = (c.n_mov + BF_TILE - 1) / BF_TILE;
  SICP_REQUIRE(c.mov_f4.cap >= (size_t)n_tiles * BF_TILE, SICP_ERR_STATE,
               "float4 copy not padded to the brute-force tile");
  const long long q_total = c.K;
  // grid: x = query groups (grid-stride), y = point chunks
  long long groups_hint = whole_set ? (c.K + BF_QPB - 1) / BF_QPB : 4;
  int gx = (int)std::min<long long>(std::max<long long>(groups_hint, 1), 4096);
  long long want_blocks = 2ll * c.num_sms;
  int n_chunks = (int)std::min<long long>(std::max<long long>(want_blocks / gx, 1), n_tiles);
  int tiles_per_chunk = (int)((n_tiles + n_chunks - 1) / n_chunks);
  n_chunks = (int)((n_tiles + tiles_per_chunk - 1) / tiles_per_chunk);
  c.bf_scratch.reserve((size_t)n_chunks * q_total * sizeof(BfPartial));
  BfPartial* partials = reinterpret_cast<BfPartial*>(c.bf_scratch.p);
  const unsigned int* qlist = whole_set ? nullptr : c.unresolved.p;
  const unsigned int* qcount = whole_set ? nullptr : c.unresolved.p + c.K;
  dim3 grid(gx, n_chunks);
  k_bf_nn<<<grid, BF_THREADS, kBfSmem, c.stream>>>(
      c.mov_f4.p, c.mov_xyz.p, c.n_mov, n_tiles * BF_TILE, c.mov_center[0], c.mov_center[1],
      c.mov_center[2], c.mov_radius, c.dev_state.p, c.q_xyz.p, qlist, qcount, q_total,
      tiles_per_chunk,
      partials);
  k_bf_finalize<<<(unsigned)((q_total + 127) / 128), 128, 0, c.stream>>>(
      partials, n_chunks, q_total, qlist, qcount, c.dev_state.p, c.q_xyz.p, c.q_nrm.p, c.mov_xyz.p,
      with_distance ? 1 : 0, c.nn_idx.p, out, with_distance ? c.lin_hist.p : nullptr,
      with_distance ? CorrOut{c.binstore.p, c.bin_cap, c.m_xyz.p, nullptr, 0, 0, mov_attr_nrm(c), mov_attr_eff(c), c.mov_cos_max}
                    : CorrOut{nullptr, 0, nullptr, nullptr, 0, 0, nullptr, nullptr, -1.0});
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 2;
}

namespace {
// per pair: sel[i] = src[rint(linspace(0, m - 1, K))] (PointCloud.select_n_points, k_select_n in
// capi.cu) and the gather of the selected fixed points, in one launch for the whole batch.  src is
// the pair's survivor list of the overlap filter (m = its length; its entries are flag positions
// flag_off + index) or, without a list, the whole cloud (m = n_fix, src = identity).
__global__ void __launch_bounds__(256)
    k_select_gather_batch(const PairDev* __restrict__ pairs, const double* __restrict__ fix_xyz,
                          const uint32_t* __restrict__ list, int away, long long* __restrict__ sel,
                          double* __restrict__ q_xyz) {
  const PairDev pd = pairs[blockIdx.y];
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= pd.K) return;
  const long long m = list ? pd.list_len : pd.n_fix, n = pd.K;
  long long j = i;
  if (n < m) {
    const double step = (n > 1) ? (double)(m - 1) / (double)(n - 1) : 0.0;
    const double y = (i == n - 1 && n > 1) ? (double)(m - 1) : (double)i * step;
    j = (long long)(away ? round(y) : rint(y));
  }
  if (list) j = (long long)list[pd.list_off + j] - pd.flag_off;
  sel[pd.q_off + i] = j;
  const double* __restrict__ src = fix_xyz + 3 * (pd.fix_off + j);
  double* __restrict__ dst = q_xyz + 3 * (pd.q_off + i);
  dst[0] = src[0];
  dst[1] = src[1];
  dst[2] = src[2];
}

// Lanes per query of the grid match family: option match_group when it names a lane count, else
// by the number n_q of queries in flight -- 16 while the search is latency-bound (few queries),
// fewer once there are enough queries to fill the machine and issue slots become the limit.  A
// family without the forms below min_lanes (they would spill) runs min_lanes; the results do not
// depend on the lanes.
int match_lanes(const Ctx& c, long long n_q, int min_lanes) {
  const int mg = (c.match_group > 1) ? c.match_group : ((n_q <= 16384) ? 16 : ((n_q <= 65536) ? 8 : 4));
  return std::max(mg, min_lanes);
}

// launch(std::integral_constant<int, L>{}) for the form L == lanes among the forms Ls of a family
template <int... Ls, class F>
void with_lanes(int lanes, F&& launch) {
  const bool found = ((lanes == Ls && (launch(std::integral_constant<int, Ls>{}), true)) || ...);
  SICP_REQUIRE(found, SICP_ERR_BAD_ARG, "no " + std::to_string(lanes) + "-lane match kernel");
}
}  // namespace

void batch_select_gather_launch(Ctx& c, Batch& b, const double* fix_xyz, bool with_list, int round_away) {
  k_select_gather_batch<<<dim3((unsigned)((b.Kmax + 255) / 256), b.n_pairs), 256, 0, c.stream>>>(
      b.pairs.p, fix_xyz, with_list ? b.ovl_list.p : nullptr, round_away, b.sel_idx.p, b.q_xyz.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void batch_overlap_launch(Ctx& c, Batch& b, const double* fix_xyz, long long max_n_fix, double r2) {
  const int mg = match_lanes(c, b.total_fix, 4);
  const dim3 grid((unsigned)((max_n_fix * mg + 127) / 128), b.n_pairs);
  with_lanes<4, 8, 16>(mg, [&](auto L) {
    k_overlap_batch<decltype(L)::value>
        <<<grid, 128, 0, c.stream>>>(b.pairs.p, b.state.p, fix_xyz, r2, c.compact.flag.p);
  });
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void map_overlap_launch(Ctx& c, Batch& b, MapStore& m, const MapCull* culls_dev, long long max_rows, double r2,
                        long long n_candidates_hint) {
  const dim3 grid((unsigned)max_rows, b.n_pairs);
  const long long words = (m.n + 31) / 32;
  with_lanes<4, 8, 16>(match_lanes(c, n_candidates_hint, 4), [&](auto L) {
    k_map_overlap<decltype(L)::value>
        <<<grid, 128, 0, c.stream>>>(b.pairs.p, b.state.p, culls_dev, m.view, r2, words, m.bits.p, m.n_searched.p);
  });
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void overlap_count_launch(Ctx& c, const GridView* views, const DevState* state, const OverlapDir* dirs, int n_dirs,
                          long long max_rows, long long stride, double r2, uint32_t* counts, long long n_candidates) {
  const uint32_t s32 = (uint32_t)std::min<long long>(stride, 0xffffffffll);
  with_lanes<8, 16>(match_lanes(c, n_candidates, 8), [&](auto L) {
    k_overlap_count<decltype(L)::value><<<dim3((unsigned)max_rows, (unsigned)n_dirs), 128, 0, c.stream>>>(
        views, state, dirs, s32, r2, counts);
  });
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void map_bits_popc_launch(Ctx& c, const uint32_t* bits, long long n_words, uint32_t* popc) {
  k_map_popc<<<(unsigned)((n_words + 255) / 256), 256, 0, c.stream>>>(bits, n_words, popc);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void map_bits_scatter_launch(Ctx& c, const uint32_t* bits, long long n_words, long long words_per_scan,
                             const uint32_t* scan, uint32_t* list) {
  k_map_scatter<<<(unsigned)((n_words + 255) / 256), 256, 0, c.stream>>>(bits, n_words, words_per_scan, scan, list);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void map_insert_flags_launch(Ctx& c, const GridView& map, const GridView& fresh, const double* fin_xyz,
                             const uint32_t* fin_idx, long long n_fin, double voxel, uint32_t* flag) {
  if (n_fin <= 0) return;
  k_map_insert_flags<<<(unsigned)((n_fin + 255) / 256), 256, 0, c.stream>>>(map, fresh, fin_xyz, fin_idx, n_fin, voxel,
                                                                            flag);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void map_thin_flags_launch(Ctx& c, const GridView& map, const double* xyz, long long n, double voxel, uint32_t* keep) {
  if (n <= 0) return;
  k_map_thin_flags<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(map, xyz, n, voxel, keep);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void map_carve_launch(Ctx& c, const GridView& map, const double* xyz, long long n, const uint32_t* off, int n_clouds,
                      const double* origins, double r, double r2, double margin, uint32_t* passes) {
  if (n <= 0) return;
  k_map_carve<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(map, xyz, n, off, n_clouds, origins, r, r2, margin,
                                                                 passes);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

// Lanes per point by the point count, the rule of match_lanes without its option: 16 while the
// search is latency-bound (few points), fewer once the points fill the machine.  The result does
// not depend on the lanes.
void map_nearest_launch(Ctx& c, const GridView& map, const double* xyz, long long n, double cap2, long long* idx,
                        double* d2, uint32_t* within) {
  if (n <= 0) return;
  const int mg = (n <= 16384) ? 16 : ((n <= 65536) ? 8 : 4);
  with_lanes<4, 8, 16>(mg, [&](auto L) {
    constexpr int M = decltype(L)::value;
    k_map_nearest<M><<<(unsigned)((n * M + 127) / 128), 128, 0, c.stream>>>(map, xyz, n, cap2, idx, d2, within);
  });
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void batch_match_launch(Ctx& c, Batch& b, bool warm) {
  BatchMatchArgs a;
  a.pairs = b.pairs.p;
  a.state = b.state.p;
  a.q_xyz = b.q_xyz.p;
  a.q_nrm = b.q_nrm.p;
  a.nn_idx = b.nn_idx.p;
  a.dist = b.dist.p;
  a.lin_hist = b.lin_hist.p;
  a.binstore = b.binstore.p;
  a.bin_cap = b.bin_cap;
  a.m_xyz = b.m_xyz.p;
  a.nn_pos = b.nn_pos.p;
  a.warm = warm ? 1 : 0;
  a.sphere = c.sphere_scan;
  const int mg = match_lanes(c, b.Kmax * b.n_pairs, b.mov_attr ? 4 : 2);
  const dim3 grid((unsigned)((b.Kmax * mg + 127) / 128), b.n_pairs);
  // programmatically dependent on the previous iteration's k_rs_batch (both kernels wait before
  // they touch anything the other writes; the pair descriptors are static)
  const bool pdl = c.pdl != 0;
  if (b.mov_attr) {
    const BatchMatchAttrArgs m{a, b.mov_nrm.p, b.q_nrm_eff.p, b.mov_cos_max};
    with_lanes<4, 8, 16>(mg, [&](auto L) {
      launch_kernel(k_match_batch_attr<decltype(L)::value>, grid, dim3(128), 0, c.stream, pdl, m);
    });
  } else {
    with_lanes<2, 4, 8, 16>(mg, [&](auto L) {
      launch_kernel(k_match_batch<decltype(L)::value>, grid, dim3(128), 0, c.stream, pdl, a);
    });
  }
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void match_launch(Ctx& c, bool with_distance, double* out_d2, cudaEvent_t mid, bool allow_bf, double cap2, bool in_loop) {
  const long long K = c.K;
  // predictor histogram for the reject kernel: zero it if an earlier match filled it and no
  // reject consumed it (the reject kernel itself leaves it zeroed)
  c.lin_hist.reserve(LH_BINS + 2);
  if (with_distance && (c.lin_hist_pending || !c.lin_hist_init)) {
    SICP_CUDA(cudaMemsetAsync(c.lin_hist.p, 0, (LH_BINS + 2) * sizeof(unsigned int), c.stream));
    c.lin_hist_init = true;
  }
  unsigned int* lh = with_distance ? c.lin_hist.p : nullptr;
  c.nn_idx.reserve(K);
  c.dist.reserve(K);
  c.unresolved.reserve(K + 1);
  reserve_binstore(c);
  c.m_xyz.reserve(3 * std::max<long long>(K, 1));
  c.nn_pos.reserve(std::max<long long>(K, 1));
  c.cert_c.reserve(3 * std::max<long long>(K, 1));
  c.cert_rho.reserve(std::max<long long>(K, 1));
  if (c.cert_count.p == nullptr) {
    c.cert_count.reserve(2);
    SICP_CUDA(cudaMemsetAsync(c.cert_count.p, 0, 2 * sizeof(unsigned int), c.stream));
  }
  const bool warm = with_distance && c.warm_start && c.nn_pos_valid && c.nn_pos_K == K;
  const CorrOut co = with_distance ? CorrOut{c.binstore.p, c.bin_cap, c.m_xyz.p, c.nn_pos.p, warm ? 1 : 0, c.sphere_scan,
                                             mov_attr_nrm(c), mov_attr_eff(c), c.mov_cos_max}
                                   : CorrOut{nullptr, 0, nullptr, nullptr, 0, 0, nullptr, nullptr, -1.0};
  // A match without distance overwrites nn_idx, which the certificates of the next warm match
  // keep: it ends the warm-start state like a new selection does.
  c.nn_pos_valid = with_distance && (c.nn_engine != SICP_NN_BRUTE) && c.match_group != 1;
  if (with_distance) c.nn_pos_K = K;
  c.cert_slot = -1;
  double* out = with_distance ? c.dist.p : out_d2;
  if (c.nn_engine == SICP_NN_BRUTE) {
    bf_launch(c, with_distance, out, true);
    if (mid) SICP_CUDA(cudaEventRecord(mid, c.stream));
    if (with_distance) c.lin_hist_pending = true;
    return;
  }
  if (!(in_loop && c.unresolved_clean))
    SICP_CUDA(cudaMemsetAsync(c.unresolved.p + K, 0, sizeof(unsigned int), c.stream));
  c.unresolved_clean = false;  // the caller's reject/solve launch declares it clean again
  const bool pdl = in_loop && c.pdl;
  const bool use_bf = (c.nn_engine == SICP_NN_AUTO) && allow_bf;
  const int rmax = use_bf ? c.grid_max_rings : (1 << 30);
  if (c.match_group == 1) {
    k_match_grid<<<(unsigned)((K + 127) / 128), 128, 0, c.stream>>>(
        c.gmov.view, c.dev_state.p, c.q_xyz.p, c.q_nrm.p, c.mov_xyz.p, K, rmax,
        with_distance ? 1 : 0, c.nn_idx.p, out, c.unresolved.p, lh, cap2, co);
  } else {
    // every match with distance writes the certificate of each query it searches (none where it
    // cannot prove one), so they are valid wherever nn_pos is; the launch counts into one of the
    // two counters and zeroes the other for the next
    MatchCert cert{nullptr, nullptr, nullptr, nullptr};
    if (with_distance) {
      c.cert_slot = c.cert_next;
      c.cert_next ^= 1;
      cert = MatchCert{c.cert_c.p, c.cert_rho.p, c.cert_count.p + c.cert_slot, c.cert_count.p + (c.cert_slot ^ 1)};
    }
    if (c.match_stamps) {
      // zeroed once, at allocation: a memset before every launch would end the programmatic
      // dependence on the previous reject/solve kernel (the kernel clears its own slots)
      if (c.match_t.p == nullptr) {
        c.match_t.reserve(16);
        SICP_CUDA(cudaMemsetAsync(c.match_t.p, 0, 16 * sizeof(unsigned long long), c.stream));
      }
      cert.stamps = c.match_t.p;
    }
    const int mg = match_lanes(c, K, 2);
    with_lanes<2, 4, 8, 16>(mg, [&](auto L) {
      launch_kernel(k_match_grid_coop<decltype(L)::value>, dim3((unsigned)((K * mg + 127) / 128)), dim3(128), 0,
                    c.stream, pdl, c.gmov.view, c.dev_state.p, c.q_xyz.p, c.q_nrm.p, c.mov_xyz.p, K, rmax,
                    with_distance ? 1 : 0, c.nn_idx.p, out, c.unresolved.p, lh, cap2, co, cert);
    });
  }
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
  if (mid) SICP_CUDA(cudaEventRecord(mid, c.stream));
  if (use_bf) bf_launch(c, with_distance, out, false);
  if (with_distance) c.lin_hist_pending = true;
}

}  // namespace sicp
