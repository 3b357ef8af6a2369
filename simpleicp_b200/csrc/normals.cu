// normals.cu — PointCloud.estimate_normals (python/simpleicp/pointcloud.py:173-203):
// k nearest neighbours (query point included) of every selected fixed point in the fixed cloud,
// covariance with ddof = 1 (np.cov), symmetric 3x3 eigen-decomposition, normal = eigenvector of
// the smallest eigenvalue, planarity = (l_mid - l_min) / l_max, both rounded to float32 exactly
// where the reference does (pointcloud.py:180-183, 194-198).
//
// Two kernels: an exact grid k-NN (float64, ring expansion until the k-th best is provably final)
// that emits the neighbours as positions in the cell-sorted record array, and the covariance /
// eigen-solve / float4 (nx, ny, nz, planarity) store, which reads those records (L2-hot) instead
// of gathering the caller-order cloud.  Neighbour indices and distances are written out only
// when the caller asked for them (option "keep_knn").
#include <algorithm>

#include "ctx.cuh"
#include "eig3.cuh"

namespace sicp {

namespace {

constexpr int kMaxK = 64;

// =============================================================================================
// Cooperative k-NN for k <= 16 (the reference's default is 10): MG lanes share one query.
//   * every lane scans its share of the grid rows (x-contiguous cell runs) and keeps its OWN best
//     KC candidates (distance, record position) in registers — a fully unrolled compare-exchange
//     insertion, no dynamically indexed array, hence no local-memory stack frame (the
//     one-thread-per-query kernel above carries a 1.3 KB frame for its 64-slot list);
//   * after each ring the group extracts the k-th smallest of the union of its lists (k rounds of
//     a shuffle arg-min over the list heads): that is the exact current k-th neighbour distance,
//     used to prune rows of the next ring and for the termination proof
//     (k-th best <= distance to every unexplored cell);
//   * the final k rounds emit the neighbours in (distance, index) order as record positions.
// The covariance / eigen-solve run in a second kernel, one thread per query (k_pca_from_knn): in
// this one three of four lanes would idle through the ~2000-instruction dgeev walk.  It reads
// the neighbours from the cell-sorted records the search just touched (L2-hot), not from the
// caller-order cloud.  Ordering (distance, then original index) and the summation order of mean
// and covariance are those of the kernel above: the float32 normals are bit-identical.
// =============================================================================================
template <int KC>
struct LaneList {
  double d[KC];
  uint32_t p[KC];
};

// (da, pa) before (db, pb)?  Equal distances are ordered by ORIGINAL index (deterministic; the
// position inside a cell depends on the order of the build's atomics); that needs the records,
// but only on an exact tie.
__device__ __forceinline__ bool cand_less(const Rec* __restrict__ recs, double da, uint32_t pa, double db,
                                          uint32_t pb) {
  if (da != db) return da < db;
  if (pb == 0xffffffffu) return pa != 0xffffffffu;
  if (pa == 0xffffffffu) return false;
  return recs[pa].idx < recs[pb].idx;
}

template <int KC>
__device__ __forceinline__ void lane_insert(const Rec* __restrict__ recs, LaneList<KC>& L, double d, uint32_t p) {
  if (!cand_less(recs, d, p, L.d[KC - 1], L.p[KC - 1])) return;
  L.d[KC - 1] = d;
  L.p[KC - 1] = p;
#pragma unroll
  for (int j = KC - 1; j >= 1; --j) {
    const bool sw = cand_less(recs, L.d[j], L.p[j], L.d[j - 1], L.p[j - 1]);
    const double td = sw ? L.d[j - 1] : L.d[j];
    const uint32_t tp = sw ? L.p[j - 1] : L.p[j];
    L.d[j - 1] = sw ? L.d[j] : L.d[j - 1];
    L.p[j - 1] = sw ? L.p[j] : L.p[j - 1];
    L.d[j] = td;
    L.p[j] = tp;
  }
}

template <int KC>
__device__ __forceinline__ void scan_range_l(const Rec* __restrict__ recs, uint32_t s, uint32_t e, double qx,
                                             double qy, double qz, double bound, LaneList<KC>& L) {
  auto visit = [&](const double rx, const double ry, const double rz, uint32_t pos) {
    const double dx = rx - qx, dy = ry - qy, dz = rz - qz;
    const double d2 = dx * dx + dy * dy + dz * dz;
    if (d2 <= bound) lane_insert<KC>(recs, L, d2, pos);
  };
  for (uint32_t i = s; i < e; i += 4) {
    // four 32-byte records in flight; the clamped tail repeats the last record, which is skipped
    const uint32_t last = e - 1;
    const uint32_t i1 = min(i + 1, last), i2 = min(i + 2, last), i3 = min(i + 3, last);
    const Rec r0 = recs[i];
    const Rec r1 = recs[i1];
    const Rec r2 = recs[i2];
    const Rec r3 = recs[i3];
    visit(r0.x, r0.y, r0.z, i);
    if (i1 != i) visit(r1.x, r1.y, r1.z, i1);
    if (i2 != i1) visit(r2.x, r2.y, r2.z, i2);
    if (i3 != i2) visit(r3.x, r3.y, r3.z, i3);
  }
}

// k rounds of arg-min over the heads of the lanes' sorted lists.  Returns the k-th smallest of
// the union (kInf if the union holds fewer than k); when out != nullptr lane 0 of the group
// stores the positions in order.
template <int MG, int KC>
__device__ __forceinline__ double union_kth(const Rec* __restrict__ recs, const LaneList<KC>& L, int k,
                                            unsigned int gmask, int sub, uint32_t* __restrict__ out) {
  int head = 0;
  double last = kInf;
  for (int round = 0; round < k; ++round) {
    double d = kInf;
    uint32_t p = 0xffffffffu;
#pragma unroll
    for (int j = 0; j < KC; ++j)
      if (j == head) {
        d = L.d[j];
        p = L.p[j];
      }
    double bd = d;
    uint32_t bp = p;
    int bl = sub;
#pragma unroll
    for (int o = MG / 2; o > 0; o >>= 1) {
      const double od = __shfl_xor_sync(gmask, bd, o, MG);
      const uint32_t op = __shfl_xor_sync(gmask, bp, o, MG);
      const int ol = __shfl_xor_sync(gmask, bl, o, MG);
      // identical (d, p) cannot come from two lanes (a record is scanned by one lane only)
      const bool take = cand_less(recs, od, op, bd, bp);
      if (take) {
        bd = od;
        bp = op;
        bl = ol;
      }
    }
    if (bl == sub && bp != 0xffffffffu) ++head;
    last = (bp == 0xffffffffu) ? kInf : bd;
    if (out != nullptr && sub == 0) out[round] = bp;
  }
  return last;
}

template <int MG, int KC>
__device__ __forceinline__ void knn_coop_body(const GridView& g, const double* __restrict__ q_xyz, long long K,
                                              int k, uint32_t* __restrict__ knn_pos, const long long gt) {
  const long long qi = gt / MG;
  const int sub = threadIdx.x & (MG - 1);
  if (qi >= K) return;  // a whole group leaves together
  const unsigned int gmask = (MG == 32) ? 0xffffffffu : (((1u << MG) - 1u) << ((threadIdx.x & 31) & ~(MG - 1)));
  const double qx = q_xyz[3 * qi + 0], qy = q_xyz[3 * qi + 1], qz = q_xyz[3 * qi + 2];
  const int cx = cell_coord(qx, g.ox, g.inv_h, g.nx);
  const int cy = cell_coord(qy, g.oy, g.inv_h, g.ny);
  const int cz = cell_coord(qz, g.oz, g.inv_h, g.nz);
  const uint32_t* __restrict__ cs = g.cell_start;
  LaneList<KC> L;
#pragma unroll
  for (int j = 0; j < KC; ++j) {
    L.d[j] = kInf;
    L.p[j] = 0xffffffffu;
  }
  double B = kInf;  // current k-th best of the union (upper bound of the final one)
  for (int r = 1;; ++r) {
    const int x0 = cx - r, x1 = cx + r;
    const int xa = max(x0, 0), xb = min(x1, g.nx - 1);
    const int side = 2 * r + 1, items = side * side;
    const double lim = B * (1.0 + 1e-12);  // strictly farther rows only: ties are still visited
    int dzr = sub / side, dyr = sub - dzr * side;
    for (int t = sub; t < items; t += MG, dyr += MG) {
      while (dyr >= side) {
        dyr -= side;
        ++dzr;
      }
      const int dz = dzr - r, dy = dyr - r;
      const int y = cy + dy, z = cz + dz;
      if (y < 0 || y >= g.ny || z < 0 || z >= g.nz) continue;
      const bool full = (r == 1) || dy == -r || dy == r || dz == -r || dz == r;
      if (r > 1) {
        const double by = (dy < 0) ? qy - (g.oy + (y + 1) * g.h) : ((dy > 0) ? (g.oy + y * g.h) - qy : 0.0);
        const double bz = (dz < 0) ? qz - (g.oz + (z + 1) * g.h) : ((dz > 0) ? (g.oz + z * g.h) - qz : 0.0);
        const double lb = fmax(by, 0.0) * fmax(by, 0.0) + fmax(bz, 0.0) * fmax(bz, 0.0);
        if (lb > lim) continue;
      }
      const long long row = ((long long)z * g.ny + y) * g.nx;
      if (full) {
        scan_range_l<KC>(g.recs, cs[row + xa], cs[row + xb + 1], qx, qy, qz, lim, L);
      } else {
        if (x0 >= 0) scan_range_l<KC>(g.recs, cs[row + x0], cs[row + x0 + 1], qx, qy, qz, lim, L);
        if (x1 < g.nx) scan_range_l<KC>(g.recs, cs[row + x1], cs[row + x1 + 1], qx, qy, qz, lim, L);
      }
    }
    B = union_kth<MG, KC>(g.recs, L, k, gmask, sub, nullptr);
    const int y0 = cy - r, y1 = cy + r, z0 = cz - r, z1 = cz + r;
    double guard = kInf;
    if (x0 > 0) guard = fmin(guard, qx - (g.ox + x0 * g.h));
    if (x1 < g.nx - 1) guard = fmin(guard, (g.ox + (x1 + 1) * g.h) - qx);
    if (y0 > 0) guard = fmin(guard, qy - (g.oy + y0 * g.h));
    if (y1 < g.ny - 1) guard = fmin(guard, (g.oy + (y1 + 1) * g.h) - qy);
    if (z0 > 0) guard = fmin(guard, qz - (g.oz + z0 * g.h));
    if (z1 < g.nz - 1) guard = fmin(guard, (g.oz + (z1 + 1) * g.h) - qz);
    if (guard >= kInf) break;  // the block covers the whole grid
    guard -= 1e-9 * g.h;
    if (B < kInf && guard > 0.0 && B <= guard * guard) break;
  }
  union_kth<MG, KC>(g.recs, L, k, gmask, sub, knn_pos + qi * k);
}

// One thread per query, 16 < k <= 64 (the reference's webots test uses k = 40): a sorted list of
// record POSITIONS in a dynamically indexed (local-memory) array, ties by original index through
// the records as everywhere, written to knn_pos for k_pca_from_knn.
struct TopKPos {
  double d2[kMaxK];
  uint32_t pos[kMaxK];
  int n, k;
  __device__ __forceinline__ bool full() const { return n == k; }
  __device__ __forceinline__ double worst() const { return d2[n - 1]; }
  __device__ __forceinline__ void consider(const Rec* __restrict__ recs, double d, uint32_t p, long long idx) {
    if (n == k) {
      if (!(d < d2[k - 1] || (d == d2[k - 1] && idx < recs[pos[k - 1]].idx))) return;
    } else {
      ++n;
    }
    int j = n - 1;
    while (j > 0 && (d2[j - 1] > d || (d2[j - 1] == d && recs[pos[j - 1]].idx > idx))) {
      d2[j] = d2[j - 1];
      pos[j] = pos[j - 1];
      --j;
    }
    d2[j] = d;
    pos[j] = p;
  }
};

__device__ __forceinline__ void scan_range_kp(const Rec* __restrict__ recs, uint32_t s, uint32_t e, double qx,
                                              double qy, double qz, TopKPos& tk) {
  for (uint32_t i = s; i < e; i += 4) {
    const uint32_t last = e - 1;
    const Rec r0 = recs[i];
    const Rec r1 = recs[min(i + 1, last)];
    const Rec r2 = recs[min(i + 2, last)];
    const Rec r3 = recs[min(i + 3, last)];
    const int n = (int)min(4u, e - i);
    const Rec* rr[4] = {&r0, &r1, &r2, &r3};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j < n) {
        const double dx = rr[j]->x - qx, dy = rr[j]->y - qy, dz = rr[j]->z - qz;
        tk.consider(recs, dx * dx + dy * dy + dz * dz, i + j, rr[j]->idx);
      }
    }
  }
}

__device__ __forceinline__ void knn_single_body(const GridView& g, const double* __restrict__ q_xyz, long long K,
                                                int k, uint32_t* __restrict__ knn_pos, const long long i) {
  if (i >= K) return;
  const double qx = q_xyz[3 * i + 0], qy = q_xyz[3 * i + 1], qz = q_xyz[3 * i + 2];
  TopKPos tk;
  tk.n = 0;
  tk.k = k;
  const int cx = cell_coord(qx, g.ox, g.inv_h, g.nx);
  const int cy = cell_coord(qy, g.oy, g.inv_h, g.ny);
  const int cz = cell_coord(qz, g.oz, g.inv_h, g.nz);
  const uint32_t* __restrict__ cs = g.cell_start;
  for (int r = 1;; ++r) {
    const int x0 = cx - r, x1 = cx + r, y0 = cy - r, y1 = cy + r, z0 = cz - r, z1 = cz + r;
    const int xa = max(x0, 0), xb = min(x1, g.nx - 1);
    const int side = 2 * r + 1, items = side * side, centre = items / 2;
    for (int t0 = 0; t0 < items; ++t0) {
      const int t = (r == 1) ? ((t0 == 0) ? centre : ((t0 <= centre) ? t0 - 1 : t0)) : t0;
      const int dz = t / side - r, dy = t % side - r;
      const int y = cy + dy, z = cz + dz;
      if (y < 0 || y >= g.ny || z < 0 || z >= g.nz) continue;
      if (tk.full()) {
        const double by = (dy < 0) ? qy - (g.oy + (y + 1) * g.h) : ((dy > 0) ? (g.oy + y * g.h) - qy : 0.0);
        const double bz = (dz < 0) ? qz - (g.oz + (z + 1) * g.h) : ((dz > 0) ? (g.oz + z * g.h) - qz : 0.0);
        const double lb = fmax(by, 0.0) * fmax(by, 0.0) + fmax(bz, 0.0) * fmax(bz, 0.0);
        if (lb > tk.worst() * (1.0 + 1e-12)) continue;
      }
      const long long row = ((long long)z * g.ny + y) * g.nx;
      const bool full = (r == 1) || dy == -r || dy == r || dz == -r || dz == r;
      if (full) {
        scan_range_kp(g.recs, cs[row + xa], cs[row + xb + 1], qx, qy, qz, tk);
      } else {
        if (x0 >= 0) scan_range_kp(g.recs, cs[row + x0], cs[row + x0 + 1], qx, qy, qz, tk);
        if (x1 < g.nx) scan_range_kp(g.recs, cs[row + x1], cs[row + x1 + 1], qx, qy, qz, tk);
      }
    }
    double guard = kInf;
    if (x0 > 0) guard = fmin(guard, qx - (g.ox + x0 * g.h));
    if (x1 < g.nx - 1) guard = fmin(guard, (g.ox + (x1 + 1) * g.h) - qx);
    if (y0 > 0) guard = fmin(guard, qy - (g.oy + y0 * g.h));
    if (y1 < g.ny - 1) guard = fmin(guard, (g.oy + (y1 + 1) * g.h) - qy);
    if (z0 > 0) guard = fmin(guard, qz - (g.oz + z0 * g.h));
    if (z1 < g.nz - 1) guard = fmin(guard, (g.oz + (z1 + 1) * g.h) - qz);
    if (guard >= kInf) break;
    guard -= 1e-9 * g.h;
    if (tk.full() && guard > 0.0 && tk.worst() <= guard * guard) break;
  }
  for (int j = 0; j < k; ++j) knn_pos[i * k + j] = (j < tk.n) ? tk.pos[j] : 0xffffffffu;
}

__global__ void __launch_bounds__(128)
    k_knn_single(GridView g, const double* __restrict__ q_xyz, long long K, int k, uint32_t* __restrict__ knn_pos) {
  knn_single_body(g, q_xyz, K, k, knn_pos, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}
__global__ void __launch_bounds__(128)
    k_knn_single_batch(const PairDev* __restrict__ pairs, const double* __restrict__ q_xyz, int k, long long Kmax,
                       uint32_t* __restrict__ knn_pos) {
  const PairDev pd = pairs[blockIdx.y];
  knn_single_body(pd.gfix, q_xyz + 3 * pd.q_off, pd.K, k, knn_pos + (size_t)blockIdx.y * Kmax * k,
                  blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

template <int MG, int KC>
__global__ void __launch_bounds__(128)
    k_knn_coop(GridView g, const double* __restrict__ q_xyz, long long K, int k, uint32_t* __restrict__ knn_pos) {
  knn_coop_body<MG, KC>(g, q_xyz, K, k, knn_pos, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

// covariance (np.cov, ddof = 1) + eigen-solve + float32 store from the neighbour positions; the
// arithmetic of knn_pca_body, the points taken from the cell-sorted records
__device__ __forceinline__ void pca_from_knn_body(const GridView& g, const double* __restrict__ q_xyz, long long K,
                                                  int k, int sign_mode, const uint32_t* __restrict__ knn_pos,
                                                  float4* __restrict__ q_nrm, long long* __restrict__ knn_idx,
                                                  double* __restrict__ knn_d2, const long long i) {
  if (i >= K) return;
  const uint32_t* __restrict__ pp = knn_pos + i * k;
  int n = 0;
  double mx = 0, my = 0, mz = 0;
  for (int j = 0; j < k; ++j) {
    const uint32_t p = pp[j];
    if (p == 0xffffffffu) break;
    const Rec r = g.recs[p];
    mx += r.x;
    my += r.y;
    mz += r.z;
    ++n;
    if (knn_idx) {
      knn_idx[i * k + j] = r.idx;
      if (knn_d2) {
        const double dx = r.x - q_xyz[3 * i + 0], dy = r.y - q_xyz[3 * i + 1], dz = r.z - q_xyz[3 * i + 2];
        knn_d2[i * k + j] = dx * dx + dy * dy + dz * dz;
      }
    }
  }
  const double inv = 1.0 / (double)n;
  mx *= inv;
  my *= inv;
  mz *= inv;
  double c00 = 0, c01 = 0, c02 = 0, c11 = 0, c12 = 0, c22 = 0;
  for (int j = 0; j < n; ++j) {
    const Rec r = g.recs[pp[j]];
    const double dx = r.x - mx, dy = r.y - my, dz = r.z - mz;
    c00 = fma(dx, dx, c00);
    c01 = fma(dx, dy, c01);
    c02 = fma(dx, dz, c02);
    c11 = fma(dy, dy, c11);
    c12 = fma(dy, dz, c12);
    c22 = fma(dz, dz, c22);
  }
  const double f = 1.0 / (double)(n - 1);
  c00 *= f;
  c01 *= f;
  c02 *= f;
  c11 *= f;
  c12 *= f;
  c22 *= f;
  double w[3], nn[3];
  eig3_smallest(c00, c01, c02, c11, c12, c22, sign_mode, w, nn);
  float4 o;
  o.x = (float)nn[0];
  o.y = (float)nn[1];
  o.z = (float)nn[2];
  o.w = (float)((w[1] - w[2]) / w[0]);
  q_nrm[i] = o;
}

__global__ void __launch_bounds__(128)
    k_pca_from_knn(GridView g, const double* __restrict__ q_xyz, long long K, int k, int sign_mode,
                   const uint32_t* __restrict__ knn_pos, float4* __restrict__ q_nrm,
                   long long* __restrict__ knn_idx, double* __restrict__ knn_d2) {
  pca_from_knn_body(g, q_xyz, K, k, sign_mode, knn_pos, q_nrm, knn_idx, knn_d2,
                    blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

// One thread per query with the list in REGISTERS (k <= KC <= 16): the insertion network of the
// cooperative kernel, one list per query (a third of the insertions of four lane lists, no
// merge rounds), no local-memory frame.  Measured at K = 100 000, k = 10: 333 us against 258 us
// of the local-memory list above (the network executes all KC compare-selects per accepted
// candidate and its 117 registers halve the resident warps), so it is selectable (option
// "knn_coop" = 2) but not a default.
template <int KC>
__device__ __forceinline__ void knn_reg_body(const GridView& g, const double* __restrict__ q_xyz, long long K,
                                             int k, uint32_t* __restrict__ knn_pos, const long long i) {
  if (i >= K) return;
  const double qx = q_xyz[3 * i + 0], qy = q_xyz[3 * i + 1], qz = q_xyz[3 * i + 2];
  const int cx = cell_coord(qx, g.ox, g.inv_h, g.nx);
  const int cy = cell_coord(qy, g.oy, g.inv_h, g.ny);
  const int cz = cell_coord(qz, g.oz, g.inv_h, g.nz);
  const uint32_t* __restrict__ cs = g.cell_start;
  // The list has KC slots but only k of them are wanted: the first KC - k slots hold -inf
  // sentinels that nothing ever displaces, so the k real entries live in the LAST k slots and the
  // k-th best is always slot KC - 1 — a compile-time index.  (Selecting slot k - 1 with a chain of
  // compares is turned into a dynamically indexed load by the compiler, which puts the whole list
  // into local memory: 144-byte frame, 450 LDL/STL, 1.7x slower.)
  LaneList<KC> L;
#pragma unroll
  for (int j = 0; j < KC; ++j) {
    L.d[j] = (j < KC - k) ? -kInf : kInf;
    L.p[j] = 0xffffffffu;
  }
  for (int r = 1;; ++r) {
    const int x0 = cx - r, x1 = cx + r, y0 = cy - r, y1 = cy + r, z0 = cz - r, z1 = cz + r;
    const int xa = max(x0, 0), xb = min(x1, g.nx - 1);
    const int side = 2 * r + 1, items = side * side, centre = items / 2;
    for (int t0 = 0; t0 < items; ++t0) {
      // the centre row first in ring 1: the list fills with near points, later rows are pruned
      const int t = (r == 1) ? ((t0 == 0) ? centre : ((t0 <= centre) ? t0 - 1 : t0)) : t0;
      const int dz = t / side - r, dy = t % side - r;
      const int y = cy + dy, z = cz + dz;
      if (y < 0 || y >= g.ny || z < 0 || z >= g.nz) continue;
      const double lim = L.d[KC - 1] * (1.0 + 1e-12);  // k-th best so far (inf until k are known)
      const double by = (dy < 0) ? qy - (g.oy + (y + 1) * g.h) : ((dy > 0) ? (g.oy + y * g.h) - qy : 0.0);
      const double bz = (dz < 0) ? qz - (g.oz + (z + 1) * g.h) : ((dz > 0) ? (g.oz + z * g.h) - qz : 0.0);
      const double lb = fmax(by, 0.0) * fmax(by, 0.0) + fmax(bz, 0.0) * fmax(bz, 0.0);
      if (lb > lim) continue;  // strictly farther: ties are still visited
      const long long row = ((long long)z * g.ny + y) * g.nx;
      const bool full = (r == 1) || dy == -r || dy == r || dz == -r || dz == r;
      if (full) {
        scan_range_l<KC>(g.recs, cs[row + xa], cs[row + xb + 1], qx, qy, qz, lim, L);
      } else {
        if (x0 >= 0) scan_range_l<KC>(g.recs, cs[row + x0], cs[row + x0 + 1], qx, qy, qz, lim, L);
        if (x1 < g.nx) scan_range_l<KC>(g.recs, cs[row + x1], cs[row + x1 + 1], qx, qy, qz, lim, L);
      }
    }
    double guard = kInf;
    if (x0 > 0) guard = fmin(guard, qx - (g.ox + x0 * g.h));
    if (x1 < g.nx - 1) guard = fmin(guard, (g.ox + (x1 + 1) * g.h) - qx);
    if (y0 > 0) guard = fmin(guard, qy - (g.oy + y0 * g.h));
    if (y1 < g.ny - 1) guard = fmin(guard, (g.oy + (y1 + 1) * g.h) - qy);
    if (z0 > 0) guard = fmin(guard, qz - (g.oz + z0 * g.h));
    if (z1 < g.nz - 1) guard = fmin(guard, (g.oz + (z1 + 1) * g.h) - qz);
    if (guard >= kInf) break;
    guard -= 1e-9 * g.h;
    const double kth = L.d[KC - 1];
    if (kth < kInf && guard > 0.0 && kth <= guard * guard) break;
  }
#pragma unroll
  for (int j = 0; j < KC; ++j)
    if (j >= KC - k) knn_pos[i * k + (j - (KC - k))] = L.p[j];
}

template <int KC>
__global__ void __launch_bounds__(128)
    k_knn_reg(GridView g, const double* __restrict__ q_xyz, long long K, int k, uint32_t* __restrict__ knn_pos) {
  knn_reg_body<KC>(g, q_xyz, K, k, knn_pos, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}
template <int KC>
__global__ void __launch_bounds__(128)
    k_knn_reg_batch(const PairDev* __restrict__ pairs, const double* __restrict__ q_xyz, int k, long long Kmax,
                    uint32_t* __restrict__ knn_pos) {
  const PairDev pd = pairs[blockIdx.y];
  knn_reg_body<KC>(pd.gfix, q_xyz + 3 * pd.q_off, pd.K, k, knn_pos + (size_t)blockIdx.y * Kmax * k,
                   blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

// batched forms: blockIdx.y = pair
template <int MG, int KC>
__global__ void __launch_bounds__(128)
    k_knn_coop_batch(const PairDev* __restrict__ pairs, const double* __restrict__ q_xyz, int k, long long Kmax,
                     uint32_t* __restrict__ knn_pos) {
  const PairDev pd = pairs[blockIdx.y];
  knn_coop_body<MG, KC>(pd.gfix, q_xyz + 3 * pd.q_off, pd.K, k, knn_pos + (size_t)blockIdx.y * Kmax * k,
                        blockIdx.x * (long long)blockDim.x + threadIdx.x);
}
__global__ void __launch_bounds__(128)
    k_pca_from_knn_batch(const PairDev* __restrict__ pairs, const double* __restrict__ q_xyz, int k, long long Kmax,
                         int sign_mode, const uint32_t* __restrict__ knn_pos, float4* __restrict__ q_nrm) {
  const PairDev pd = pairs[blockIdx.y];
  pca_from_knn_body(pd.gfix, q_xyz + 3 * pd.q_off, pd.K, k, sign_mode, knn_pos + (size_t)blockIdx.y * Kmax * k,
                    q_nrm + pd.q_off, nullptr, nullptr, blockIdx.x * (long long)blockDim.x + threadIdx.x);
}

}  // namespace

void estimate_normals_launch(Ctx& c, int k) {
  SICP_REQUIRE(k >= 2 && k <= kMaxK, SICP_ERR_BAD_ARG,
               "neighbors must be between 2 and 64 (got " + std::to_string(k) + ")");
  SICP_REQUIRE((long long)k <= c.n_fix, SICP_ERR_BAD_ARG,
               "neighbors exceeds the number of points in the fixed cloud");
  c.q_nrm.reserve(std::max<long long>(c.K, 1));
  // the neighbour lists leave the SM only when somebody wants to look at them (option "keep_knn")
  long long* kidx = nullptr;
  double* kd2 = nullptr;
  if (c.keep_knn) {
    c.knn_idx.reserve((size_t)c.K * k);
    c.knn_d2.reserve((size_t)c.K * k);
    kidx = c.knn_idx.p;
    kd2 = c.knn_d2.p;
  }
  c.knn_k = c.keep_knn ? k : 0;
  // All k-NN kernels hand record positions to k_pca_from_knn.  knn_coop: 1 = cooperative lanes
  // (k <= 16), 0 = one thread per query with the list in local memory, 2 = one thread per query
  // with the list in registers (k <= 16), -1 (default) = cooperative while the search is
  // latency-bound (few queries), one thread per query with the local-memory list once the queries
  // fill the machine (K = 100 000, k = 10: faster than a register list or cooperative lanes — the
  // fixed-length insertion network costs more than the early-exit loop saves in memory traffic).
  const bool coop = (k <= 16) && (c.knn_coop == 1 || (c.knn_coop < 0 && c.K <= 16384));
  const bool reg = (k <= 16) && c.knn_coop == 2;
  c.knn_pos.reserve((size_t)c.K * k);
  const GridView g = c.gfix.view();
  if (coop) {
    const int mg = (c.K <= 32768) ? 8 : 4;
    const unsigned blocks = (unsigned)((c.K * mg + 127) / 128);
    if (mg == 8) {
      if (k <= 12) k_knn_coop<8, 12><<<blocks, 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
      else k_knn_coop<8, 16><<<blocks, 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
    } else {
      if (k <= 12) k_knn_coop<4, 12><<<blocks, 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
      else k_knn_coop<4, 16><<<blocks, 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
    }
  } else if (reg && k <= 12) {
    k_knn_reg<12><<<(unsigned)((c.K + 127) / 128), 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
  } else if (reg) {
    k_knn_reg<16><<<(unsigned)((c.K + 127) / 128), 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
  } else {
    k_knn_single<<<(unsigned)((c.K + 127) / 128), 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.knn_pos.p);
  }
  k_pca_from_knn<<<(unsigned)((c.K + 127) / 128), 128, 0, c.stream>>>(g, c.q_xyz.p, c.K, k, c.sign_mode,
                                                                      c.knn_pos.p, c.q_nrm.p, kidx, kd2);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 2;
}

void batch_normals_launch(Ctx& c, Batch& b, int k) {
  SICP_REQUIRE(k >= 2 && k <= kMaxK, SICP_ERR_BAD_ARG,
               "neighbors must be between 2 and 64 (got " + std::to_string(k) + ")");
  const long long total = b.Kmax * b.n_pairs;
  const bool coop = (k <= 16) && (c.knn_coop == 1 || (c.knn_coop < 0 && total <= 16384));
  const bool reg = (k <= 16) && c.knn_coop == 2;
  b.knn_pos.reserve((size_t)b.n_pairs * b.Kmax * k);
  if (coop) {
    const dim3 grid((unsigned)((b.Kmax * 8 + 127) / 128), b.n_pairs);
    if (k <= 12) k_knn_coop_batch<8, 12><<<grid, 128, 0, c.stream>>>(b.pairs.p, b.q_xyz.p, k, b.Kmax, b.knn_pos.p);
    else k_knn_coop_batch<8, 16><<<grid, 128, 0, c.stream>>>(b.pairs.p, b.q_xyz.p, k, b.Kmax, b.knn_pos.p);
  } else if (reg && k <= 12) {
    k_knn_reg_batch<12><<<dim3((unsigned)((b.Kmax + 127) / 128), b.n_pairs), 128, 0, c.stream>>>(
        b.pairs.p, b.q_xyz.p, k, b.Kmax, b.knn_pos.p);
  } else if (reg) {
    k_knn_reg_batch<16><<<dim3((unsigned)((b.Kmax + 127) / 128), b.n_pairs), 128, 0, c.stream>>>(
        b.pairs.p, b.q_xyz.p, k, b.Kmax, b.knn_pos.p);
  } else {
    k_knn_single_batch<<<dim3((unsigned)((b.Kmax + 127) / 128), b.n_pairs), 128, 0, c.stream>>>(
        b.pairs.p, b.q_xyz.p, k, b.Kmax, b.knn_pos.p);
  }
  k_pca_from_knn_batch<<<dim3((unsigned)((b.Kmax + 127) / 128), b.n_pairs), 128, 0, c.stream>>>(
      b.pairs.p, b.q_xyz.p, k, b.Kmax, c.sign_mode, b.knn_pos.p, b.q_nrm.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 2;
}

}  // namespace sicp
