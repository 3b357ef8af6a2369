// joint.cu — the device work of sicp_register_joint per iteration, after the batched match of
// every edge (batch_match_launch, unchanged):
//
//   k_joint_reject   one block per edge: median / MAD of all distances (upper middle elements, by a
//                    bitonic sort of the order-preserving keys in shared memory), the linearised
//                    keep rule, the edge's point-to-plane normal equations N, h = sum a d from the
//                    kept rows a = [w x n, n] with w = R_e (p - c_m) (centred about the edge's movable
//                    centre c_f = R_e c_m in frame a), and the edge's 6 x 6 block Ad^T N Ad and
//                    right-hand side -Ad^T h in the common world parameterisation
//   k_joint_prior    with pose priors only (DESIGN.md §6.12): one thread per prior, its observation
//                    at the current pose and the cloud's block and right-hand side
//   k_joint_relative with relative observations only (DESIGN.md §6.13): one thread per observation,
//                    its value at the current poses and the blocks and right-hand sides of its clouds
//   k_joint_solve    one cooperative launch: assembly of the dense 6F x 6F normal matrix, augmented
//                    by the right-hand side as one more row, from the edge blocks in ascending edge
//                    order; right-looking tiled Cholesky (the augmented row leaves L^-1 b behind);
//                    back substitution; the pose update of every free cloud, each edge's new
//                    relative transform, increment, residual statistics, record and stop rule
//   k_joint_sparse_solve  in its place under option "joint_solver" 1: the same system by the
//                    supernodal Cholesky of joint_plan.h's nested-dissection plan, level by level,
//                    and the same tail spread over the grid (DESIGN.md §6.11)
//
// and, on the first sicp_get_joint_covariances after a call, from what its final iteration left:
//
//   k_joint_cov_ss     one block per edge: the sum of the squared final residuals of its kept rows
//   k_joint_inv        one cooperative launch: Z = L^-1 of the final factor, by 32 x 32 tiles
//   k_joint_cov_cloud  one block per free cloud: s0^2, the block (N^-1)_cc = sum_k Z_kc^T Z_kc and
//                      C_c = s0^2 J_c (N^-1)_cc J_c^T
//   k_joint_cov_edge   one block per edge: the cross block of two free clouds and C_e
//
// and, on the first sicp_get_joint_selected_covariances after a call under joint_solver 1
// (DESIGN.md §6.14), after k_joint_cov_ss:
//
//   k_joint_sel_parked  per edge whose cross block lies outside the pattern: w_a^T w_b, w_c = L^-1 E_c
//   k_joint_selinv      one cooperative launch: Z = N'^-1 on the pattern of the sparse factor, by
//                       Takahashi's recurrence from the roots down, one block per supernode
//   k_joint_sel_s0      one warp: s0^2 (the statement k_joint_cov_cloud uses)
//   k_joint_sel_cloud   one thread per free cloud: C_c = s0^2 J'_c (N'^-1)_cc J'_c^T
//   k_joint_sel_edge    one thread per edge: the cross block and C_e
//
// DESIGN.md §6.9 gives the rule, the Ad mapping and the centring.  Every sum runs in a fixed
// order (no atomics), so repeated calls give the same bits.
#include "ctx.cuh"

namespace sicp {

namespace {

constexpr int JR_THREADS = 512;
constexpr int JR_WARPS = JR_THREADS / 32;
constexpr int JR_CAP = 4096;  // correspondences per edge (sicp_register_pairs' limit)
constexpr int JS_THREADS = 256;
constexpr int TS = 32;        // Cholesky tile

// Ascending bitonic sort of P (a power of two) keys in shared memory by the whole block.
__device__ void bitonic_sort(unsigned long long* k, int P) {
  for (int size = 2; size <= P; size <<= 1)
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < P / 2; t += blockDim.x) {
        const int lo = 2 * t - (t & (stride - 1)), hi = lo + stride;
        const bool up = (lo & size) == 0;
        const unsigned long long x = k[lo], y = k[hi];
        if ((x > y) == up) {
          k[lo] = y;
          k[hi] = x;
        }
      }
    }
  __syncthreads();
}

// xi = Ad y: a world-frame increment y = (omega, t') about the world centre c_w, carried into
// frame a about the edge centre c_f (Ra: rotation of the pose of cloud a, v = T_a c_f - c_w):
// alpha = Ra^T omega, t_c = Ra^T (t' - v x omega).
__device__ __forceinline__ void ad_apply(const double* Ra, const double* v, const double* y, double* xi) {
  const double w0 = y[0], w1 = y[1], w2 = y[2];
  const double u0 = y[3] - (v[1] * w2 - v[2] * w1), u1 = y[4] - (v[2] * w0 - v[0] * w2),
               u2 = y[5] - (v[0] * w1 - v[1] * w0);
  for (int r = 0; r < 3; ++r) {
    xi[r] = Ra[0 * 3 + r] * w0 + Ra[1 * 3 + r] * w1 + Ra[2 * 3 + r] * w2;
    xi[3 + r] = Ra[0 * 3 + r] * u0 + Ra[1 * 3 + r] * u1 + Ra[2 * 3 + r] * u2;
  }
}

__device__ __forceinline__ int tri(int r, int c) { return r * (r + 1) / 2 + c; }  // c <= r

__global__ void __launch_bounds__(JR_THREADS) k_joint_reject(const JointArgs a) {
  __shared__ unsigned long long key[JR_CAP];
  __shared__ double red[JR_WARPS][JE_NSUM];
  __shared__ double tot[JE_NSUM];
  const int e = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (a.flags->done) return;
  DevState* st = a.state + e;
  if (st->stop) return;  // no overlap: the edge takes no part
  const PairDev& pd = a.pairs[e];
  const long long q = pd.q_off;
  const int K = (int)pd.K;
  int P = 1;
  while (P < K) P <<= 1;
  // median and MAD over every distance: the element at K / 2 of the sorted keys
  for (int i = tid; i < P; i += JR_THREADS) key[i] = (i < K) ? f64_to_key(a.dist[q + i]) : ~0ull;
  bitonic_sort(key, P);
  const double med = key_to_f64(key[K >> 1]);
  __syncthreads();
  for (int i = tid; i < P; i += JR_THREADS) key[i] = (i < K) ? f64_to_key(fabs(a.dist[q + i] - med)) : ~0ull;
  bitonic_sort(key, P);
  const double mad = key_to_f64(key[K >> 1]);
  const double lim = 3.0 * (1.4826 * mad);

  const Rigid R = st->T;
  const double cm0 = pd.cm[0], cm1 = pd.cm[1], cm2 = pd.cm[2];
  double acc[JE_NSUM];
#pragma unroll
  for (int j = 0; j < JE_NSUM; ++j) acc[j] = 0.0;
  for (int i = tid; i < K; i += JR_THREADS) {
    const float4 nr = a.q_nrm[q + i];
    const double d = a.dist[q + i];
    const bool kp = (double)nr.w >= a.min_planarity && fabs(d - med) <= lim;
    a.keep[q + i] = kp ? 1 : 0;
    if (!kp) continue;
    const double u0 = a.m_xyz[3 * (q + i) + 0] - cm0, u1 = a.m_xyz[3 * (q + i) + 1] - cm1,
                 u2 = a.m_xyz[3 * (q + i) + 2] - cm2;
    const double w0 = R.r[0] * u0 + R.r[1] * u1 + R.r[2] * u2;
    const double w1 = R.r[3] * u0 + R.r[4] * u1 + R.r[5] * u2;
    const double w2 = R.r[6] * u0 + R.r[7] * u1 + R.r[8] * u2;
    const double n0 = (double)nr.x, n1 = (double)nr.y, n2 = (double)nr.z;
    const double row[6] = {w1 * n2 - w2 * n1, w2 * n0 - w0 * n2, w0 * n1 - w1 * n0, n0, n1, n2};
#pragma unroll
    for (int r = 0; r < 6; ++r) {
#pragma unroll
      for (int c = 0; c <= r; ++c) acc[tri(r, c)] = fma(row[r], row[c], acc[tri(r, c)]);
      acc[21 + r] = fma(row[r], d, acc[21 + r]);
      acc[27 + r] += row[r];
    }
    acc[33] += d;
    acc[34] = fma(d, d, acc[34]);
    acc[35] += 1.0;
  }
#pragma unroll
  for (int j = 0; j < JE_NSUM; ++j) {
    const double v = warp_sum(acc[j]);
    if (lane == 0) red[warp][j] = v;
  }
  __syncthreads();
  if (tid < JE_NSUM) {
    double v = 0.0;
    for (int w = 0; w < JR_WARPS; ++w) v += red[w][tid];
    tot[tid] = v;
  }
  __syncthreads();
  if (tid != 0) return;

  JointEdge& je = a.edges[e];
  const long long n = (long long)(tot[35] + 0.5);
  const double mean_d = n > 0 ? tot[33] / (double)n : nan("");
  const double var_d1 = n > 1 ? fmax(tot[34] - (double)n * mean_d * mean_d, 0.0) / (double)(n - 1) : nan("");
  sicp_iter_record* rec = a.rec + (size_t)e * a.rec_stride + a.it;
  rec->n_kept = n;
  rec->median = med;
  rec->mad = mad;
  rec->mean_dist = mean_d;
  rec->std_dist = sqrt(var_d1);
  rec->distance_weight = 1.0;
  rec->lm_iterations = n >= 6 ? 1 : 0;
  rec->n_bruteforce = 0;
  je.part = n >= 6 ? 1 : 0;
  je.n = n;
  for (int j = 0; j < 21; ++j) je.N[j] = tot[j];
  for (int j = 0; j < 6; ++j) {
    je.h[j] = tot[21 + j];
    je.s[j] = tot[27 + j];
  }
  je.sd = tot[33];
  je.sd2 = tot[34];
  // the edge centre in frame a and in the world, and the rotation of cloud a's pose: Ad
  double cf[3], wc[3];
  rigid_apply(R, cm0, cm1, cm2, cf[0], cf[1], cf[2]);
  const Rigid& Ta = a.pose[a.fix_id[e]];
  rigid_apply(Ta, cf[0], cf[1], cf[2], wc[0], wc[1], wc[2]);
  for (int j = 0; j < 3; ++j) {
    je.cf[j] = cf[j];
    je.v[j] = wc[j] - a.cw[j];
  }
  for (int j = 0; j < 9; ++j) je.Ra[j] = Ta.r[j];
  // columns of Ad: Ad e_k, then N Ad and Ad^T N Ad, Ad^T (-h)
  double Ad[6][6], NA[6][6];
  for (int k = 0; k < 6; ++k) {
    double y[6] = {0, 0, 0, 0, 0, 0}, col[6];
    y[k] = 1.0;
    ad_apply(je.Ra, je.v, y, col);
    for (int r = 0; r < 6; ++r) Ad[r][k] = col[r];
  }
  for (int r = 0; r < 6; ++r)
    for (int k = 0; k < 6; ++k) {
      double v = 0.0;
      for (int m = 0; m < 6; ++m) v = fma(je.N[r >= m ? tri(r, m) : tri(m, r)], Ad[m][k], v);
      NA[r][k] = v;
    }
  for (int r = 0; r < 6; ++r) {
    for (int k = 0; k <= r; ++k) {
      double v = 0.0;
      for (int m = 0; m < 6; ++m) v = fma(Ad[m][r], NA[m][k], v);
      je.Nw[r * 6 + k] = v;
      je.Nw[k * 6 + r] = v;
    }
    double g = 0.0;
    for (int m = 0; m < 6; ++m) g = fma(Ad[m][r], -je.h[m], g);
    je.gw[r] = g;
  }
}

// Grid barrier of the cooperative k_joint_solve (every block resident): bar[0] arrivals, bar[1]
// generation; the fences make the tiles other blocks wrote visible after it.
__device__ void joint_grid_sync(unsigned int* bar) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int gen = *(volatile unsigned int*)(bar + 1);
    if (atomicAdd(bar, 1u) == gridDim.x - 1u) {
      *(volatile unsigned int*)bar = 0u;
      __threadfence();
      atomicAdd(bar + 1, 1u);
    } else {
      while (*(volatile unsigned int*)(bar + 1) == gen) __nanosleep(64);
    }
    __threadfence();
  }
  __syncthreads();
}

struct SolveSmem {
  double t0[TS][TS + 1];
  double t1[TS][TS + 1];
  double xs[JOINT_MAX_PAD];
  int bad;
  int conv;
};

__device__ void load_tile(double (&t)[TS][TS + 1], const double* A, int npad, int ti, int tj) {
  for (int e = threadIdx.x; e < TS * TS; e += JS_THREADS)
    t[e / TS][e % TS] = __ldcg(&A[(size_t)(ti * TS + e / TS) * npad + tj * TS + e % TS]);
}
__device__ void store_tile(const double (&t)[TS][TS + 1], double* A, int npad, int ti, int tj) {
  for (int e = threadIdx.x; e < TS * TS; e += JS_THREADS)
    __stcg(&A[(size_t)(ti * TS + e / TS) * npad + tj * TS + e % TS], t[e / TS][e % TS]);
}

__device__ __forceinline__ double change_pct(double v, double v0) {
  return (v0 == 0.0) ? ((v == 0.0) ? 0.0 : kInf) : fabs((v - v0) / v0 * 100.0);
}

// ---- the tail of an iteration, shared by k_joint_solve and k_joint_sparse_solve --------------------

// poses: T_c <- dH(x_c) T_c for free cloud f, x_c = (omega, t' - omega x c_w), y = (omega, t')
__device__ __forceinline__ void joint_pose_update(const JointArgs& a, int f, const double* y) {
  const double x[6] = {y[0], y[1], y[2], y[3] - (y[1] * a.cw[2] - y[2] * a.cw[1]),
                       y[4] - (y[2] * a.cw[0] - y[0] * a.cw[2]), y[5] - (y[0] * a.cw[1] - y[1] * a.cw[0])};
  Rigid& T = a.pose[a.free_ids[f]];
  T = rigid_compose(rigid_from_x(x), T);
}

// edge e after the pose update, as the body of a loop over the edges: new relative transform,
// increment, residual statistics, record, stop rule, from xs (6 per free cloud, in free-cloud order);
// conv is cleared when the edge takes part and does not meet the stop rule.  A macro rather than a
// function, so that k_joint_solve compiles to the instructions it had before it shared this code.
#define JOINT_EDGE_UPDATE(a, e, xs, conv)                                                                                \
  {                                                                                                                      \
    DevState& st = a.state[e];                                                                                           \
    if (st.stop) continue;                                                                                               \
    const JointEdge& je = a.edges[e];                                                                                    \
    const int ca = a.fix_id[e], cb = a.mov_id[e];                                                                        \
    const Rigid Rold = st.T;                                                                                             \
    const Rigid Rn = rigid_compose(rigid_inverse(a.pose[ca]), a.pose[cb]);                                               \
    st.T = Rn;                                                                                                           \
    st.Tinv = rigid_inverse(Rn);                                                                                         \
    st.H_rep = Rn;                                                                                                       \
    st.T_new = Rn;                                                                                                       \
    st.T_res = Rn;                                                                                                       \
    st.n_kept = je.n;                                                                                                    \
    st.iterations_done = a.it + 1;                                                                                       \
    st.lm_ok = 1;                                                                                                        \
    for (int j = 0; j < 6; ++j) st.sigma[j] = nan("");                                                                   \
    if (!je.part) continue;                                                                                              \
    const int fa = a.free_of[ca], fb = a.free_of[cb];                                                                    \
    double y[6], xi[6];                                                                                                  \
    for (int j = 0; j < 6; ++j) y[j] = (fb >= 0 ? xs[6 * fb + j] : 0.0) - (fa >= 0 ? xs[6 * fa + j] : 0.0);              \
    ad_apply(je.Ra, je.v, y, xi);                                                                                        \
    /* residuals a . xi + d of the kept rows: their sum and sum of squares from the sums */                           \
    double sr = je.sd, quad = 0.0, lin = 0.0;                                                                            \
    for (int r = 0; r < 6; ++r) {                                                                                        \
      sr = fma(je.s[r], xi[r], sr);                                                                                      \
      lin = fma(je.h[r], xi[r], lin);                                                                                    \
      double row = 0.0;                                                                                                  \
      for (int c = 0; c < 6; ++c) row = fma(je.N[r >= c ? tri(r, c) : tri(c, r)], xi[c], row);                           \
      quad = fma(row, xi[r], quad);                                                                                      \
    }                                                                                                                    \
    const double nn = (double)je.n;                                                                                      \
    const double mean = sr / nn;                                                                                         \
    const double sr2 = quad + 2.0 * lin + je.sd2;                                                                        \
    const double sd = sqrt(fmax(sr2 - nn * mean * mean, 0.0) / (nn - 1.0));                                              \
    /* the origin-based increment of frame a: t = t_c - alpha x c_f */                                                \
    const double ex[6] = {xi[0], xi[1], xi[2], xi[3] - (xi[1] * je.cf[2] - xi[2] * je.cf[1]),                            \
                          xi[4] - (xi[2] * je.cf[0] - xi[0] * je.cf[2]), xi[5] - (xi[0] * je.cf[1] - xi[1] * je.cf[0])}; \
    Rigid L;                                                                                                             \
    L.r[0] = 1.0; L.r[1] = -ex[2]; L.r[2] = ex[1];                                                                       \
    L.r[3] = ex[2]; L.r[4] = 1.0; L.r[5] = -ex[0];                                                                       \
    L.r[6] = -ex[1]; L.r[7] = ex[0]; L.r[8] = 1.0;                                                                       \
    L.t[0] = ex[3]; L.t[1] = ex[4]; L.t[2] = ex[5];                                                                      \
    st.T_res = rigid_compose(L, Rold);                                                                                   \
    sicp_iter_record* rec = a.rec + (size_t)e * a.rec_stride + a.it;                                                     \
    for (int j = 0; j < 6; ++j) {                                                                                        \
      rec->x[j] = ex[j];                                                                                                 \
      st.x_new[j] = ex[j];                                                                                               \
    }                                                                                                                    \
    rec->mean_res = mean;                                                                                                \
    rec->std_res = sd;                                                                                                   \
    const bool stop = change_pct(mean, st.prev_mean) < a.min_change && change_pct(sd, st.prev_std) < a.min_change;       \
    if (!stop) conv = 0;                                                                                                 \
    st.prev_mean = mean;                                                                                                 \
    st.prev_std = sd;                                                                                                    \
  }

// edge e when the call ends at this iteration (conv: every edge met the stop rule)
__device__ __forceinline__ void joint_edge_finish(const JointArgs& a, int e, int conv) {
  DevState& st = a.state[e];
  if (st.stop) return;
  st.converged = conv;
  st.stop = a.edges[e].part ? (conv ? 1 : 0) : 2;
}

// relative observation o's term of the block of free clouds (fr row, fc column), entry (ri, cj)
__device__ __forceinline__ double rel_entry(const JointRel& o, int fr, int fc, int ri, int cj) {
  if (fr == fc) return o.N[fr == o.fa ? 0 : 1][6 * ri + cj];
  return fr == o.fb ? o.N[2][6 * ri + cj] : o.N[2][6 * cj + ri];
}

__global__ void __launch_bounds__(JS_THREADS) k_joint_solve(const JointArgs a, const JointRelArgs ro) {
  __shared__ SolveSmem sm;
  const int tid = threadIdx.x, bid = blockIdx.x, G = gridDim.x;
  if (a.flags->done) return;  // uniform: only block 0 writes it, at the very end of this launch
  const int n = 6 * a.F, npad = a.npad, KT = npad / TS;
  double* A = a.A;

  // ---- assembly of the lower triangle: edge blocks in ascending edge order, then the prior, then
  // the relative observations in ascending order; the right-hand side as row n, identity padding
  for (long long idx = (long long)bid * JS_THREADS + tid; idx < (long long)npad * npad; idx += (long long)G * JS_THREADS) {
    const int i = (int)(idx / npad), j = (int)(idx % npad);
    if (j > i) continue;
    double v = 0.0;
    if (i < n) {
      const int p = i / 6, qq = j / 6, ri = i % 6, cj = j % 6;
      const int b = a.blk_of[p * a.F + qq];
      if (b >= 0)
        for (int l = a.blk_off[b]; l < a.blk_off[b + 1]; ++l) {
          const JointEdge& je = a.edges[a.blk_edge[l] >> 1];
          if (je.part) v += (p == qq) ? je.Nw[ri * 6 + cj] : -je.Nw[ri * 6 + cj];
        }
      if (p == qq && a.prior_of && a.prior_of[p] >= 0) v += a.prior[a.prior_of[p]].Nw[ri * 6 + cj];
      if (ro.off && b >= 0)
#pragma unroll 1
        for (int l = ro.off[b]; l < ro.off[b + 1]; ++l) v += rel_entry(ro.rel[ro.k[l]], p, qq, ri, cj);
    } else if (i == n && j < n) {
      const int p = j / 6, b = a.blk_of[p * a.F + p];
      if (b >= 0)  // none: a cloud whose edges all lost their overlap, held by its prior
        for (int l = a.blk_off[b]; l < a.blk_off[b + 1]; ++l) {
          const JointEdge& je = a.edges[a.blk_edge[l] >> 1];
          if (je.part) v += (a.blk_edge[l] & 1) ? -je.gw[j % 6] : je.gw[j % 6];
        }
      if (a.prior_of && a.prior_of[p] >= 0) v += a.prior[a.prior_of[p]].gw[j % 6];
      if (ro.off && b >= 0)  // none: a cloud held by its prior alone
        for (int l = ro.off[b]; l < ro.off[b + 1]; ++l) {
          const JointRel& o = ro.rel[ro.k[l]];
          v += o.g[p == o.fa ? 0 : 1][j % 6];
        }
    } else if (i == j) {
      v = 1.0;
    }
    __stcg(&A[(size_t)i * npad + j], v);
  }
  if (tid == 0) sm.bad = 0;
  joint_grid_sync(a.bar);

  // ---- right-looking tiled Cholesky of the augmented matrix
  for (int k = 0; k < KT; ++k) {
    if (bid == 0) {
      load_tile(sm.t0, A, npad, k, k);
      __syncthreads();
      for (int j = 0; j < TS; ++j) {
        const int gj = k * TS + j;
        if (tid == 0) {
          double d = sm.t0[j][j];
          if (gj < n) {
            if (!(d > 0.0) || !isfinite(d)) sm.bad = 1;
          } else {
            d = 1.0;  // the right-hand side's row and the padding
          }
          sm.t0[j][j] = sqrt(d);
        }
        __syncthreads();
        if (tid > j && tid < TS) sm.t0[tid][j] /= sm.t0[j][j];
        __syncthreads();
        for (int e = tid; e < TS * TS; e += JS_THREADS) {
          const int r = e / TS, c = e % TS;
          if (c > j && r >= c) sm.t0[r][c] = fma(-sm.t0[r][j], sm.t0[c][j], sm.t0[r][c]);
        }
        __syncthreads();
      }
      store_tile(sm.t0, A, npad, k, k);
    }
    joint_grid_sync(a.bar);
    // panel: X L_kk^T = A_ik for every tile below the diagonal tile
    for (int i = k + 1 + bid; i < KT; i += G) {
      load_tile(sm.t0, A, npad, k, k);
      load_tile(sm.t1, A, npad, i, k);
      __syncthreads();
      if (tid < TS)
        for (int j = 0; j < TS; ++j) {
          double v = sm.t1[tid][j];
          for (int m = 0; m < j; ++m) v = fma(-sm.t1[tid][m], sm.t0[j][m], v);
          sm.t1[tid][j] = v / sm.t0[j][j];
        }
      __syncthreads();
      store_tile(sm.t1, A, npad, i, k);
      __syncthreads();
    }
    joint_grid_sync(a.bar);
    // trailing update A_ij -= L_ik L_jk^T, k < j <= i
    const int m = KT - k - 1;
    for (int t = bid; t < m * (m + 1) / 2; t += G) {
      int ii = 0;
      while ((ii + 1) * (ii + 2) / 2 <= t) ++ii;
      const int jj = t - ii * (ii + 1) / 2, ti = k + 1 + ii, tj = k + 1 + jj;
      load_tile(sm.t0, A, npad, ti, k);
      load_tile(sm.t1, A, npad, tj, k);
      __syncthreads();
      for (int e = tid; e < TS * TS; e += JS_THREADS) {
        const int r = e / TS, c = e % TS;
        double s = 0.0;
        for (int mm = 0; mm < TS; ++mm) s = fma(sm.t0[r][mm], sm.t1[c][mm], s);
        double* dst = &A[(size_t)(ti * TS + r) * npad + tj * TS + c];
        __stcg(dst, __ldcg(dst) - s);
      }
      __syncthreads();
    }
    joint_grid_sync(a.bar);
  }
  if (bid != 0) return;

  // ---- back substitution L^T y = L^-1 b (row n of the factor), block 0
  for (int i = tid; i < n; i += JS_THREADS) sm.xs[i] = __ldcg(&A[(size_t)n * npad + i]);
  __syncthreads();
  if (sm.bad) {
    if (tid == 0) {
      a.flags->singular = 1;
      a.flags->done = 1;
    }
    return;
  }
  for (int k = (n - 1) / TS; k >= 0; --k) {
    const int lo = k * TS, hi = min(lo + TS, n);
    if (tid < 32) {
      for (int r = hi - 1; r >= lo; --r) {
        const double xr = sm.xs[r] / __ldcg(&A[(size_t)r * npad + r]);
        __syncwarp();
        if (lo + tid < r) sm.xs[lo + tid] = fma(-__ldcg(&A[(size_t)r * npad + lo + tid]), xr, sm.xs[lo + tid]);
        if (tid == 0) sm.xs[r] = xr;
        __syncwarp();
      }
    }
    __syncthreads();
    for (int mcol = tid; mcol < lo; mcol += JS_THREADS) {
      double v = sm.xs[mcol];
      for (int r = lo; r < hi; ++r) v = fma(-__ldcg(&A[(size_t)r * npad + mcol]), sm.xs[r], v);
      sm.xs[mcol] = v;
    }
    __syncthreads();
  }

  // ---- poses, then the edges' new relative transforms, records and stop rule
  for (int f = tid; f < a.F; f += JS_THREADS) {
    joint_pose_update(a, f, sm.xs + 6 * f);
    if (a.prior_of && a.prior_of[f] >= 0)
      for (int q = 0; q < 6; ++q) a.prior[a.prior_of[f]].y[q] = sm.xs[6 * f + q];
    if (ro.y)
      for (int q = 0; q < 6; ++q) ro.y[6 * f + q] = sm.xs[6 * f + q];
  }
  __syncthreads();
  int conv = a.it > 0 ? 1 : 0;
  for (int e = tid; e < a.n_edges; e += JS_THREADS) JOINT_EDGE_UPDATE(a, e, sm.xs, conv)
  conv = __syncthreads_and(conv);
  const bool finish = conv || a.last;
  if (finish)
    for (int e = tid; e < a.n_edges; e += JS_THREADS) joint_edge_finish(a, e, conv);
  if (tid == 0) {
    a.flags->converged = conv;
    a.flags->done = finish ? 1 : 0;
  }
}
// ---- k_joint_sparse_solve: the supernodal Cholesky of joint_plan.h (DESIGN.md §6.11) -----------------

// Column k of edge e's Ad for a cloud whose increment (omega, u) is taken about its own origin o:
// Ad with the lever v - d = T_a c_f - o (d = o - c_w), metres where v itself can be kilometres.
__device__ __forceinline__ void ad_column(const JointEdge& je, const double* d, int k, double (&col)[6]) {
  const double lever[3] = {je.v[0] - d[0], je.v[1] - d[1], je.v[2] - d[2]};
  double y[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  y[k] = 1.0;
  ad_apply(je.Ra, lever, y, col);
}

// Supernode k by the whole block: assembly of its panel P (column-major, R = 6 (ns + nt) + 1 rows,
// C = 6 ns columns, the right-hand side as row R - 1) from the edges in ascending edge order, then
// each cloud's pose prior on its diagonal block and right-hand side (k_joint_prior), then each
// block's relative observations in ascending order (k_joint_relative), each
// cloud's unknowns taken about its own origin: Ad_r^T N Ad_c and -Ad_c^T h from the edge's sums in
// frame a (ad_column), never from Nw / gw, whose kilometre levers about c_w cost precision that a
// change of variables after the fact cannot recover; the left-looking updates from its descendants
// in ascending order; the right-looking Cholesky of the diagonal block, whose column steps also
// divide the rows below it (the right-hand side's row is left holding L^-1 b).  A non-positive or
// non-finite pivot sets *bad.
__device__ void sparse_factor(const JointSparseArgs& s, int k) {
  const JointArgs& a = s.j;
  const int tid = threadIdx.x;
  const JointSuper& m = s.sn[k];
  const int ns = m.ns, C = 6 * ns, R = 6 * (ns + m.nt) + 1;
  double* P = s.L + s.panel[k];
  for (int idx = tid; idx < R * C; idx += JS_THREADS) {
    const int c = idx / R, r = idx % R, cj = c / 6;
    const double* dcol = s.dc + 3 * s.perm[m.first + cj];
    double v = 0.0;
    if (r < R - 1) {
      const int ri = r / 6, l = s.blk[m.table + ri * ns + cj];
      const int pr = ri < ns ? m.first + ri : s.st[m.st_off + ri - ns];
      const double* drow = s.dc + 3 * s.perm[pr];
      if (l >= 0)
        for (int q = s.lst_off[l]; q < s.lst_off[l + 1]; ++q) {
          const JointEdge& je = a.edges[s.lst_edge[q] >> 1];
          if (!je.part) continue;
          double ar[6], ac[6];
          ad_column(je, drow, r % 6, ar);
          ad_column(je, dcol, c % 6, ac);
          double w = 0.0;
          for (int x = 0; x < 6; ++x) {
            double row = 0.0;
            for (int y = 0; y < 6; ++y) row = fma(je.N[x >= y ? tri(x, y) : tri(y, x)], ac[y], row);
            w = fma(ar[x], row, w);
          }
          v += (ri == cj) ? w : -w;
        }
    } else {
      const int l = s.blk[m.table + cj * ns + cj];
      if (l >= 0)
        for (int q = s.lst_off[l]; q < s.lst_off[l + 1]; ++q) {
          const JointEdge& je = a.edges[s.lst_edge[q] >> 1];
          if (!je.part) continue;
          double ac[6];
          ad_column(je, dcol, c % 6, ac);
          double w = 0.0;
          for (int y = 0; y < 6; ++y) w = fma(ac[y], -je.h[y], w);
          v += (s.lst_edge[q] & 1) ? -w : w;
        }
    }
    P[(size_t)c * R + r] = v;
  }
  __syncthreads();
  if (a.prior_of) {  // each cloud's prior on its diagonal block and right-hand side
    for (int idx = tid; idx < 42 * ns; idx += JS_THREADS) {
      const int cj = idx / 42, q = idx % 42, pk = a.prior_of[s.perm[m.first + cj]];
      if (pk < 0) continue;
      const JointPrior& pr = a.prior[pk];
      if (q < 36) P[(size_t)(6 * cj + q % 6) * R + 6 * cj + q / 6] += pr.Nw[q];
      else P[(size_t)(6 * cj + q - 36) * R + R - 1] += pr.gw[q - 36];
    }
    __syncthreads();
  }
  if (s.r.off) {  // each block's relative observations in ascending order (rel_entry)
    for (int idx = tid; idx < (ns + m.nt) * C * 6 + C; idx += JS_THREADS) {
      const int bq = idx / 36, e = idx % 36, rhs = bq >= (ns + m.nt) * ns;
      const int ri = rhs ? (idx - 36 * (ns + m.nt) * ns) / 6 : bq / ns, cj = rhs ? ri : bq % ns;
      const int l = s.blk[m.table + ri * ns + cj];
      if (l < 0) continue;
      const int fc = s.perm[m.first + cj], r6 = rhs ? 0 : e / 6, c6 = rhs ? idx % 6 : e % 6;
      const int fr = s.perm[ri < ns ? m.first + ri : s.st[m.st_off + ri - ns]];
      double& x = P[(size_t)(6 * cj + c6) * R + (rhs ? R - 1 : 6 * ri + r6)];
      double v = x;
#pragma unroll 1
      for (int q = s.r.off[l]; q < s.r.off[l + 1]; ++q) {
        const JointRel& o = s.r.rel[s.r.k[q]];
        v += rhs ? o.g[fc == o.fa ? 0 : 1][c6] : rel_entry(o, fr, fc, r6, c6);
      }
      x = v;
    }
    __syncthreads();
  }
  // P[map(i), map(j)] -= sum_k Ld[i][k] Ld[j][k] over the rows i of descendant d from its first
  // struct entry in s on (and its right-hand side's row), the columns j of those inside s
  for (int u = m.u0; u < m.u1; ++u) {
    const int* up = s.up + 4 * u;
    const JointSuper& dm = s.sn[up[0]];
    const int Cd = 6 * dm.ns, Rd = 6 * (dm.ns + dm.nt) + 1, r0 = Cd + 6 * up[1];
    const int nr = Rd - r0, nj = 6 * up[2];
    const int* map = s.map + up[3];
    const double* Pd = s.L + s.panel[up[0]];
    for (int idx = tid; idx < nr * nj; idx += JS_THREADS) {
      const int i = idx % nr, j = idx / nr;
      const int ti = (i < nr - 1) ? 6 * map[i / 6] + i % 6 : R - 1, tj = 6 * map[j / 6] + j % 6;
      if (ti < tj) continue;  // above the diagonal
      double v = 0.0;
      for (int q = 0; q < Cd; ++q) v = fma(__ldcg(&Pd[(size_t)q * Rd + r0 + i]), __ldcg(&Pd[(size_t)q * Rd + r0 + j]), v);
      P[(size_t)tj * R + ti] -= v;
    }
    __syncthreads();
  }
  for (int j = 0; j < C; ++j) {
    const double d = P[(size_t)j * R + j];
    if (tid == 0 && (!(d > 0.0) || !isfinite(d))) *s.bad = 1;
    const double piv = sqrt(d);
    for (int r = j + 1 + tid; r < R; r += JS_THREADS) P[(size_t)j * R + r] /= piv;
    __syncthreads();
    if (tid == 0) P[(size_t)j * R + j] = piv;
    for (int r = j + 1 + tid; r < R; r += JS_THREADS) {
      const double lr = P[(size_t)j * R + r];
      const int ce = min(r, C - 1);
      for (int c = j + 1; c <= ce; ++c) P[(size_t)c * R + r] = fma(-lr, P[(size_t)j * R + c], P[(size_t)c * R + r]);
    }
    __syncthreads();
  }
}

// Supernode k by the whole block, after every ancestor: x_s = L_ss^-T (y_s - L_ts^T x_t), y_s its
// right-hand side's row, t its struct; the solution goes to xf in free-cloud order.
__device__ void sparse_back(const JointSparseArgs& s, int k) {
  const int tid = threadIdx.x;
  const JointSuper& m = s.sn[k];
  const int nt = m.nt, C = 6 * m.ns, R = 6 * (m.ns + nt) + 1;
  const double* P = s.L + s.panel[k];
  double* x = s.x + 6 * m.first;
  for (int c = tid; c < C; c += JS_THREADS) {
    double v = P[(size_t)c * R + R - 1];
    for (int r = 0; r < 6 * nt; ++r)
      v = fma(-P[(size_t)c * R + C + r], __ldcg(&s.xf[6 * s.perm[s.st[m.st_off + r / 6]] + r % 6]), v);
    x[c] = v;
  }
  __syncthreads();
  for (int c = C - 1; c >= 0; --c) {
    const double xc = x[c] / P[(size_t)c * R + c];
    for (int i = tid; i < c; i += JS_THREADS) x[i] = fma(-P[(size_t)i * R + c], xc, x[i]);
    if (tid == 0) s.xf[6 * s.perm[m.first + c / 6] + c % 6] = xc;
    __syncthreads();
  }
}

// One cooperative launch per iteration in place of k_joint_solve: the factor bottom-up by level and
// the back substitution top-down (one supernode per block, one grid barrier per level), then the
// tail of k_joint_solve spread over the grid.
__global__ void __launch_bounds__(JS_THREADS) k_joint_sparse_solve(const JointSparseArgs s) {
  __shared__ int conv_s;
  const JointArgs& a = s.j;
  const int tid = threadIdx.x, bid = blockIdx.x, G = gridDim.x;
  if (a.flags->done) return;  // uniform: only block 0 writes it, at the very end of this launch
  for (int l = 0; l < s.depth; ++l) {
    for (int i = s.lv_off[l] + bid; i < s.lv_off[l + 1]; i += G) sparse_factor(s, s.lv[i]);
    joint_grid_sync(a.bar);
  }
  if (__ldcg(s.bad)) {
    if (bid == 0 && tid == 0) {
      a.flags->singular = 1;
      a.flags->done = 1;
    }
    return;
  }
  for (int l = s.depth - 1; l >= 0; --l) {
    for (int i = s.lv_off[l] + bid; i < s.lv_off[l + 1]; i += G) sparse_back(s, s.lv[i]);
    joint_grid_sync(a.bar);
  }
  const int gt = bid * JS_THREADS + tid, GT = G * JS_THREADS;
  // (omega, u) about each cloud's centre -> (omega, t') about c_w, in place for the edges
  for (int f = gt; f < a.F; f += GT) {
    double y[6];
    for (int q = 0; q < 6; ++q) y[q] = __ldcg(&s.xf[6 * f + q]);
    const double* d = s.dc + 3 * f;
    y[3] += d[1] * y[2] - d[2] * y[1];
    y[4] += d[2] * y[0] - d[0] * y[2];
    y[5] += d[0] * y[1] - d[1] * y[0];
    for (int q = 3; q < 6; ++q) s.xf[6 * f + q] = y[q];
    joint_pose_update(a, f, y);
  }
  joint_grid_sync(a.bar);
  const double* xs = s.xf;
  int conv = a.it > 0 ? 1 : 0;
  for (int e = gt; e < a.n_edges; e += GT) JOINT_EDGE_UPDATE(a, e, xs, conv)
  conv = __syncthreads_and(conv);
  if (tid == 0) s.conv[bid] = conv;
  joint_grid_sync(a.bar);
  if (tid == 0) {
    int v = 1;
    for (int b = 0; b < G; ++b) v &= __ldcg(&s.conv[b]);
    conv_s = v;
  }
  __syncthreads();
  conv = conv_s;
  const bool finish = conv || a.last;
  if (finish)
    for (int e = gt; e < a.n_edges; e += GT) joint_edge_finish(a, e, conv);
  if (bid == 0 && tid == 0) {
    a.flags->converged = conv;
    a.flags->done = finish ? 1 : 0;
  }
}

// ---- sicp_get_joint_covariances: Cov(y) = s0^2 N^-1 = s0^2 Z^T Z with Z = L^-1 -------------------

constexpr int JC_THREADS = 256;
constexpr int JC_WARPS = JC_THREADS / 32;

// k_joint_cov_ss, one block per edge: ss[e] = the sum of the squared final residuals of the kept
// rows (final_residual: the values sicp_get_batch_outputs returns) of an edge that took part in the
// final iteration, else 0.
__global__ void __launch_bounds__(JC_THREADS) k_joint_cov_ss(const JointCovArgs a) {
  __shared__ double red[JC_WARPS];
  const int e = blockIdx.x, tid = threadIdx.x;
  double acc = 0.0;
  if (a.edges[e].part) {
    const PairDev& pd = a.pairs[e];
    const Rigid Tn = a.state[e].T_res;
    for (long long i = tid; i < pd.K; i += JC_THREADS)
      if (a.keep[pd.q_off + i]) {
        const double r = final_residual(Tn, a.m_xyz, a.q_xyz, a.q_nrm, pd.q_off + i);
        acc = fma(r, r, acc);
      }
  }
  acc = warp_sum(acc);
  if ((tid & 31) == 0) red[tid >> 5] = acc;
  __syncthreads();
  if (tid == 0) {
    double v = 0.0;
    for (int w = 0; w < JC_WARPS; ++w) v += red[w];
    a.ss[e] = v;
  }
}

// tile (ti, tj) of the factor of N: the rows and columns from n on are the identity's
__device__ void load_l_tile(double (&t)[TS][TS + 1], const double* L, int npad, int n, int ti, int tj) {
  for (int e = threadIdx.x; e < TS * TS; e += JS_THREADS) {
    const int r = ti * TS + e / TS, c = tj * TS + e % TS;
    t[e / TS][e % TS] = (r < n && c < n) ? L[(size_t)r * npad + c] : (r == c ? 1.0 : 0.0);
  }
}

// p[q] = (X Y)[r][c] for the element e = tid + q JS_THREADS, r = e / TS, c = e % TS
constexpr int TQ = TS * TS / JS_THREADS;
__device__ __forceinline__ void tile_mul(const double (&X)[TS][TS + 1], const double (&Y)[TS][TS + 1], double (&p)[TQ]) {
#pragma unroll
  for (int q = 0; q < TQ; ++q) {
    const int e = threadIdx.x + q * JS_THREADS, r = e / TS, c = e % TS;
    double s = 0.0;
#pragma unroll 8
    for (int m = 0; m < TS; ++m) s = fma(X[r][m], Y[m][c], s);
    p[q] = s;
  }
}

// k_joint_inv, one cooperative launch: Z = L^-1 by tiles.  First every diagonal tile Z_kk = L_kk^-1
// (forward substitution, one column per thread); then, for k = 0, 1, .., the right-looking update of
// the block rows below k: B_ij -= L_ik Z_kj for i > k, j <= k (B_ij starts at 0, so its first update,
// at k = j, is a store), and the tiles of row k + 1, whose sum is then complete, become
// Z_(k+1)j = Z_(k+1)(k+1) B_(k+1)j.  One grid barrier per k; each B_ij takes its updates in
// ascending k.  Only tiles on or below the diagonal are written.
__global__ void __launch_bounds__(JS_THREADS) k_joint_inv(const JointCovArgs a) {
  __shared__ double t0[TS][TS + 1];
  __shared__ double t1[TS][TS + 1];
  const int tid = threadIdx.x, bid = blockIdx.x, G = gridDim.x;
  const int n = 6 * a.F, npad = a.npad, KN = (n + TS - 1) / TS;
  for (int k = bid; k < KN; k += G) {
    load_l_tile(t0, a.L, npad, n, k, k);
    __syncthreads();
    if (tid < TS) {
      const int c = tid;
      for (int r = 0; r < TS; ++r) {
        double v = 0.0;
        if (r >= c) {
          v = (r == c) ? 1.0 : 0.0;
          for (int m = c; m < r; ++m) v = fma(-t0[r][m], t1[m][c], v);
          v /= t0[r][r];
        }
        t1[r][c] = v;
      }
    }
    __syncthreads();
    store_tile(t1, a.Z, npad, k, k);
    __syncthreads();
  }
  joint_grid_sync(a.bar);
  for (int k = 0; k + 1 < KN; ++k) {
    const int w = k + 1, cnt = (KN - 1 - k) * w;
    for (int t = bid; t < cnt; t += G) {
      const int i = k + 1 + t / w, j = t % w;
      load_l_tile(t0, a.L, npad, n, i, k);
      load_tile(t1, a.Z, npad, k, j);
      __syncthreads();
      double p[TQ], bv[TQ];
      tile_mul(t0, t1, p);
#pragma unroll
      for (int q = 0; q < TQ; ++q) {
        const int e = tid + q * JS_THREADS;
        const size_t at = (size_t)(i * TS + e / TS) * npad + j * TS + e % TS;
        bv[q] = (j == k) ? -p[q] : __ldcg(&a.Z[at]) - p[q];
      }
      if (i == k + 1) {
        __syncthreads();
        load_tile(t0, a.Z, npad, i, i);
#pragma unroll
        for (int q = 0; q < TQ; ++q) {
          const int e = tid + q * JS_THREADS;
          t1[e / TS][e % TS] = bv[q];
        }
        __syncthreads();
        tile_mul(t0, t1, bv);
      }
#pragma unroll
      for (int q = 0; q < TQ; ++q) {
        const int e = tid + q * JS_THREADS;
        __stcg(&a.Z[(size_t)(i * TS + e / TS) * npad + j * TS + e % TS], bv[q]);
      }
      __syncthreads();
    }
    joint_grid_sync(a.bar);
  }
}

// g[6 i + j] = sum over k >= max(c0, c1) of Z[k][c0 + i] Z[k][c1 + j] (a 6 x 6 block of Z^T Z), by
// the whole block: rows strided over the threads, then the warps' sums in warp order.  Z is lower
// triangular: an entry above the diagonal counts as 0 and is not read.
__device__ void gram6(const double* Z, int npad, int n, int c0, int c1, double (&red)[JC_WARPS][36], double* g) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double acc[36];
#pragma unroll
  for (int j = 0; j < 36; ++j) acc[j] = 0.0;
  for (int k = max(c0, c1) + tid; k < n; k += JC_THREADS) {
    const double* row = Z + (size_t)k * npad;
    double x[6], y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      x[i] = (k >= c0 + i) ? row[c0 + i] : 0.0;
      y[i] = (k >= c1 + i) ? row[c1 + i] : 0.0;
    }
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
      for (int j = 0; j < 6; ++j) acc[6 * i + j] = fma(x[i], y[j], acc[6 * i + j]);
  }
#pragma unroll
  for (int j = 0; j < 36; ++j) {
    const double v = warp_sum(acc[j]);
    if (lane == 0) red[warp][j] = v;
  }
  __syncthreads();
  if (tid < 36) {
    double v = 0.0;
    for (int w = 0; w < JC_WARPS; ++w) v += red[w][tid];
    g[tid] = v;
  }
  __syncthreads();
}

// out = A M B^T, 6 x 6 row-major
__device__ void abt6(const double* A, const double* M, const double* B, double* out) {
  double AM[36];
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      double v = 0.0;
      for (int m = 0; m < 6; ++m) v = fma(A[6 * r + m], M[6 * m + c], v);
      AM[6 * r + c] = v;
    }
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) {
      double v = 0.0;
      for (int m = 0; m < 6; ++m) v = fma(AM[6 * r + m], B[6 * c + m], v);
      out[6 * r + c] = v;
    }
}

// [[P, 0], [-P [d]x, P]] with P = I (Q null) or Q^T (Q a row-major rotation): J_c for d = o_c - c_w,
// G_a for Q = R_a, d = o_b - o_a
__device__ void lever6(const double* Q, const double* d, double* out) {
  double P[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) P[3 * r + c] = Q ? Q[3 * c + r] : (r == c ? 1.0 : 0.0);
  const double S[9] = {0.0, -d[2], d[1], d[2], 0.0, -d[0], -d[1], d[0], 0.0};
  for (int j = 0; j < 36; ++j) out[j] = 0.0;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double ps = 0.0;
      for (int m = 0; m < 3; ++m) ps = fma(P[3 * r + m], S[3 * m + c], ps);
      out[6 * r + c] = P[3 * r + c];
      out[6 * (r + 3) + c + 3] = P[3 * r + c];
      out[6 * (r + 3) + c] = -ps;
    }
}

// ---- k_joint_prior: the pose priors (DESIGN.md §6.12) -------------------------------------------------

// w = rotvec(M) for a rotation M (row-major): the angle in [0, pi] from atan2(|s|, (tr M - 1) / 2),
// s = vee(M - M^T) / 2 = sin(angle) n; the axis from s while the angle is below 2 pi / 3, else from
// the symmetric part (M + M^T) / 2 - cos I = (1 - cos) n n^T, turned to the side of s
__device__ void rotvec(const double* M, double* w) {
  const double s[3] = {0.5 * (M[7] - M[5]), 0.5 * (M[2] - M[6]), 0.5 * (M[3] - M[1])};
  const double sn = sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]);
  const double cs = 0.5 * (M[0] + M[4] + M[8] - 1.0);
  const double th = atan2(sn, cs);
  if (cs > -0.5) {
    const double k = sn > 0.0 ? th / sn : 1.0;
    for (int q = 0; q < 3; ++q) w[q] = k * s[q];
    return;
  }
  int kk = 0;
  for (int q = 1; q < 3; ++q)
    if (M[4 * q] > M[4 * kk]) kk = q;
  const double bkk = M[4 * kk] - cs;
  double n[3];
  for (int q = 0; q < 3; ++q) n[q] = (q == kk) ? bkk : 0.5 * (M[3 * q + kk] + M[3 * kk + q]);
  const double sc = 1.0 / sqrt(bkk * (1.0 - cs));
  const double sg = (n[0] * s[0] + n[1] * s[1] + n[2] * s[2]) < 0.0 ? -sc : sc;
  for (int q = 0; q < 3; ++q) w[q] = th * sg * n[q];
}

// one thread per prior k of free cloud f, at its current pose T_c: l = (rotvec(R_P R_c^T), o_P - o_c),
// the lever d = o_c - c_w - dc_f of J_c (dc null: the dense solve's unknowns about c_w; else the
// sparse solve's about each cloud's start origin), Nw = J^T W J and gw = J^T W l
__global__ void __launch_bounds__(128) k_joint_prior(const JointArgs a, const double* dc) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (a.flags->done || k >= a.n_prior) return;
  JointPrior& pr = a.prior[k];
  const int f = pr.f;
  const Rigid T = a.pose[a.free_ids[f]];
  double M[9], l[6], d[3], Jc[36];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      M[3 * r + c] = pr.P.r[3 * r + 0] * T.r[3 * c + 0] + pr.P.r[3 * r + 1] * T.r[3 * c + 1] +
                     pr.P.r[3 * r + 2] * T.r[3 * c + 2];
  rotvec(M, l);
  for (int q = 0; q < 3; ++q) {
    l[3 + q] = pr.P.t[q] - T.t[q];
    d[q] = (T.t[q] - a.cw[q]) - (dc ? dc[3 * f + q] : 0.0);
  }
  lever6(nullptr, d, Jc);
  for (int r = 0; r < 6; ++r) {
    for (int c = 0; c < 6; ++c) {
      double v = 0.0;
      for (int q = 0; q < 6; ++q) v = fma(Jc[6 * q + r] * pr.w[q], Jc[6 * q + c], v);
      pr.Nw[6 * r + c] = v;
    }
    double g = 0.0;
    for (int q = 0; q < 6; ++q) g = fma(Jc[6 * q + r] * pr.w[q], l[q], g);
    pr.gw[r] = g;
    pr.l[r] = l[r];
  }
  for (int q = 0; q < 3; ++q) pr.lev[q] = d[q];
}

// ---- k_joint_relative: the relative observations (DESIGN.md §6.13) ---------------------------------

// one thread per observation k of clouds a, b at their current poses: l = (rotvec(R_Z R_ab^T),
// t_Z - t_ab) with R_ab = R_a^T R_b, t_ab = R_a^T (o_b - o_a); per free end c the lever d_c of J_c
// (k_joint_prior's), B_c = G_c J_c with G_b = diag(R_a^T, R_a^T) and G_a = lever6(R_a, o_b - o_a);
// then the blocks B_c^T W B_c, -B_b^T W B_a and the right-hand sides -B_a^T W l, B_b^T W l
__global__ void __launch_bounds__(128) k_joint_relative(const JointArgs a, const JointRelArgs ro, const double* dc) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (a.flags->done || k >= ro.n) return;
  JointRel& o = ro.rel[k];
  const Rigid Ta = a.pose[o.ca], Tb = a.pose[o.cb];
  double Rab[9], M[9], l[6], dba[3];
  for (int q = 0; q < 3; ++q) dba[q] = Tb.t[q] - Ta.t[q];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      Rab[3 * r + c] = Ta.r[r] * Tb.r[c] + Ta.r[3 + r] * Tb.r[3 + c] + Ta.r[6 + r] * Tb.r[6 + c];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      M[3 * r + c] = o.Z.r[3 * r + 0] * Rab[3 * c + 0] + o.Z.r[3 * r + 1] * Rab[3 * c + 1] +
                     o.Z.r[3 * r + 2] * Rab[3 * c + 2];
  rotvec(M, l);
  for (int q = 0; q < 3; ++q) l[3 + q] = o.Z.t[q] - (Ta.r[q] * dba[0] + Ta.r[3 + q] * dba[1] + Ta.r[6 + q] * dba[2]);
  double B[2][36];
  for (int e = 0; e < 2; ++e) {
    const int f = e ? o.fb : o.fa;
    const Rigid& T = e ? Tb : Ta;
    double d[3], Jc[36], G[36];
    for (int q = 0; q < 3; ++q) {
      d[q] = (T.t[q] - a.cw[q]) - (dc && f >= 0 ? dc[3 * f + q] : 0.0);
      o.lev[e][q] = d[q];
    }
    if (f < 0) continue;
    const double zero[3] = {0.0, 0.0, 0.0};
    lever6(nullptr, d, Jc);
    lever6(Ta.r, e ? zero : dba, G);
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) {
        double v = 0.0;
        for (int m = 0; m < 6; ++m) v = fma(G[6 * r + m], Jc[6 * m + c], v);
        B[e][6 * r + c] = v;
      }
    for (int r = 0; r < 6; ++r) {
      for (int c = 0; c < 6; ++c) {
        double v = 0.0;
        for (int q = 0; q < 6; ++q) v = fma(B[e][6 * q + r] * o.w[q], B[e][6 * q + c], v);
        o.N[e][6 * r + c] = v;
      }
      double g = 0.0;
      for (int q = 0; q < 6; ++q) g = fma(B[e][6 * q + r] * o.w[q], l[q], g);
      o.g[e][r] = e ? g : -g;
    }
  }
  if (o.fa >= 0 && o.fb >= 0)
    for (int r = 0; r < 6; ++r)
      for (int c = 0; c < 6; ++c) {
        double v = 0.0;
        for (int q = 0; q < 6; ++q) v = fma(B[1][6 * q + r] * o.w[q], B[0][6 * q + c], v);
        o.N[2][6 * r + c] = -v;
      }
  for (int q = 0; q < 6; ++q) o.l[q] = l[q];
  for (int q = 0; q < 3; ++q) o.dba[q] = dba[q];
  for (int q = 0; q < 9; ++q) o.Ra[q] = Ta.r[q];
}

// the lower triangle of C mirrored, NaN everywhere when s0^2 is
__device__ void store_sym6(const double* C, double s0sq, double* out) {
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c <= r; ++c) {
      const double v = (s0sq == s0sq) ? C[6 * r + c] : s0sq;
      out[6 * r + c] = v;
      out[6 * c + r] = v;
    }
}

// s0^2's sums by warp 0 (lane: the thread's lane; every lane ends with the totals ss and m): over
// the edges that took part, ss[e] and the kept counts; then the pose priors' v^T W v and non-zero
// weights (DESIGN.md §6.12); then the relative observations' (§6.13).  Their residuals v use the
// final unknowns (pr.y, rel_y) in the variables of the levers pr.lev, o.lev: the solve's.  A macro
// rather than a function, so that k_joint_cov_cloud compiles to the instructions it had before it
// shared this statement with k_joint_sel_s0.
#define JOINT_S0_SUMS(a, lane, ss, m)                                                                                   \
  double ss = 0.0, m = 0.0;                                                                                             \
  for (int e = lane; e < a.n_edges; e += 32)                                                                            \
    if (a.edges[e].part) {                                                                                              \
      ss += a.ss[e];                                                                                                    \
      m += (double)a.edges[e].n;                                                                                        \
    }                                                                                                                   \
  /* the pose priors: v^T W v with v = J y - l, and their non-zero weights (DESIGN.md §6.12) */                         \
  for (int k = lane; k < a.n_prior; k += 32) {                                                                          \
    const JointPrior& pr = a.prior[k];                                                                                  \
    const double* y = pr.y;                                                                                             \
    const double* d = pr.lev;                                                                                           \
    const double u[6] = {y[0], y[1], y[2], y[3] - (d[1] * y[2] - d[2] * y[1]), y[4] - (d[2] * y[0] - d[0] * y[2]),      \
                         y[5] - (d[0] * y[1] - d[1] * y[0])};                                                           \
    for (int q = 0; q < 6; ++q)                                                                                         \
      if (pr.w[q] != 0.0) {                                                                                             \
        const double v = u[q] - pr.l[q];                                                                                \
        ss = fma(pr.w[q] * v, v, ss);                                                                                   \
        m += 1.0;                                                                                                       \
      }                                                                                                                 \
  }                                                                                                                     \
  /* the relative observations: v = G_b J_b y_b - G_a J_a y_a - l, after the priors (DESIGN.md §6.13) */                \
  for (int k = lane; k < a.n_rel; k += 32) {                                                                            \
    const JointRel& o = a.rel[k];                                                                                       \
    double pu[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};  /* R_a u */                                                         \
    for (int e = 1; e >= 0; --e) {                                                                                      \
      const int f = e ? o.fb : o.fa;                                                                                    \
      if (f < 0) continue;                                                                                              \
      const double* y = a.rel_y + 6 * f;                                                                                \
      const double* d = o.lev[e];                                                                                       \
      const double u[6] = {y[0], y[1], y[2], y[3] - (d[1] * y[2] - d[2] * y[1]), y[4] - (d[2] * y[0] - d[0] * y[2]),    \
                           y[5] - (d[0] * y[1] - d[1] * y[0])};                                                         \
      const double* b = o.dba;                                                                                          \
      for (int q = 0; q < 3; ++q) {                                                                                     \
        pu[q] += e ? u[q] : -u[q];                                                                                      \
        pu[3 + q] += e ? u[3 + q] : -(u[3 + q] - (b[(q + 1) % 3] * u[(q + 2) % 3] - b[(q + 2) % 3] * u[(q + 1) % 3]));  \
      }                                                                                                                 \
    }                                                                                                                   \
    for (int q = 0; q < 6; ++q)                                                                                         \
      if (o.w[q] != 0.0) {                                                                                              \
        const int h = q < 3 ? 0 : 3, r = q - h;                                                                         \
        const double v = (o.Ra[r] * pu[h] + o.Ra[3 + r] * pu[h + 1] + o.Ra[6 + r] * pu[h + 2]) - o.l[q];                \
        ss = fma(o.w[q] * v, v, ss);                                                                                    \
        m += 1.0;                                                                                                       \
      }                                                                                                                 \
  }                                                                                                                     \
  ss = warp_sum(ss);                                                                                                    \
  m = warp_sum(m);

// k_joint_cov_cloud, one block per free cloud p: s0^2 from the edges' sums (warp 0, fixed order;
// block 0 stores it), the diagonal block (N^-1)_pp and C_c = s0^2 J_c (N^-1)_pp J_c^T
__global__ void __launch_bounds__(JC_THREADS) k_joint_cov_cloud(const JointCovArgs a) {
  __shared__ double red[JC_WARPS][36];
  __shared__ double g[36];
  __shared__ double s0sq_s;
  const int p = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const int n = 6 * a.F;
  if (tid < 32) {
    JOINT_S0_SUMS(a, lane, ss, m)
    if (lane == 0) {
      const double dof = m - (double)n;
      s0sq_s = dof > 0.0 ? ss / dof : nan("");
      if (p == 0) *a.s0sq = s0sq_s;
    }
  }
  gram6(a.Z, a.npad, n, 6 * p, 6 * p, red, g);
  if (tid != 0) return;
  const Rigid& T = a.pose[a.free_ids[p]];
  const double d[3] = {T.t[0] - a.cw[0], T.t[1] - a.cw[1], T.t[2] - a.cw[2]};
  double Jc[36], C[36], M[36];
  lever6(nullptr, d, Jc);
  for (int j = 0; j < 36; ++j) M[j] = s0sq_s * g[j];
  abt6(Jc, M, Jc, C);
  store_sym6(C, s0sq_s, a.cov_f + 36 * (size_t)p);
}

// C_e of edge e = (a, b) from g = (N^-1)_ab (read with both clouds free): C_ab = s0^2 J_a g J_b^T; then
// C_e = G_b C_b G_b^T + G_a C_a G_a^T - M - M^T, M = G_a C_ab G_b^T, at the returned poses (a fixed
// cloud's blocks are 0).  dc: nullptr for the dense solve's unknowns about c_w, else the sparse solve's
// start origins minus c_w, whose J'_c take the lever o_c - o_c^0.  A macro rather than a function, so
// that k_joint_cov_edge compiles to the instructions it had before it shared this statement.
#define JOINT_EDGE_COV(a, e, ca, cb, fa, fb, g, dc)                                                                   \
  {                                                                                                                   \
  const double s0sq = *a.s0sq;                                                                                        \
  const Rigid &Ta = a.pose[ca], &Tb = a.pose[cb];                                                                     \
  const double dba[3] = {Tb.t[0] - Ta.t[0], Tb.t[1] - Ta.t[1], Tb.t[2] - Ta.t[2]}, zero[3] = {0.0, 0.0, 0.0};         \
  double Ga[36], Gb[36], C[36], X[36];                                                                                \
  lever6(Ta.r, dba, Ga);                                                                                              \
  lever6(Ta.r, zero, Gb);                                                                                             \
  for (int j = 0; j < 36; ++j) C[j] = 0.0;                                                                            \
  if (fb >= 0) {                                                                                                      \
    abt6(Gb, a.cov_f + 36 * (size_t)fb, Gb, X);                                                                       \
    for (int j = 0; j < 36; ++j) C[j] += X[j];                                                                        \
  }                                                                                                                   \
  if (fa >= 0) {                                                                                                      \
    abt6(Ga, a.cov_f + 36 * (size_t)fa, Ga, X);                                                                       \
    for (int j = 0; j < 36; ++j) C[j] += X[j];                                                                        \
  }                                                                                                                   \
  if (fa >= 0 && fb >= 0) {                                                                                           \
    const Rigid &Pa = a.pose[ca], &Pb = a.pose[cb];                                                                   \
    double da[3] = {Pa.t[0] - a.cw[0], Pa.t[1] - a.cw[1], Pa.t[2] - a.cw[2]},                                         \
           db[3] = {Pb.t[0] - a.cw[0], Pb.t[1] - a.cw[1], Pb.t[2] - a.cw[2]};                                         \
    if (dc != nullptr)                                                                                                        \
      for (int q = 0; q < 3; ++q) {                                                                                   \
        da[q] -= (dc)[3 * fa + q];                                                                                      \
        db[q] -= (dc)[3 * fb + q];                                                                                      \
      }                                                                                                               \
    double Ja[36], Jb[36], Cab[36], M[36];                                                                            \
    lever6(nullptr, da, Ja);                                                                                          \
    lever6(nullptr, db, Jb);                                                                                          \
    for (int j = 0; j < 36; ++j) M[j] = s0sq * g[j];                                                                  \
    abt6(Ja, M, Jb, Cab);                                                                                             \
    abt6(Ga, Cab, Gb, M);                                                                                             \
    for (int r = 0; r < 6; ++r)                                                                                       \
      for (int c = 0; c < 6; ++c) C[6 * r + c] -= M[6 * r + c] + M[6 * c + r];                                        \
  }                                                                                                                   \
  store_sym6(C, s0sq, a.cov_e + 36 * (size_t)e);                                                                      \
  }

// k_joint_cov_edge, one block per edge e = (a, b): with both clouds free the cross block
// (N^-1)_ab by gram6, then C_e (joint_edge_cov)
__global__ void __launch_bounds__(JC_THREADS) k_joint_cov_edge(const JointCovArgs a) {
  __shared__ double red[JC_WARPS][36];
  __shared__ double g[36];
  const int e = blockIdx.x, tid = threadIdx.x;
  const int ca = a.fix_id[e], cb = a.mov_id[e], fa = a.free_of[ca], fb = a.free_of[cb];
  if (fa >= 0 && fb >= 0) gram6(a.Z, a.npad, 6 * a.F, 6 * fa, 6 * fb, red, g);
  if (tid != 0) return;
  JOINT_EDGE_COV(a, e, ca, cb, fa, fb, g, (const double*)nullptr)
}

// ---- sicp_get_joint_selected_covariances after a sparse call: Z = N'^-1 on the pattern of L ----------
// (DESIGN.md §6.14).  Supernode k's block of Z has the rows of its factor panel without the right-hand
// side's (Rz = 6 (ns + nt)) and the same columns: Z_JJ in full (both triangles), then Z_TJ.

constexpr int SEL_MAX_PATH = JOINT_SEL_MAX_PATH;  // supernodes on a path to a root, at most

// the supernode holding position p: the last k with first[k] <= p (supernodes in elimination order)
__device__ int sel_owner(const JointSparseArgs& s, int p) {
  int lo = 0, hi = s.lv_off[s.depth];
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (s.sn[mid].first <= p) lo = mid;
    else hi = mid;
  }
  return lo;
}
// the parent of supernode k: the owner of its struct's first position, -1 for a root
__device__ __forceinline__ int sel_parent(const JointSparseArgs& s, int k) {
  return s.sn[k].nt > 0 ? sel_owner(s, s.st[s.sn[k].st_off]) : -1;
}
__device__ __forceinline__ double* sel_z(const JointSelArgs& g, int k) {
  return g.Z + (g.s.panel[k] - 6ll * g.s.sn[k].first);
}

// struct(k) as runs of the ancestors t it falls in, ascending: run i holds the entries b0[i] ..
// b0[i + 1] - 1, and map[mo[i] + b - b0[i]] is entry b's panel cloud row in t (the row map of the
// update of t from k); z, rz: t's block of Z and its rows
struct SelRuns {
  double* z[SEL_MAX_PATH];
  int rz[SEL_MAX_PATH], b0[SEL_MAX_PATH + 1], mo[SEL_MAX_PATH];
  int n;
};
__device__ __forceinline__ int sel_run(const SelRuns& r, int b) {
  int lo = 0, hi = r.n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (r.b0[mid] <= b) lo = mid;
    else hi = mid;
  }
  return lo;
}

// Supernode k by the whole block, after every ancestor (Takahashi's recurrence; W = L_TJ L_JJ^-1):
//   X = Z_TT L_TJ, gathered from the ancestors' blocks through the update row maps;
//   Z_TJ = -X L_JJ^-1, row by row in place;
//   Z_JJ from Z_JJ L_JJ = L_JJ^-T - Z_TJ^T L_TJ, column by column from the last, the off-diagonal
//   entries of a column before its diagonal one, each mirrored above the diagonal.
// Every sum runs in a fixed order (ascending index; the diagonal entries by warp_sum), no atomics.
__device__ void sel_node(const JointSelArgs& g, int k, SelRuns& r) {
  const JointSparseArgs& s = g.s;
  const int tid = threadIdx.x, lane = tid & 31;
  const JointSuper& m = s.sn[k];
  const int nt = m.nt, C = 6 * m.ns, T = 6 * nt, Rl = C + T + 1, Rz = C + T;
  const double* L = s.L + s.panel[k];
  double* Z = sel_z(g, k);
  if (tid == 0) {
    int n = 0;
    for (int b = 0; b < nt; ++n) {
      const int t = sel_owner(s, s.st[m.st_off + b]);
      const JointSuper& tm = s.sn[t];
      int lo = tm.u0, hi = tm.u1 - 1;  // the update of t from k: t's updates by ascending descendant
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s.up[4 * mid] < k) lo = mid + 1;
        else hi = mid;
      }
      r.z[n] = sel_z(g, t);
      r.rz[n] = 6 * (tm.ns + tm.nt);
      r.b0[n] = b;
      r.mo[n] = s.up[4 * lo + 3];
      b += s.up[4 * lo + 2];
    }
    r.n = n;
    r.b0[n] = nt;
  }
  __syncthreads();
  // X = Z_TT L_TJ into the rows of Z_TJ: Z_TT's block (ca, cb) lies in the column of the earlier of
  // the two clouds, in the block of Z of its supernode, at the later one's row there
  for (int idx = tid; idx < T * C; idx += JS_THREADS) {
    const int row = idx % T, j = idx / T, ca = row / 6, qa = row % 6, ia = sel_run(r, ca);
    const double* Lc = L + (size_t)j * Rl + C;
    double v = 0.0;
    for (int i = 0; i < r.n; ++i)
      for (int cb = r.b0[i]; cb < r.b0[i + 1]; ++cb) {
        const double* zc;
        int rr;
        if (cb <= ca) {  // Z(ca, cb) in cb's ancestor: column cb, row ca
          zc = r.z[i] + (size_t)(6 * s.map[r.mo[i] + cb - r.b0[i]]) * r.rz[i];
          rr = 6 * s.map[r.mo[i] + ca - r.b0[i]] + qa;
          for (int qb = 0; qb < 6; ++qb) v = fma(zc[(size_t)qb * r.rz[i] + rr], Lc[6 * cb + qb], v);
        } else {  // Z(cb, ca)^T in ca's ancestor: column ca, row cb
          zc = r.z[ia] + (size_t)(6 * s.map[r.mo[ia] + ca - r.b0[ia]] + qa) * r.rz[ia];
          rr = 6 * s.map[r.mo[ia] + cb - r.b0[ia]];
          for (int qb = 0; qb < 6; ++qb) v = fma(zc[rr + qb], Lc[6 * cb + qb], v);
        }
      }
    Z[(size_t)j * Rz + C + row] = v;
  }
  __syncthreads();
  // Z_TJ L_JJ = -X: Z[t][j] = (-X[t][j] - sum_{c > j} Z[t][c] L[c][j]) / L[j][j]
  for (int row = tid; row < T; row += JS_THREADS)
    for (int j = C - 1; j >= 0; --j) {
      double v = -Z[(size_t)j * Rz + C + row];
      for (int c = j + 1; c < C; ++c) v = fma(-Z[(size_t)c * Rz + C + row], L[(size_t)j * Rl + c], v);
      Z[(size_t)j * Rz + C + row] = v / L[(size_t)j * Rl + j];
    }
  __syncthreads();
  // B = -Z_TJ^T L_TJ on and below the diagonal, into Z_JJ's slots
  for (int idx = tid; idx < C * C; idx += JS_THREADS) {
    const int i = idx % C, j = idx / C;
    if (i < j) continue;
    const double* zi = Z + (size_t)i * Rz + C;
    const double* lj = L + (size_t)j * Rl + C;
    double v = 0.0;
    for (int t = 0; t < T; ++t) v = fma(-zi[t], lj[t], v);
    Z[(size_t)j * Rz + i] = v;
  }
  __syncthreads();
  for (int j = C - 1; j >= 0; --j) {
    const double ljj = L[(size_t)j * Rl + j];
    for (int i = j + 1 + tid; i < C; i += JS_THREADS) {
      double v = Z[(size_t)j * Rz + i];
      for (int c = j + 1; c < C; ++c) v = fma(-Z[(size_t)c * Rz + i], L[(size_t)j * Rl + c], v);
      v /= ljj;
      Z[(size_t)j * Rz + i] = v;
      Z[(size_t)i * Rz + j] = v;
    }
    __syncthreads();
    if (tid < 32) {
      double v = 0.0;
      for (int c = j + 1 + lane; c < C; c += 32) v = fma(Z[(size_t)j * Rz + c], L[(size_t)j * Rl + c], v);
      v = warp_sum(v);
      if (lane == 0) Z[(size_t)j * Rz + j] = (1.0 / ljj + Z[(size_t)j * Rz + j] - v) / ljj;
    }
    __syncthreads();
  }
}

// k_joint_selinv, one cooperative launch: the final unknowns y' = (omega, u) about each start origin
// from xf (u = t' - dc x omega) into y and every read prior's y, for k_joint_sel_s0; then the
// supernodes by level from the roots down, one block per supernode, one grid barrier per level.
__global__ void __launch_bounds__(JS_THREADS) k_joint_selinv(const JointSelArgs g) {
  __shared__ SelRuns r;
  const JointSparseArgs& s = g.s;
  const JointArgs& a = s.j;
  const int tid = threadIdx.x, bid = blockIdx.x, G = gridDim.x;
  for (int f = bid * JS_THREADS + tid; f < a.F; f += G * JS_THREADS) {
    double y[6];
    for (int q = 0; q < 6; ++q) y[q] = s.xf[6 * f + q];
    const double* d = s.dc + 3 * f;
    y[3] -= d[1] * y[2] - d[2] * y[1];
    y[4] -= d[2] * y[0] - d[0] * y[2];
    y[5] -= d[0] * y[1] - d[1] * y[0];
    for (int q = 0; q < 6; ++q) g.y[6 * f + q] = y[q];
    if (a.prior_of && a.prior_of[f] >= 0)
      for (int q = 0; q < 6; ++q) a.prior[a.prior_of[f]].y[q] = y[q];
  }
  for (int l = s.depth - 1; l >= 0; --l) {
    for (int i = s.lv_off[l] + bid; i < s.lv_off[l + 1]; i += G) sel_node(g, s.lv[i], r);
    joint_grid_sync(a.bar);
  }
}

// k_joint_sel_parked, before k_joint_selinv (its scratch is Z's memory): for each parked edge, one
// block at a time, (N'^-1)_ab = w_a^T w_b, w_c = L^-1 E_c by forward substitution along the path from
// c's supernode to its root (the only supernodes where w_c is non-zero), into the edge's slot of
// cov_e (k_joint_sel_edge reads it there).  Clouds in different trees: no common supernode, 0.
__global__ void __launch_bounds__(JS_THREADS) k_joint_sel_parked(const JointSelArgs g) {
  __shared__ int path[2][SEL_MAX_PATH], np[2];
  __shared__ long long off[2][SEL_MAX_PATH + 1];
  const JointSparseArgs& s = g.s;
  const JointArgs& a = s.j;
  const int tid = threadIdx.x;
  double* W = g.Z + (size_t)blockIdx.x * g.scratch;
  for (int i = blockIdx.x; i < g.n_parked; i += gridDim.x) {
    const int e = g.parked[i];
    const int f[2] = {a.free_of[a.fix_id[e]], a.free_of[a.mov_id[e]]};
    if (tid < 2) {
      int n = 0;
      long long o = 0;
      for (int k = sel_owner(s, g.pos[f[tid]]); k >= 0; k = sel_parent(s, k), ++n) {
        path[tid][n] = k;
        off[tid][n] = o;
        o += 6 * s.sn[k].ns;
      }
      np[tid] = n;
      off[tid][n] = o;
    }
    __syncthreads();
    double* v[2] = {W, W + 6 * off[0][np[0]]};
    for (int side = 0; side < 2; ++side) {
      double* w = v[side];
      const long long La = off[side][np[side]];
      for (long long x = tid; x < 6 * La; x += JS_THREADS) w[x] = 0.0;
      __syncthreads();
      if (tid < 6) w[tid * La + 6 * (g.pos[f[side]] - s.sn[path[side][0]].first) + tid] = 1.0;
      __syncthreads();
      for (int h = 0; h < np[side]; ++h) {
        const JointSuper& m = s.sn[path[side][h]];
        const int C = 6 * m.ns, T = 6 * m.nt, Rl = C + T + 1;
        const double* L = s.L + s.panel[path[side][h]];
        const long long o = off[side][h];
        for (int j = 0; j < C; ++j) {
          const double ljj = L[(size_t)j * Rl + j];
          for (int x = tid; x < 6 * (C - j - 1); x += JS_THREADS) {
            const int q = x % 6, ii = j + 1 + x / 6;
            const double xj = w[q * La + o + j] / ljj;
            w[q * La + o + ii] = fma(-L[(size_t)j * Rl + ii], xj, w[q * La + o + ii]);
          }
          __syncthreads();
          if (tid < 6) w[tid * La + o + j] /= ljj;
          __syncthreads();
        }
        // the struct's rows: w_T -= L_TJ w_J, each on its ancestor's place in the path
        for (int x = tid; x < 6 * T; x += JS_THREADS) {
          const int q = x % 6, t = x / 6, p = s.st[m.st_off + t / 6];
          int h2 = h + 1;
          while (p >= s.sn[path[side][h2]].first + s.sn[path[side][h2]].ns) ++h2;
          const long long at = q * La + off[side][h2] + 6 * (p - s.sn[path[side][h2]].first) + t % 6;
          double acc = 0.0;
          for (int c = 0; c < C; ++c) acc = fma(L[(size_t)c * Rl + C + t], w[q * La + o + c], acc);
          w[at] -= acc;
        }
        __syncthreads();
      }
    }
    // the common supernodes: from the first of a's path that b's path holds on, both paths agree
    if (tid < 36) {
      const int qa = tid / 6, qb = tid % 6;
      const long long La = off[0][np[0]], Lb = off[1][np[1]];
      int h0 = 0, h1 = -1;
      for (; h0 < np[0]; ++h0) {
        for (int x = 0; x < np[1]; ++x)
          if (path[1][x] == path[0][h0]) h1 = x;
        if (h1 >= 0) break;
      }
      double acc = 0.0;
      if (h1 >= 0)
        for (int h = h0; h < np[0]; ++h, ++h1)
          for (long long x = 0; x < off[0][h + 1] - off[0][h]; ++x)
            acc = fma(v[0][qa * La + off[0][h] + x], v[1][qb * Lb + off[1][h1] + x], acc);
      g.c.cov_e[36 * (size_t)e + tid] = acc;
    }
    __syncthreads();
  }
}

// k_joint_sel_s0, one warp: s0^2 of the call into *s0sq by JOINT_S0_SUMS, the statement
// k_joint_cov_cloud uses, from the unknowns k_joint_selinv left in y and the priors' y
__global__ void __launch_bounds__(32) k_joint_sel_s0(const JointCovArgs a) {
  const int lane = threadIdx.x;
  JOINT_S0_SUMS(a, lane, ss, m)
  if (lane == 0) {
    const double dof = m - (double)(6 * a.F);
    *a.s0sq = dof > 0.0 ? ss / dof : nan("");
  }
}

// k_joint_sel_cloud, one thread per position p of free cloud f: C_c = s0^2 J'_c (N'^-1)_cc J'_c^T,
// with the lever o_c - o_c^0 of J'_c
__global__ void __launch_bounds__(128) k_joint_sel_cloud(const JointSelArgs g) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const JointSparseArgs& s = g.s;
  const JointCovArgs& a = g.c;
  if (p >= a.F) return;
  const int f = s.perm[p], k = sel_owner(s, p), cj = p - s.sn[k].first;
  const int Rz = 6 * (s.sn[k].ns + s.sn[k].nt);
  const double* Z = sel_z(g, k) + (size_t)(6 * cj) * Rz + 6 * cj;
  const double s0sq = *a.s0sq;
  const Rigid& T = a.pose[a.free_ids[f]];
  double d[3], Jc[36], C[36], M[36];
  for (int q = 0; q < 3; ++q) d[q] = (T.t[q] - a.cw[q]) - s.dc[3 * f + q];
  lever6(nullptr, d, Jc);
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) M[6 * r + c] = s0sq * Z[(size_t)c * Rz + r];
  abt6(Jc, M, Jc, C);
  store_sym6(C, s0sq, a.cov_f + 36 * (size_t)f);
}

// k_joint_sel_edge, one thread per edge e = (a, b): with both clouds free the cross block (N'^-1)_ab
// from the block of Z of the earlier position's supernode, at the later one's row there, or, for a
// pair outside the pattern, from k_joint_sel_parked's value in e's slot of cov_e; then C_e
// (JOINT_EDGE_COV in the sparse unknowns)
__global__ void __launch_bounds__(128) k_joint_sel_edge(const JointSelArgs g) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  const JointSparseArgs& s = g.s;
  const JointCovArgs& a = g.c;
  if (e >= a.n_edges) return;
  const int ca = a.fix_id[e], cb = a.mov_id[e], fa = a.free_of[ca], fb = a.free_of[cb];
  double gx[36];
  if (fa >= 0 && fb >= 0) {
    const int pa = g.pos[fa], pb = g.pos[fb], lo = min(pa, pb), hi = max(pa, pb);
    const int k = sel_owner(s, lo);
    const JointSuper& m = s.sn[k];
    int ri = -1;
    if (hi < m.first + m.ns) {
      ri = hi - m.first;
    } else {
      int l = 0, h = m.nt;  // struct(k) ascending
      while (l < h) {
        const int mid = (l + h) >> 1;
        if (s.st[m.st_off + mid] < hi) l = mid + 1;
        else h = mid;
      }
      if (l < m.nt && s.st[m.st_off + l] == hi) ri = m.ns + l;
    }
    if (ri >= 0) {
      const int Rz = 6 * (m.ns + m.nt);
      const double* Z = sel_z(g, k) + (size_t)(6 * (lo - m.first)) * Rz + 6 * ri;  // rows hi, columns lo
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) gx[6 * r + c] = (pa == hi) ? Z[(size_t)c * Rz + r] : Z[(size_t)r * Rz + c];
    } else {
      for (int j = 0; j < 36; ++j) gx[j] = a.cov_e[36 * (size_t)e + j];
    }
  }
  JOINT_EDGE_COV(a, e, ca, cb, fa, fb, gx, s.dc)
}

}  // namespace

void joint_reject_launch(Ctx& c, const JointArgs& a, int n_edges) {
  k_joint_reject<<<n_edges, JR_THREADS, 0, c.stream>>>(a);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void joint_prior_launch(Ctx& c, const JointArgs& a, const double* dc) {
  k_joint_prior<<<(a.n_prior + 127) / 128, 128, 0, c.stream>>>(a, dc);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void joint_relative_launch(Ctx& c, const JointArgs& a, const JointRelArgs& r, const double* dc) {
  k_joint_relative<<<(r.n + 127) / 128, 128, 0, c.stream>>>(a, r, dc);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void joint_solve_launch(Ctx& c, const JointArgs& a, const JointRelArgs& r) {
  JointArgs args = a;
  JointRelArgs rel = r;
  void* p[] = {&args, &rel};
  SICP_CUDA(cudaLaunchCooperativeKernel((void*)k_joint_solve, dim3(c.num_sms), dim3(JS_THREADS), p, 0, c.stream));
  c.tm.kernel_launches += 1;
}

void joint_sparse_solve_launch(Ctx& c, const JointSparseArgs& a) {
  JointSparseArgs args = a;
  void* p[] = {&args};
  SICP_CUDA(cudaLaunchCooperativeKernel((void*)k_joint_sparse_solve, dim3(c.num_sms), dim3(JS_THREADS), p, 0,
                                        c.stream));
  c.tm.kernel_launches += 1;
}

// sicp_timings describe the last registration call: these launches do not count in it
void joint_cov_launch(Ctx& c, const JointCovArgs& a) {
  k_joint_cov_ss<<<a.n_edges, JC_THREADS, 0, c.stream>>>(a);
  SICP_CUDA(cudaGetLastError());
  JointCovArgs args = a;
  void* p[] = {&args};
  SICP_CUDA(cudaLaunchCooperativeKernel((void*)k_joint_inv, dim3(c.num_sms), dim3(JS_THREADS), p, 0, c.stream));
  k_joint_cov_cloud<<<a.F, JC_THREADS, 0, c.stream>>>(a);
  SICP_CUDA(cudaGetLastError());
  k_joint_cov_edge<<<a.n_edges, JC_THREADS, 0, c.stream>>>(a);
  SICP_CUDA(cudaGetLastError());
}

void joint_sel_launch(Ctx& c, const JointSelArgs& a, int parked_blocks) {
  k_joint_cov_ss<<<a.c.n_edges, JC_THREADS, 0, c.stream>>>(a.c);
  SICP_CUDA(cudaGetLastError());
  if (parked_blocks > 0) {
    k_joint_sel_parked<<<parked_blocks, JS_THREADS, 0, c.stream>>>(a);
    SICP_CUDA(cudaGetLastError());
  }
  JointSelArgs args = a;
  void* p[] = {&args};
  SICP_CUDA(cudaLaunchCooperativeKernel((void*)k_joint_selinv, dim3(c.num_sms), dim3(JS_THREADS), p, 0, c.stream));
  k_joint_sel_s0<<<1, 32, 0, c.stream>>>(a.c);
  SICP_CUDA(cudaGetLastError());
  k_joint_sel_cloud<<<(a.c.F + 127) / 128, 128, 0, c.stream>>>(a);
  SICP_CUDA(cudaGetLastError());
  k_joint_sel_edge<<<(a.c.n_edges + 127) / 128, 128, 0, c.stream>>>(a);
  SICP_CUDA(cudaGetLastError());
}

}  // namespace sicp
