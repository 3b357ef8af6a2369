// reject_solve.cuh — device-resident loop state and kernel argument blocks shared by the
// match and reject/solve kernels.
#pragma once
#include "common.cuh"

namespace sicp {

// Lives in device memory for the whole run: the iteration loop never needs the host to carry
// a value from one kernel to the next, so iterations can be queued back to back (or replayed
// from a CUDA graph) and the host only reads the small per-iteration record.
struct DevState {
  Rigid T;      // current cumulative transform H(x)
  Rigid Tinv;
  double x[6];
  double x_new[6];
  Rigid T_new;
  double An[36];   // unweighted J^T M J at the last solution (for the sigmas)
  double sigma[6];
  double w;        // distance weight in use (frozen after iteration 0, simpleicp.py:229-234)
  double prev_mean, prev_std;
  long long n_kept;
  int skip;        // fewer than 6 correspondences or solve not requested
  int stop;        // stop rule met: every later queued kernel returns immediately
  int converged;
  int iterations_done;
  int lm_ok;
  int pad;
  // Predictor for the next iteration's order statistics: the match kernel bins every
  // point-to-plane distance of a planarity survivor into a linear histogram centred on the
  // previous median, +-4 previous MADs wide (see lh_bin below).
  double pred_med, pred_mad, pred_minpl;
  int pred_valid;   // pred_* describe a finished reject phase of this run
  // Linearised variant (SICP_VARIANT_LINEARIZED*): T_res is the affine map (I + [alpha]x) T + t
  // whose point-to-plane residuals are the reference's "A x - l" (c++/src/corrpts.cpp:155);
  // H_rep is the matrix the reference driver reports (dH * H, or H * dH for the C++ driver).
  // In the default variant T_res == T_new and H_rep == T.
  Rigid T_res;
  Rigid H_rep;
};

// Linear histogram shared by the match kernels (producers) and k_reject_solve (consumer).
// LH_BINS regular bins over [med - 4 mad, med + 4 mad), then one underflow and one overflow
// counter.  The bin function is monotone non-decreasing in d, which is all the exactness of the
// selection needs; both sides evaluate this very expression.
constexpr int LH_BINS = 4096;
__host__ __device__ inline int lh_bin(double d, double med, double mad) {
  const double lo = med - 4.0 * mad;
  const double inv_w = (double)LH_BINS / (8.0 * mad);
  const double t = (d - lo) * inv_w;
  if (!(t >= 0.0)) return LH_BINS;  // underflow (and NaN)
  if (t >= (double)LH_BINS) return LH_BINS + 1;
  return (int)t;
}

// Diagnostics written by block 0, thread 0 of the reject/solve kernels (sicp_get_phase_times).
// Slot 29: which selection produced the record's median and MAD.
enum SelectPath : int {
  SEL_PATH_RADIX = 0,    // radix_median: iteration 0, the stage API, every fallback
  SEL_PATH_BINSTORE = 2, // fused_select: per-bin key store of k_rs_fused / k_rs_batch
};
// Slot 30 (last k_rs_fused / k_rs_batch launch): outcome of the attempt to select from the
// predictor histogram.  0 = used, else the first check that failed.  _capi.py mirrors these values.
enum SelectOutcome : int {
  SEL_OK = 0,
  SEL_NO_PREDICTION = 1,      // no histogram, no valid predictor, or one for another planarity bound
  SEL_MEDIAN_OUTSIDE = 3,     // a middle rank lies in the under- or overflow counter
  SEL_MEDIAN_GAP = 5,         // the bins of the two middle ranks are more than 4 bins apart
  SEL_MEDIAN_CANDIDATES = 6,  // the median bins hold more than RS_CAP - 2 members
  SEL_MAD_BRACKET = 7,        // the regular bins hold fewer than k2 + 1 members: no MAD bracket
  SEL_MAD_WINDOW = 8,         // the MAD candidate window runs past the regular bins
  SEL_MAD_CANDIDATES = 9,     // the MAD window holds more than RS_CAP - 2 members
  SEL_BIN_CAP = 10,           // fused_select: a candidate bin has more members than the key store holds
};

struct RSArgs {
  long long K;
  const double* dist;
  const float4* q_nrm;
  const double* q_xyz;
  const double* m_xyz;  // matched movable point (caller coordinates), K x 3
  uint8_t* keep;
  double* resid;
  unsigned int* unresolved;  // [K] = queries the grid left to the brute-force pass; reset by the kernel after reading
  DevState* state;
  sicp_iter_record* rec;
  double min_planarity;  // compared against the float32 planarity promoted to float64
  double min_change;
  double w_param;
  double obs[6];
  double wobs[6];
  double cm[3];
  int it;
  int do_solve;
  int arm_stop;
  int hist_expected;  // the preceding match launch fed lin_hist (if the predictor was valid; fused kernel)
  int variant;        // sicp_variant
  double stat_minpl;  // planarity bound of the set the median/MAD are taken over (-inf: everybody)
  // fused kernel only (k_rs_fused): what the match kernels left per correspondence
  const unsigned long long* binstore;  // LH_BINS x bin_cap: f64_to_key(distance) of the members of each predictor-histogram bin
  int bin_cap;
  int want_sigma;              // evaluate the parameter sigmas even if the stop rule does not fire
  // q_nrm is the match kernel's per-iteration copy whose .w is the signed effective planarity
  // (nn.cu: effective_planarity): |w| enters both planarity tests, a set sign bit = rejected by
  // the angle between the normals after the distance rejection
  int pl_signed;
};
__device__ __forceinline__ double pl_stat(float w, int pl_signed) { return (double)(pl_signed ? fabsf(w) : w); }
__device__ __forceinline__ bool pl_keep(float w, double min_planarity, int pl_signed) {
  if (pl_signed) return (double)fabsf(w) >= min_planarity && !signbit(w);
  return (double)w >= min_planarity;
}

// Outcome of the select every block of k_rs_fused (split form) computes; block 0 hands it to k_rs_solve.
struct RsSelect {
  double median, mad;
  unsigned int n1;  // planarity survivors
  int ok;           // 0: the prediction did not bracket the order statistics
};

// Where the rehearsal of k_rs_solve sends every store of the serial tail.
struct RsScratch {
  DevState st;
  sicp_iter_record rec;
  unsigned long long phase_t[32];
  unsigned int lin_hist[LH_BINS + 2];
  unsigned int unresolved;
};

struct RSWork {
  unsigned int* hist;
  unsigned int* hist_other;
  unsigned long long* cand;
  unsigned int* counters;
  unsigned int* counters_other;
  unsigned long long* minkey;
  unsigned long long* minkey_other;
  double* partials;
  unsigned long long* phase_t;  // 32 x %globaltimer stamps of block 0 (diagnostics)
  unsigned int* barrier;        // {arrival count, generation} of the grid barrier
  unsigned int* lin_hist;       // LH_BINS + 2 counters filled by the match kernels
  // fused kernel, split form: the other half of the double-buffered partials (the previous
  // iteration's), the select outcome and the rehearsal's store target
  const double* partials_prev;
  RsSelect* sel;
  RsScratch* scratch;
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Residual of query i at the final transform Tn, in the reference's operation order
// (optimization.py:117-124): the matched movable point moved by Tn, minus the fixed point, dotted
// with the fixed normal.  The only definition: k_finish_batch takes its statistics from it,
// k_final_residuals and k_batch_residuals return it, k_joint_cov_ss sums its squares.
__device__ __forceinline__ double final_residual(const Rigid& Tn, const double* m_xyz, const double* q_xyz,
                                                 const float4* q_nrm, long long i) {
  double tx, ty, tz;
  rigid_apply(Tn, m_xyz[3 * i + 0], m_xyz[3 * i + 1], m_xyz[3 * i + 2], tx, ty, tz);
  const float4 nr = q_nrm[i];
  const double dx = tx - q_xyz[3 * i + 0], dy = ty - q_xyz[3 * i + 1], dz = tz - q_xyz[3 * i + 2];
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, (double)nr.x), __dmul_rn(dy, (double)nr.y)), __dmul_rn(dz, (double)nr.z));
}
#endif

}  // namespace sicp
