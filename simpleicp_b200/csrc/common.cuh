// common.cuh — shared device/host helpers for libsicp_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <limits>
#include <string>
#include <utility>
#include <vector>

#include "../../include/sicp_b200.h"

namespace sicp {

// ------------------------------------------------------------------------------------------
// Error handling: every CUDA call is checked; failures become SICP_ERR_CUDA with a message.
// ------------------------------------------------------------------------------------------
struct Error {
  int32_t code;
  std::string msg;
};
void set_thread_error(const std::string& m);

#define SICP_CUDA(call)                                                                     \
  do {                                                                                      \
    cudaError_t e__ = (call);                                                               \
    if (e__ != cudaSuccess)                                                                 \
      throw ::sicp::Error{SICP_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e__) + \
                                             " (" __FILE__ ":" + std::to_string(__LINE__) + ")"}; \
  } while (0)

#define SICP_REQUIRE(cond, code, message) \
  do {                                    \
    if (!(cond)) throw ::sicp::Error{(code), (message)}; \
  } while (0)

// ------------------------------------------------------------------------------------------
// Plain device buffer (cudaMalloc'd once, grown on demand).  Internal scratch only — caller
// arrays never pass through here.
// ------------------------------------------------------------------------------------------
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t cap = 0;
  ~DevBuf() { release(); }
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
  }
  void reserve(size_t n) {
    if (n <= cap) return;
    release();
    // a few elements of slack: 16-byte bulk copies / vector loads may read past an odd tail
    SICP_CUDA(cudaMalloc(&p, (n + 8) * sizeof(T)));
    cap = n;
  }
  void swap(DevBuf& o) {
    std::swap(p, o.p);
    std::swap(cap, o.cap);
  }
};

// pinned host buffer of at least n elements, grown on demand (contents not kept)
template <typename T>
void pinned_reserve(T*& p, size_t& cap, size_t n) {
  if (n <= cap) return;
  if (p) cudaFreeHost(p);
  p = nullptr;
  SICP_CUDA(cudaMallocHost(&p, n * sizeof(T)));
  cap = n;
}

// ------------------------------------------------------------------------------------------
// Geometry types
// ------------------------------------------------------------------------------------------
// One point of a cell-sorted cloud: 32 bytes = one L2 sector.
struct __align__(32) Rec {
  double x, y, z;
  long long idx;  // index in the caller's (unsorted) cloud
};

// Uniform grid over one cloud (cells cubic, x fastest).  cell_start has n_cells + 1 entries.
struct GridView {
  const Rec* recs;
  const uint32_t* cell_start;
  double ox, oy, oz;  // origin (bbox min)
  double h, inv_h;
  int nx, ny, nz;
  long long n_points;
};

// p' = R p + t, row-major R.
struct Rigid {
  double r[9];
  double t[3];
};

__host__ __device__ inline void rigid_apply(const Rigid& T, double x, double y, double z,
                                            double& ox, double& oy, double& oz) {
  ox = fma(T.r[2], z, fma(T.r[1], y, T.r[0] * x)) + T.t[0];
  oy = fma(T.r[5], z, fma(T.r[4], y, T.r[3] * x)) + T.t[1];
  oz = fma(T.r[8], z, fma(T.r[7], y, T.r[6] * x)) + T.t[2];
}

// inverse of a rigid transform: p = R^T (p' - t)
__host__ __device__ inline Rigid rigid_inverse(const Rigid& T) {
  Rigid I;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) I.r[i * 3 + j] = T.r[j * 3 + i];
  for (int i = 0; i < 3; ++i)
    I.t[i] = -(I.r[i * 3 + 0] * T.t[0] + I.r[i * 3 + 1] * T.t[1] + I.r[i * 3 + 2] * T.t[2]);
  return I;
}

inline Rigid rigid_from_H(const double H[16]) {
  Rigid T;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) T.r[i * 3 + j] = H[i * 4 + j];
    T.t[i] = H[i * 4 + 3];
  }
  return T;
}

// Euler angles -> R = Rx(a1) Ry(a2) Rz(a3), element layout of the reference
// (python/simpleicp/mathutils.py:39-68).
__host__ __device__ inline void euler_to_R(double a1, double a2, double a3, double* R) {
  double s1, c1, s2, c2, s3, c3;
  sincos(a1, &s1, &c1);
  sincos(a2, &s2, &c2);
  sincos(a3, &s3, &c3);
  R[0] = c2 * c3;
  R[1] = -c2 * s3;
  R[2] = s2;
  R[3] = c1 * s3 + s1 * s2 * c3;
  R[4] = c1 * c3 - s1 * s2 * s3;
  R[5] = -s1 * c2;
  R[6] = s1 * s3 - c1 * s2 * c3;
  R[7] = s1 * c3 + c1 * s2 * s3;
  R[8] = c1 * c2;
}

__host__ __device__ inline Rigid rigid_from_x(const double* x) {
  Rigid T;
  euler_to_R(x[0], x[1], x[2], T.r);
  T.t[0] = x[3];
  T.t[1] = x[4];
  T.t[2] = x[5];
  return T;
}

// A after B: p -> A(B(p))
__host__ __device__ inline Rigid rigid_compose(const Rigid& A, const Rigid& B) {
  Rigid C;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j)
      C.r[i * 3 + j] = A.r[i * 3 + 0] * B.r[0 * 3 + j] + A.r[i * 3 + 1] * B.r[1 * 3 + j] + A.r[i * 3 + 2] * B.r[2 * 3 + j];
    C.t[i] = A.r[i * 3 + 0] * B.t[0] + A.r[i * 3 + 1] * B.t[1] + A.r[i * 3 + 2] * B.t[2] + A.t[i];
  }
  return C;
}

inline void H_from_rigid(const Rigid& T, double H[16]) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) H[i * 4 + j] = T.r[i * 3 + j];
    H[i * 4 + 3] = T.t[i];
  }
  H[12] = H[13] = H[14] = 0.0;
  H[15] = 1.0;
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------
// Order-preserving map double <-> uint64 (for atomicMin/Max and radix work)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned long long f64_to_key(double v) {
  unsigned long long b = (unsigned long long)__double_as_longlong(v);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ double key_to_f64(unsigned long long k) {
  unsigned long long b = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  return __longlong_as_double((long long)b);
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- mbarrier + 1-D TMA bulk copies (cp.async.bulk; SASS: SYNCS.*, UBLKCP) -------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "LAB_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
      "@P1 bra DONE;\n"
      "bra LAB_WAIT;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// Programmatic dependent launch (sm_90+).  A kernel launched with the programmatic-stream-
// serialization attribute may start while its predecessor in the stream is still running — once
// every block of the predecessor has executed launch_dependents (or exited); it must not touch
// anything the predecessor writes before pdl_wait(), which returns when the predecessor has
// completed and its writes are visible.  Both are no-ops in a plain launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ int cell_coord(double v, double o, double inv_h, int n) {
  int c = __double2int_rd((v - o) * inv_h);  // saturating
  return min(max(c, 0), n - 1);
}
#endif  // __CUDACC__

constexpr int kBfTile = 2048;  // float4 points per TMA stage of the brute-force engine
constexpr double kInf = std::numeric_limits<double>::infinity();

}  // namespace sicp
