// transform.cu — PointCloud.transform_by_H (python/simpleicp/pointcloud.py:205-217) for the one
// place the product still needs it: the final X_mov_transformed = H * X_mov
// (python/simpleicp/simpleicp.py:316).  Pure HBM streaming: 24 B read + 24 B written per point.
// The homogeneous divide of mathutils.py:19-26 is the identity (w = 0*x + 0*y + 0*z + 1*1 = 1).
#include <algorithm>

#include "ctx.cuh"

namespace sicp {

namespace {

// Two points (48 B = 3 x 16 B) per thread so that every access is a 128-bit vector.
__global__ void __launch_bounds__(256)
    k_transform(Rigid T, const double2* __restrict__ in, double2* __restrict__ out, long long n_pairs,
                const double* __restrict__ in_tail, double* __restrict__ out_tail, int has_tail) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n_pairs) {
    const double2 a = __ldg(in + 3 * i + 0), b = __ldg(in + 3 * i + 1), c = __ldg(in + 3 * i + 2);
    double x0, y0, z0, x1, y1, z1;
    rigid_apply(T, a.x, a.y, b.x, x0, y0, z0);
    rigid_apply(T, b.y, c.x, c.y, x1, y1, z1);
    out[3 * i + 0] = make_double2(x0, y0);
    out[3 * i + 1] = make_double2(z0, x1);
    out[3 * i + 2] = make_double2(y1, z1);
  }
  if (has_tail && i == 0) {
    double x, y, z;
    rigid_apply(T, in_tail[0], in_tail[1], in_tail[2], x, y, z);
    out_tail[0] = x;
    out_tail[1] = y;
    out_tail[2] = z;
  }
}

// sicp_get_batch_outputs: the movable cloud of pair ids[blockIdx.y] (read at its offset mov_off)
// moved by its applied transform DevState::T, into out from point off[blockIdx.y] on.  Pairs that
// share a movable cloud read the same points and write their own slices.  A slice starts at an
// arbitrary point offset (16-byte aligned only when it is even), so every access is a scalar double.
__global__ void __launch_bounds__(256)
    k_transform_pairs(const PairDev* __restrict__ pairs, const DevState* __restrict__ state,
                      const int* __restrict__ ids, const long long* __restrict__ off, const double* __restrict__ in,
                      double* __restrict__ out) {
  const int pair = ids[blockIdx.y];
  const long long n = pairs[pair].n_mov, i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long p = 3 * (pairs[pair].mov_off + i), o = 3 * (off[blockIdx.y] + i);
  double x, y, z;
  rigid_apply(state[pair].T, __ldg(in + p + 0), __ldg(in + p + 1), __ldg(in + p + 2), x, y, z);
  out[o + 0] = x;
  out[o + 1] = y;
  out[o + 2] = z;
}

}  // namespace

void batch_transform_launch(Ctx& c, Batch& b, const int* ids, int n_ids, const long long* off, long long max_n_mov,
                            double* out) {
  const long long blocks = std::max<long long>((max_n_mov + 255) / 256, 1);
  k_transform_pairs<<<dim3((unsigned)blocks, (unsigned)n_ids), 256, 0, c.stream>>>(b.pairs.p, b.state.p, ids, off,
                                                                                 b.xyz.p, out);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void transform_launch(Ctx& c, const Rigid& T, const double* in, double* out, long long n) {
  if (n <= 0) return;
  const long long n_pairs = n / 2;
  const int has_tail = (int)(n & 1);
  const long long blocks = std::max<long long>((n_pairs + 255) / 256, 1);
  k_transform<<<(unsigned)blocks, 256, 0, c.stream>>>(
      T, reinterpret_cast<const double2*>(in), reinterpret_cast<double2*>(out), n_pairs,
      in + 3 * (n - 1), out + 3 * (n - 1), has_tail);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

}  // namespace sicp
