// grid.cu — build the static uniform grid over a cloud (done ONCE per cloud; the reference
// rebuilds a kd-tree over the transformed movable cloud every iteration,
// python/simpleicp/corrpts.py:131 — here the cloud never moves, the queries do).
//
// One builder, grid_build, grids one cloud or many in one segmented counting sort:
//   * all clouds share one record array (cloud i owns [rec_base, rec_base + n)) and one cell table
//     (cloud i owns [cell_base, cell_base + n_cells]); cell-table entries are GLOBAL record
//     positions, so one exclusive scan over the concatenated counters serves every cloud and the
//     end sentinel of a cloud is the first entry of the next;
//   * blockIdx.y selects the cloud in every per-point kernel;
//   * the cell sizes follow grid_plan.h; the host sees the bounding boxes and the occupancies of
//     all clouds at once (one read-back each per attempt, not per cloud).
// Rec::idx is the index inside its own cloud.
//
// Pipeline (all HBM-streaming, one pass each over n points or n_cells cells):
//   k_bbox        : min/max of x,y,z                (reads 24 n B)
//   k_cell_count  : cell id per point + histogram   (reads 24 n B, n atomics into L2), per attempt
//   scan          : exclusive prefix over cells     (reads/writes 4 n_cells B, 4 kernels)
//   k_scatter     : cell-sorted 32-byte records     (reads 28 n B, writes 32 n B)
#include <algorithm>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "ctx.cuh"

namespace sicp {

namespace {

constexpr int kScanItems = 4096;  // cells per scan block (256 threads x 16)

// The grid kernels take the cloud of their block from the plan table, plans[blockIdx.y]; a build
// of one cloud passes plans == nullptr and its plan by value in `one` (no plan table to upload).
__global__ void k_bbox_init(unsigned long long* keys, int n_clouds) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 6 * n_clouds) keys[i] = ((i % 6) < 3) ? ~0ull : 0ull;
}

__global__ void __launch_bounds__(256) k_bbox(const CloudPlan* __restrict__ plans, CloudPlan one,
                                              unsigned long long* __restrict__ keys) {
  const CloudPlan pl = plans ? plans[blockIdx.y] : one;
  const double* __restrict__ xyz = pl.xyz;
  double mn[3] = {kInf, kInf, kInf}, mx[3] = {-kInf, -kInf, -kInf};
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < pl.n;
       i += (long long)gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double v = xyz[3 * i + a];
      mn[a] = fmin(mn[a], v);
      mx[a] = fmax(mx[a], v != v ? kInf : v);  // fmax drops NaN: count it as +inf, which the host refuses
    }
  }
  __shared__ double smn[8][3], smx[8][3];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    mn[a] = warp_min(mn[a]);
    mx[a] = warp_max(mx[a]);
    if (lane == 0) {
      smn[w][a] = mn[a];
      smx[w][a] = mx[a];
    }
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    const int a = threadIdx.x;
    double lo = smn[0][a], hi = smx[0][a];
    for (int i = 1; i < 8; ++i) {
      lo = fmin(lo, smn[i][a]);
      hi = fmax(hi, smx[i][a]);
    }
    atomicMin(&keys[6 * blockIdx.y + a], f64_to_key(lo));
    atomicMax(&keys[6 * blockIdx.y + 3 + a], f64_to_key(hi));
  }
}

__global__ void __launch_bounds__(256) k_cell_count(const CloudPlan* __restrict__ plans, CloudPlan one,
                                                    uint32_t* __restrict__ cid, uint32_t* __restrict__ count,
                                                    unsigned int* __restrict__ occ) {
  const CloudPlan pl = plans ? plans[blockIdx.y] : one;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  int first = 0;
  if (i < pl.n) {
    const int cx = cell_coord(pl.xyz[3 * i + 0], pl.ox, pl.inv_h, pl.nx);
    const int cy = cell_coord(pl.xyz[3 * i + 1], pl.oy, pl.inv_h, pl.ny);
    const int cz = cell_coord(pl.xyz[3 * i + 2], pl.oz, pl.inv_h, pl.nz);
    const uint32_t cell = (uint32_t)(((long long)cz * pl.ny + cy) * pl.nx + cx);
    cid[pl.rec_base + i] = cell;
    first = (atomicAdd(&count[pl.cell_base + cell], 1u) == 0u) ? 1 : 0;
  }
  // occupied cells of this cloud: ONE atomic per block (one per first touch serialised 30 000
  // same-address atomics per cloud: 113 us for 1.6 M points, ncu r2)
  const int n_first = __syncthreads_count(first);
  if (threadIdx.x == 0 && n_first) atomicAdd(&occ[blockIdx.y], (unsigned int)n_first);
}

// ---- 3-kernel exclusive scan of uint32 or uint8 values ----------------------------------------
// Any n below 2^32 whose total is below 2^32 (the outputs are uint32): k_scan_blocksums walks the
// ceil(n / 4096) block sums 1024 at a time with a carry.  tests/test_gpu_scale.py runs it at
// 2^27 + 4097 elements (a map crop) and at totals of about 3.9e9 (the map filter's survivors).
template <typename T>
__global__ void __launch_bounds__(256) k_scan_reduce(const T* __restrict__ in, long long n,
                                                     uint32_t* __restrict__ block_sums) {
  long long base = (long long)blockIdx.x * kScanItems;
  uint32_t s = 0;
  for (int j = threadIdx.x; j < kScanItems; j += 256) {
    long long i = base + j;
    if (i < n) s += in[i];
  }
  __shared__ uint32_t sh[8];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int i = 0; i < 8; ++i) t += sh[i];
    block_sums[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(1024) k_scan_blocksums(uint32_t* __restrict__ block_sums, int nb) {
  // single block, sequential chunks of 1024 with a running carry
  __shared__ uint32_t sh[1024];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < nb; base += 1024) {
    int i = base + threadIdx.x;
    uint32_t v = (i < nb) ? block_sums[i] : 0;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      uint32_t t = (threadIdx.x >= o) ? sh[threadIdx.x - o] : 0;
      __syncthreads();
      sh[threadIdx.x] += t;
      __syncthreads();
    }
    uint32_t incl = sh[threadIdx.x];
    uint32_t c = carry;
    if (i < nb) block_sums[i] = c + incl - v;  // exclusive
    __syncthreads();
    if (threadIdx.x == 1023) carry = c + incl;
    __syncthreads();
  }
}

// Exclusive scan of one 4096-item block, fully coalesced: thread t moves uint4 number j*256 + t
// (j = 0..3), i.e. 16-byte accesses with unit stride across the warp in both directions; the
// four 256-wide slabs are scanned one after the other with a running carry.  uint8 inputs are
// read one value at a time.
template <typename T>
__global__ void __launch_bounds__(256) k_scan_down(const T* __restrict__ in, long long n,
                                                   const uint32_t* __restrict__ block_offsets,
                                                   uint32_t* __restrict__ out) {
  constexpr bool kVec = std::is_same<T, uint32_t>::value;
  const long long base = (long long)blockIdx.x * kScanItems;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __shared__ uint32_t wsum[8];
  __shared__ uint32_t carry_s;
  uint32_t carry = block_offsets[blockIdx.x];
  const bool vec_ok = kVec && (base + kScanItems <= n) && ((reinterpret_cast<uintptr_t>(in + base) & 15) == 0) &&
                      ((reinterpret_cast<uintptr_t>(out + base) & 15) == 0);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const long long i0 = base + 4ll * (j * 256 + threadIdx.x);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (vec_ok) {
      if constexpr (kVec) v = *reinterpret_cast<const uint4*>(in + i0);
    } else {
      if (i0 + 0 < n) v.x = in[i0 + 0];
      if (i0 + 1 < n) v.y = in[i0 + 1];
      if (i0 + 2 < n) v.z = in[i0 + 2];
      if (i0 + 3 < n) v.w = in[i0 + 3];
    }
    const uint32_t s = v.x + v.y + v.z + v.w;
    uint32_t incl = s;
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    __syncthreads();  // wsum / carry_s of the previous slab have been consumed
    if (lane == 31) wsum[w] = incl;
    __syncthreads();
    uint32_t woff = 0, tot = 0;
    for (int i = 0; i < 8; ++i) {
      if (i < w) woff += wsum[i];
      tot += wsum[i];
    }
    uint32_t run = carry + woff + incl - s;
    uint4 o4;
    o4.x = run;
    o4.y = run + v.x;
    o4.z = o4.y + v.y;
    o4.w = o4.z + v.z;
    if (vec_ok) {
      *reinterpret_cast<uint4*>(out + i0) = o4;
    } else {
      if (i0 + 0 < n) out[i0 + 0] = o4.x;
      if (i0 + 1 < n) out[i0 + 1] = o4.y;
      if (i0 + 2 < n) out[i0 + 2] = o4.z;
      if (i0 + 3 < n) out[i0 + 3] = o4.w;
    }
    carry += tot;
  }
  (void)carry_s;
}

template <typename T>
__global__ void k_scan_total(const T* __restrict__ in, long long n, uint32_t* __restrict__ out) {
  // out[n] = out[n-1] + in[n-1]
  if (threadIdx.x == 0 && blockIdx.x == 0) out[n] = (n > 0) ? out[n - 1] + in[n - 1] : 0;
}

// ---- ordered compaction (compact_bounds, compact_scatter) ---------------------------------------
// b[i] = scan[b[i]]: the host uploads the offsets into b and reads the boundaries back from it
__global__ void k_compact_bounds(const uint32_t* __restrict__ scan, int m, uint32_t* __restrict__ b) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) b[i] = scan[b[i]];
}

// Every j < n with flag[j] != 0 goes to o = scan[j]: pos[o] = j, and the W doubles of row from[j]
// (row j without from) of src to row o of rows.  A null pos or rows is not written.
template <typename F, typename I, int W>
__global__ void __launch_bounds__(256)
    k_compact(const F* __restrict__ flag, long long n, const uint32_t* __restrict__ scan, I* __restrict__ pos,
              const double* __restrict__ src, const long long* __restrict__ from, double* __restrict__ rows) {
  const long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (j >= n || !flag[j]) return;
  const long long o = scan[j];
  if (pos) pos[o] = (I)j;
  if (rows) {
    const long long r = from ? from[j] : j;
#pragma unroll
    for (int a = 0; a < W; ++a) rows[W * o + a] = src[W * r + a];
  }
}

__global__ void __launch_bounds__(256) k_scatter(const CloudPlan* __restrict__ plans, CloudPlan one,
                                                 const uint32_t* __restrict__ cid,
                                                 const uint32_t* __restrict__ cell_start,
                                                 uint32_t* __restrict__ fill, Rec* __restrict__ recs) {
  const CloudPlan pl = plans ? plans[blockIdx.y] : one;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= pl.n) return;
  const uint32_t cell = cid[pl.rec_base + i];
  const uint32_t pos = cell_start[pl.cell_base + cell] + atomicAdd(&fill[pl.cell_base + cell], 1u);
  Rec r;
  r.x = pl.xyz[3 * i + 0];
  r.y = pl.xyz[3 * i + 1];
  r.z = pl.xyz[3 * i + 2];
  r.idx = i;
  recs[pos] = r;
}

// Cells hold their points in arrival order of the atomics; sort each cell by original index so
// the layout (and therefore every memory trace) is reproducible run to run.  Cells are tiny
// (target occupancy ~3), insertion sort by one thread per cell.
__global__ void __launch_bounds__(256) k_sort_cells(const uint32_t* __restrict__ cell_start,
                                                    long long n_cells, Rec* __restrict__ recs) {
  long long c = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (c >= n_cells) return;
  uint32_t s = cell_start[c], e = cell_start[c + 1];
  for (uint32_t i = s + 1; i < e; ++i) {
    Rec r = recs[i];
    uint32_t j = i;
    while (j > s && recs[j - 1].idx > r.idx) {
      recs[j] = recs[j - 1];
      --j;
    }
    recs[j] = r;
  }
}

__global__ void __launch_bounds__(256) k_float4_copy(const double* __restrict__ xyz, long long n,
                                                     long long n_pad, double cx, double cy,
                                                     double cz, float4* __restrict__ out) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n_pad) return;
  float4 v;
  if (i < n) {
    v.x = (float)(xyz[3 * i + 0] - cx);
    v.y = (float)(xyz[3 * i + 1] - cy);
    v.z = (float)(xyz[3 * i + 2] - cz);
    v.w = 0.f;
  } else {
    v.x = v.y = v.z = 3.0e18f;  // padding: never the nearest neighbour
    v.w = 0.f;
  }
  out[i] = v;
}

// key_to_f64 on the host
inline double host_key_to_f64(unsigned long long k) {
  const unsigned long long b = (k & 0x8000000000000000ull) ? (k & 0x7fffffffffffffffull) : ~k;
  double v;
  std::memcpy(&v, &b, sizeof(v));
  return v;
}

}  // namespace

template <typename T>
static void scan_launch(Ctx& c, const T* in, long long n, uint32_t* out, DevBuf<uint32_t>& block_sums) {
  cudaStream_t st = c.stream;
  const long long nsb = (n + kScanItems - 1) / kScanItems;
  block_sums.reserve(nsb + 1);
  k_scan_reduce<<<(unsigned)nsb, 256, 0, st>>>(in, n, block_sums.p);
  k_scan_blocksums<<<1, 1024, 0, st>>>(block_sums.p, (int)nsb);
  k_scan_down<<<(unsigned)nsb, 256, 0, st>>>(in, n, block_sums.p, out);
  k_scan_total<<<1, 32, 0, st>>>(in, n, out);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 4;
}

void scan_u32(Ctx& c, const uint32_t* in, long long n, uint32_t* out, DevBuf<uint32_t>& block_sums) {
  scan_launch(c, in, n, out, block_sums);
}

void scan_u32(Ctx& c, const uint8_t* in, long long n, uint32_t* out, DevBuf<uint32_t>& block_sums) {
  scan_launch(c, in, n, out, block_sums);
}

const uint32_t* compact_bounds(Ctx& c, const uint32_t* scan, const std::vector<long long>& off) {
  CompactScratch& s = c.compact;
  const int m = (int)off.size();
  pinned_reserve(s.host, s.host_cap, (size_t)m);
  s.bounds.reserve((size_t)m);
  for (int i = 0; i < m; ++i) s.host[i] = (uint32_t)off[(size_t)i];
  cudaStream_t st = c.stream;
  SICP_CUDA(cudaMemcpyAsync(s.bounds.p, s.host, sizeof(uint32_t) * (size_t)m, cudaMemcpyHostToDevice, st));
  k_compact_bounds<<<(m + 255) / 256, 256, 0, st>>>(scan, m, s.bounds.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
  SICP_CUDA(cudaMemcpyAsync(s.host, s.bounds.p, sizeof(uint32_t) * (size_t)m, cudaMemcpyDeviceToHost, st));
  SICP_CUDA(cudaStreamSynchronize(st));
  return s.host;
}

void compact_scatter(Ctx& c, const uint32_t* flag, long long n, const uint32_t* scan, uint32_t* pos,
                     const double* xyz, const long long* from, double* xyz_out) {
  k_compact<uint32_t, uint32_t, 3><<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(flag, n, scan, pos, xyz, from,
                                                                                     xyz_out);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void compact_scatter(Ctx& c, const uint8_t* flag, long long n, const uint32_t* scan, long long* pos,
                     const double* src, double* out) {
  k_compact<uint8_t, long long, 1><<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(flag, n, scan, pos, src,
                                                                                      nullptr, out);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

void grid_build(Ctx& c, GridBufs& g, const std::vector<HostCloud>& clouds, const CellPolicy& policy,
                std::vector<GridView>& views, std::vector<double>& centres) {
  cudaStream_t st = c.stream;
  static const bool trace = std::getenv("SICP_TRACE_RUN") != nullptr;
  const auto tr0 = std::chrono::steady_clock::now();
  auto tr = [&](const char* what) {
    if (trace)
      fprintf(stderr, "[grid_build] %-12s t=%.1f us\n", what,
              std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - tr0).count());
  };
  const int nc = (int)clouds.size();
  long long total_pts = 0, max_n = 0;
  for (const auto& cl : clouds) {
    total_pts = std::max(total_pts, cl.point_off + cl.n);
    max_n = std::max(max_n, cl.n);
  }
  SICP_REQUIRE(total_pts < (1ll << 32), SICP_ERR_BAD_ARG, "a batch is limited to 2^32 - 1 points in total");
  pinned_reserve(c.grid_host, c.grid_host_cap, (size_t)nc * 6);
  c.bbox_keys.reserve((size_t)nc * 6);
  c.grid_occ.reserve(nc);
  g.cid.reserve(total_pts);
  g.recs.reserve(total_pts);
  std::vector<CloudPlan> plans((size_t)nc);
  for (int i = 0; i < nc; ++i) {
    plans[(size_t)i] = CloudPlan{};
    plans[(size_t)i].xyz = clouds[(size_t)i].xyz_dev;
    plans[(size_t)i].n = clouds[(size_t)i].n;
    plans[(size_t)i].rec_base = clouds[(size_t)i].point_off;
  }
  // several clouds read their plans from a table on the device, one cloud gets it by value
  const CloudPlan* table = nullptr;
  auto upload_plans = [&]() {
    if (nc == 1) return;
    c.grid_plans.reserve(nc);
    // pageable source: the runtime stages it before returning, `plans` may change afterwards
    SICP_CUDA(cudaMemcpyAsync(c.grid_plans.p, plans.data(), sizeof(CloudPlan) * (size_t)nc, cudaMemcpyHostToDevice, st));
    table = c.grid_plans.p;
  };

  // ---- bounding boxes: one read-back for all clouds
  upload_plans();
  const long long bx = policy.kind == CellPolicy::kOnePair ? std::min<long long>((max_n + 255) / 256, (long long)c.num_sms * 8)
                                                           : std::min<long long>((max_n + 255) / 256, 64);
  k_bbox_init<<<(6 * nc + 255) / 256, 256, 0, st>>>(c.bbox_keys.p, nc);
  k_bbox<<<dim3((unsigned)std::max<long long>(bx, 1), nc), 256, 0, st>>>(table, plans[0], c.bbox_keys.p);
  SICP_CUDA(cudaMemcpyAsync(c.grid_host, c.bbox_keys.p, sizeof(unsigned long long) * 6 * (size_t)nc,
                            cudaMemcpyDeviceToHost, st));
  c.tm.kernel_launches += 2;
  tr("bbox queued");
  SICP_CUDA(cudaStreamSynchronize(st));
  tr("bbox synced");
  std::vector<double> lo((size_t)nc * 3), ext((size_t)nc * 3);
  std::vector<CellPlan> cp((size_t)nc);
  for (int i = 0; i < nc; ++i) {
    for (int a = 0; a < 3; ++a) {
      lo[(size_t)i * 3 + a] = host_key_to_f64(c.grid_host[6 * i + a]);
      ext[(size_t)i * 3 + a] = host_key_to_f64(c.grid_host[6 * i + 3 + a]) - lo[(size_t)i * 3 + a];
      SICP_REQUIRE(std::isfinite(lo[(size_t)i * 3 + a]) && std::isfinite(ext[(size_t)i * 3 + a]), SICP_ERR_BAD_ARG,
                   "point cloud contains non-finite coordinates");
    }
    cp[(size_t)i] = first_cell_plan(&ext[(size_t)i * 3], plans[(size_t)i].n, policy);
  }

  // ---- cell sizes: count under every cloud's plan, one occupancy read-back per attempt
  const unsigned cx = (unsigned)((max_n + 255) / 256);
  long long total_cells = 0;
  for (int attempt = 0;; ++attempt) {
    total_cells = 0;
    for (int i = 0; i < nc; ++i) {
      CloudPlan& pl = plans[(size_t)i];
      const CellPlan& q = cp[(size_t)i];
      pl.ox = lo[(size_t)i * 3 + 0];
      pl.oy = lo[(size_t)i * 3 + 1];
      pl.oz = lo[(size_t)i * 3 + 2];
      pl.h = q.h;
      pl.inv_h = 1.0 / q.h;
      pl.nx = (int)q.d[0];
      pl.ny = (int)q.d[1];
      pl.nz = (int)q.d[2];
      pl.cell_base = total_cells;
      total_cells += q.cells();
    }
    SICP_REQUIRE(total_cells < (1ll << 31), SICP_ERR_BAD_ARG, "batch needs too many grid cells: use smaller batches");
    upload_plans();
    g.cell_table.reserve(total_cells + 1);
    g.fill.reserve(total_cells + 1);
    SICP_CUDA(cudaMemsetAsync(g.fill.p, 0, (size_t)total_cells * sizeof(uint32_t), st));
    SICP_CUDA(cudaMemsetAsync(c.grid_occ.p, 0, (size_t)nc * sizeof(unsigned int), st));
    k_cell_count<<<dim3(cx, nc), 256, 0, st>>>(table, plans[0], g.cid.p, g.fill.p, c.grid_occ.p);
    c.tm.kernel_launches += 1;
    unsigned int* occ_host = reinterpret_cast<unsigned int*>(c.grid_host);
    SICP_CUDA(cudaMemcpyAsync(occ_host, c.grid_occ.p, sizeof(unsigned int) * (size_t)nc, cudaMemcpyDeviceToHost, st));
    tr("count queued");
    SICP_CUDA(cudaStreamSynchronize(st));
    tr("count synced");
    bool again = false;
    for (int i = 0; i < nc; ++i) {
      CellPlan& q = cp[(size_t)i];
      if (q.final) continue;
      next_cell_plan(q, &ext[(size_t)i * 3], plans[(size_t)i].n, occ_host[i], attempt, policy);
      again = again || !q.final;
    }
    if (!again) break;
  }

  // ---- exclusive scan of the concatenated counters -> global record positions, then the records
  scan_u32(c, g.fill.p, total_cells, g.cell_table.p, g.block_sums);
  SICP_CUDA(cudaMemsetAsync(g.fill.p, 0, (size_t)total_cells * sizeof(uint32_t), st));
  k_scatter<<<dim3(cx, nc), 256, 0, st>>>(table, plans[0], g.cid.p, g.cell_table.p, g.fill.p, g.recs.p);
  c.tm.kernel_launches += 1;
  // optional: order the records of every cell by index (reproducible memory layout for profiling;
  // the search results never depend on it because ties are broken by index)
  if (c.grid_sort_cells) {
    k_sort_cells<<<(unsigned)((total_cells + 255) / 256), 256, 0, st>>>(g.cell_table.p, total_cells, g.recs.p);
    c.tm.kernel_launches += 1;
  }
  SICP_CUDA(cudaGetLastError());
  tr("scatter queued");
  views.resize((size_t)nc);
  centres.resize((size_t)nc * 3);
  for (int i = 0; i < nc; ++i) {
    const CloudPlan& pl = plans[(size_t)i];
    GridView v;
    v.recs = g.recs.p;
    v.cell_start = g.cell_table.p + pl.cell_base;
    v.ox = pl.ox;
    v.oy = pl.oy;
    v.oz = pl.oz;
    v.h = pl.h;
    v.inv_h = pl.inv_h;
    v.nx = pl.nx;
    v.ny = pl.ny;
    v.nz = pl.nz;
    v.n_points = total_pts;  // positions in the shared record array are global
    views[(size_t)i] = v;
    centres[(size_t)i * 3 + 0] = pl.ox + 0.5 * pl.nx * pl.h;
    centres[(size_t)i * 3 + 1] = pl.oy + 0.5 * pl.ny * pl.h;
    centres[(size_t)i * 3 + 2] = pl.oz + 0.5 * pl.nz * pl.h;
  }
}

void grid_build_pair(Ctx& c, Grid& g, const double* xyz, long long n) {
  g.built = false;
  std::vector<GridView> views;
  std::vector<double> centres;  // the one-pair solve centres on make_float4_copy's mov_center instead
  grid_build(c, g.bufs, {HostCloud{xyz, n, 0}}, CellPolicy{CellPolicy::kOnePair, c.grid_target_occ}, views, centres);
  g.view = views[0];
  g.built = true;
}

void make_float4_copy(Ctx& c) {
  // centred float4 copy of the movable cloud in caller order (TMA brute-force engine)
  const GridView v = c.gmov.view;
  double hi[3] = {v.ox + v.nx * v.h, v.oy + v.ny * v.h, v.oz + v.nz * v.h};
  c.mov_center[0] = 0.5 * (v.ox + hi[0]);
  c.mov_center[1] = 0.5 * (v.oy + hi[1]);
  c.mov_center[2] = 0.5 * (v.oz + hi[2]);
  c.mov_radius = 0.5 * std::max(hi[0] - v.ox, std::max(hi[1] - v.oy, hi[2] - v.oz));
  long long n_pad = ((c.n_mov + kBfTile - 1) / kBfTile) * kBfTile;
  c.mov_f4.reserve(n_pad);
  k_float4_copy<<<(unsigned)((n_pad + 255) / 256), 256, 0, c.stream>>>(
      c.mov_xyz.p, c.n_mov, n_pad, c.mov_center[0], c.mov_center[1], c.mov_center[2], c.mov_f4.p);
  SICP_CUDA(cudaGetLastError());
  c.tm.kernel_launches += 1;
}

}  // namespace sicp
