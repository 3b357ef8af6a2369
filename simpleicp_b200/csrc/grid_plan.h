// grid_plan.h — the cell-size rules of the grid builder (grid.cu: grid_build).  Plain host code:
// tests/native/grid_plan_host.cpp compiles it with g++.
//
// A cloud's grid cuts its bounding box [lo, lo + ext] into cubic cells of size h, with
// dims[a] = floor(ext[a] / h) + 1.  The first h assumes a 2-D manifold in 3-D (scans); every
// later attempt rescales h from the occupancy the previous one measured (points per occupied
// cell), for at most four attempts.  The two policies differ in the cell cap and in when a plan is
// final:
//   one pair (sicp_set_clouds, sicp_estimate_normals, sicp_register): cap 2^25 cells; final at the
//     last attempt, inside the band, or when the cells are too full and twice as many would pass
//     the cap;
//   batch (both sides of a batch, the resident map, the grids of sicp_map_insert): cap
//     min(2^25, max(4096, 32 n)); final at the last attempt, inside the band, or once the cap has
//     forced h up.
#pragma once
#include <algorithm>
#include <cmath>

namespace sicp {

constexpr long long kMaxGridCells = 1ll << 25;  // 32 M cells (128 MB of cell table)
constexpr int kGridAttempts = 4;

struct CellPolicy {
  enum Kind { kOnePair, kBatch } kind;
  double target;  // points per occupied cell (option "grid_target_occupancy")
  long long cap(long long n) const {
    return kind == kOnePair ? kMaxGridCells : std::min<long long>(kMaxGridCells, std::max<long long>(4096, 32 * n));
  }
};

// One cloud's cell size and dims during a build.
struct CellPlan {
  double h = 1.0;
  long long d[3] = {1, 1, 1};
  bool capped = false;  // the last fit had to grow h to stay under the cap
  bool final = false;
  long long cells() const { return d[0] * d[1] * d[2]; }
};

// dims of the plan's h; h grows by 1.26 (2x fewer cells per step) while they exceed the cap
inline void fit_dims(CellPlan& pl, const double ext[3], long long cap) {
  pl.capped = false;
  for (;;) {
    for (int a = 0; a < 3; ++a) pl.d[a] = std::max<long long>(1, (long long)std::floor(ext[a] / pl.h) + 1);
    if (pl.cells() <= cap) return;
    pl.h *= 1.26;
    pl.capped = true;
  }
}

// the plan of the first attempt: h ~ sqrt(target * A / n), A the product of the two largest extents
inline CellPlan first_cell_plan(const double ext[3], long long n, const CellPolicy& p) {
  double e[3] = {ext[0], ext[1], ext[2]};
  std::sort(e, e + 3);
  const double emax = std::max(e[2], 1e-12);
  const double area = std::max(e[2] * std::max(e[1], 1e-3 * emax), 1e-300);
  CellPlan pl;
  pl.h = std::max(std::sqrt(p.target * area / (double)std::max<long long>(n, 1)), emax * 1e-6);
  fit_dims(pl, ext, p.cap(n));
  return pl;
}

inline bool occupancy_in_band(double occ, double target) { return occ <= target * 1.6 && occ >= target / 1.6; }

// the occupancy of occupied cells scales ~ h^dim with dim in [2, 3] for scan data; use 2.3
inline double refine_factor(double occ, double target) {
  const double f = std::pow(target / occ, 1.0 / 2.3);
  return std::min(std::max(f, 0.25), 4.0);
}

// Attempt `attempt` counted n_occupied occupied cells under the plan: mark it final, or rescale h
// and fit the dims for the next attempt.
inline void next_cell_plan(CellPlan& pl, const double ext[3], long long n, long long n_occupied, int attempt,
                           const CellPolicy& p) {
  const double occ = (double)n / (double)std::max<long long>(n_occupied, 1);
  const bool stop = attempt == kGridAttempts - 1 || occupancy_in_band(occ, p.target) ||
                    (p.kind == CellPolicy::kOnePair ? occ > p.target && pl.cells() * 2 > kMaxGridCells : pl.capped);
  if (stop) {
    pl.final = true;
    return;
  }
  pl.h *= refine_factor(occ, p.target);
  fit_dims(pl, ext, p.cap(n));
}

}  // namespace sicp
