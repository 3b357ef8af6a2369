// Host shim for tests: exposes the cell-size rules of the grid builder (grid_plan.h) to ctypes.
// The plan travels as (h, d[3], capped); one_pair selects the policy.
#include "../../simpleicp_b200/csrc/grid_plan.h"

namespace {
sicp::CellPolicy policy(int one_pair, double target) {
  return sicp::CellPolicy{one_pair ? sicp::CellPolicy::kOnePair : sicp::CellPolicy::kBatch, target};
}
void store(const sicp::CellPlan& pl, double* h, long long* d, int* capped) {
  *h = pl.h;
  for (int a = 0; a < 3; ++a) d[a] = pl.d[a];
  *capped = pl.capped ? 1 : 0;
}
}  // namespace

extern "C" {
void grid_plan_first(int one_pair, double target, const double* ext, long long n, double* h, long long* d,
                     int* capped) {
  store(sicp::first_cell_plan(ext, n, policy(one_pair, target)), h, d, capped);
}
// returns 1 when the plan is final (h, d, capped unchanged), else 0 with the next attempt's plan
int grid_plan_next(int one_pair, double target, const double* ext, long long n, long long n_occupied, int attempt,
                   double* h, long long* d, int* capped) {
  sicp::CellPlan pl;
  pl.h = *h;
  for (int a = 0; a < 3; ++a) pl.d[a] = d[a];
  pl.capped = *capped != 0;
  sicp::next_cell_plan(pl, ext, n, n_occupied, attempt, policy(one_pair, target));
  store(pl, h, d, capped);
  return pl.final ? 1 : 0;
}
}
