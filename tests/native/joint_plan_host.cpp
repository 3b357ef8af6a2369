// Host shim for tests: exposes the sparse joint solve's plan (joint_plan.h) to ctypes.  The plan
// travels as one int64 array: F, n_super, depth, then each array of the plan as its length followed
// by its entries, in the order of JOINT_PLAN_FIELDS in tests/test_joint_plan_host.py.
#include <utility>
#include <vector>

#include "../../simpleicp_b200/csrc/joint_plan.h"

extern "C" {
// the plan of F free clouds joined by the n pairs (pairs[2 i], pairs[2 i + 1]); returns the length
// of the serialised plan and writes it to out when it fits in cap
long long joint_plan_build(int F, int n, const int* pairs, long long* out, long long cap) {
  std::vector<std::pair<int, int>> p;
  for (int i = 0; i < n; ++i) p.emplace_back(pairs[2 * i], pairs[2 * i + 1]);
  const sicp::JointPlan pl = sicp::make_joint_plan(F, p);
  std::vector<long long> v{pl.F, pl.n_super, pl.depth};
  auto put = [&](const auto& a) {
    v.push_back((long long)a.size());
    v.insert(v.end(), a.begin(), a.end());
  };
  put(pl.perm);
  put(pl.first);
  put(pl.parent);
  put(pl.level);
  put(pl.st_off);
  put(pl.st);
  put(pl.up_off);
  put(pl.up);
  put(pl.up_i0);
  put(pl.up_nj);
  put(pl.up_map);
  put(pl.map);
  put(pl.lv_off);
  put(pl.lv);
  put(pl.panel);
  if ((long long)v.size() <= cap)
    for (size_t i = 0; i < v.size(); ++i) out[i] = v[i];
  return (long long)v.size();
}
long long joint_plan_limits(int which) {
  return which == 0 ? sicp::JOINT_SPARSE_MAX_FREE : which == 1 ? sicp::JOINT_PLAN_LEAF : sicp::JOINT_SPARSE_MAX_BYTES;
}
}
