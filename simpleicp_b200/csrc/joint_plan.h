// joint_plan.h — the host plan of the sparse joint solve (option "joint_solver" 1, DESIGN.md §6.11):
// a nested-dissection ordering of the free clouds, its supernodes, the symbolic factorisation and
// the level schedule of k_joint_sparse_solve.  Plain C++ (the tests compile it with g++); a pure
// function of F and the free-free adjacency, so the same edges give the same plan.
#pragma once
#include <algorithm>
#include <utility>
#include <vector>

namespace sicp {

constexpr int JOINT_SPARSE_MAX_FREE = 16384;
constexpr int JOINT_PLAN_LEAF = 16;                          // clouds per leaf of the dissection, at most
constexpr long long JOINT_SPARSE_MAX_BYTES = 4ll << 30;      // the factor's panels, at most

// Supernode s holds the clouds at positions first[s] .. first[s + 1] - 1 of the new order (6 unknowns
// each).  Its panel is the column-major (6 ns + 6 nt + 1) x 6 ns block of the factor: its own
// columns' rows, then the rows of struct(s) (nt clouds, ascending positions), then the right-hand
// side's row.  Supernodes are numbered in elimination order, so every descendant precedes s.
struct JointPlan {
  int F = 0, n_super = 0, depth = 0;
  std::vector<int> perm;        // position -> free cloud
  std::vector<int> pos;         // free cloud -> position
  std::vector<int> first;       // n_super + 1
  std::vector<int> parent;      // -1 for a root
  std::vector<int> level;       // 0 for a leaf of the tree, else 1 + the largest level of its children
  std::vector<int> st_off, st;  // struct(s) = st[st_off[s] .. st_off[s + 1]): positions after s's
  // the descendants d whose struct meets s, ascending: up[u] = d, up_i0[u] = the first entry of
  // struct(d) at or after first[s], up_nj[u] = the entries inside s; map[up_map[u] + i] = the
  // panel cloud row of s that entry up_i0[u] + i of struct(d) falls on
  std::vector<int> up_off, up, up_i0, up_nj, up_map, map;
  std::vector<int> lv_off, lv;  // the supernodes of each level, ascending
  std::vector<long long> panel; // n_super + 1 offsets into the factor, in doubles
  int ns(int s) const { return first[(size_t)s + 1] - first[(size_t)s]; }
  int nt(int s) const { return st_off[(size_t)s + 1] - st_off[(size_t)s]; }
  long long factor_bytes() const { return 8 * panel.back(); }
};

namespace joint_plan_detail {

struct Dissect {
  const std::vector<std::vector<int>>& adj;
  std::vector<int> tag, lvl;
  int next_tag = 1;
  JointPlan& pl;

  int degree_in(int v, int t) const {
    int d = 0;
    for (int u : adj[(size_t)v]) d += tag[(size_t)u] == t;
    return d;
  }
  // BFS of the vertices tagged t from r, neighbours in ascending order: the visit order, and the
  // level of every visited vertex in lvl
  std::vector<int> bfs(int r, int t) {
    std::vector<int> order{r};
    lvl[(size_t)r] = 0;
    std::vector<int> seen{r};
    tag[(size_t)r] = -t;  // visited
    for (size_t h = 0; h < order.size(); ++h)
      for (int u : adj[(size_t)order[h]])
        if (tag[(size_t)u] == t) {
          tag[(size_t)u] = -t;
          lvl[(size_t)u] = lvl[(size_t)order[h]] + 1;
          order.push_back(u);
        }
    for (int v : order) tag[(size_t)v] = t;
    return order;
  }
  void emit(const std::vector<int>& V) {
    pl.perm.insert(pl.perm.end(), V.begin(), V.end());
    pl.first.push_back((int)pl.perm.size());
  }
  // V: one connected set of vertices tagged t, ascending
  void run(const std::vector<int>& V, int t) {
    if ((int)V.size() <= JOINT_PLAN_LEAF) return emit(V);
    // pseudo-peripheral vertex (George-Liu): from the smallest index, move to the vertex of least
    // degree (then smallest index) in the last level while the eccentricity grows
    int r = V[0];
    std::vector<int> order = bfs(r, t);
    for (;;) {
      const int ecc = lvl[(size_t)order.back()];
      int best = -1;
      for (int v : order)
        if (lvl[(size_t)v] == ecc &&
            (best < 0 || degree_in(v, t) < degree_in(best, t) || (degree_in(v, t) == degree_in(best, t) && v < best)))
          best = v;
      std::vector<int> o2 = bfs(best, t);
      if (lvl[(size_t)o2.back()] <= ecc) {
        order = bfs(r, t);
        break;
      }
      r = best;
      order = std::move(o2);
    }
    const int e = lvl[(size_t)order.back()];
    if (e < 2) return emit(V);  // every vertex within one step of r: no separating level
    // the level of the middle vertex in BFS order, kept off both ends
    const int k = std::min(std::max(lvl[(size_t)order[order.size() / 2]], 1), e - 1);
    std::vector<int> S;
    const int ts = next_tag++;
    for (int v : V)
      if (lvl[(size_t)v] == k) {
        S.push_back(v);
        tag[(size_t)v] = ts;
      }
    // the pieces: components of V \ S in order of their smallest vertex
    std::vector<std::pair<std::vector<int>, int>> pieces;
    for (int v : V) {
      if (tag[(size_t)v] != t) continue;
      const int tp = next_tag++;
      std::vector<int> comp{v};
      tag[(size_t)v] = tp;
      for (size_t h = 0; h < comp.size(); ++h)
        for (int u : adj[(size_t)comp[h]])
          if (tag[(size_t)u] == t) {
            tag[(size_t)u] = tp;
            comp.push_back(u);
          }
      std::sort(comp.begin(), comp.end());
      pieces.emplace_back(std::move(comp), tp);
    }
    for (auto& p : pieces) run(p.first, p.second);
    emit(S);
  }
};

}  // namespace joint_plan_detail

// The plan of F free clouds joined by the undirected pairs (a, b) of free indices (duplicates and
// self pairs are ignored).
inline JointPlan make_joint_plan(int F, const std::vector<std::pair<int, int>>& pairs) {
  JointPlan pl;
  pl.F = F;
  std::vector<std::vector<int>> adj((size_t)F);
  for (const auto& p : pairs)
    if (p.first != p.second) {
      adj[(size_t)p.first].push_back(p.second);
      adj[(size_t)p.second].push_back(p.first);
    }
  for (auto& a : adj) {
    std::sort(a.begin(), a.end());
    a.erase(std::unique(a.begin(), a.end()), a.end());
  }

  // ---- ordering: nested dissection of every connected component
  pl.first.push_back(0);
  {
    joint_plan_detail::Dissect d{adj, std::vector<int>((size_t)F, 0), std::vector<int>((size_t)F, 0), 1, pl};
    for (int v = 0; v < F; ++v) {
      if (d.tag[(size_t)v] != 0) continue;
      const int t = d.next_tag++;
      std::vector<int> comp{v};
      d.tag[(size_t)v] = t;
      for (size_t h = 0; h < comp.size(); ++h)
        for (int u : adj[(size_t)comp[h]])
          if (d.tag[(size_t)u] == 0) {
            d.tag[(size_t)u] = t;
            comp.push_back(u);
          }
      std::sort(comp.begin(), comp.end());
      d.run(comp, t);
    }
  }
  const int S = pl.n_super = (int)pl.first.size() - 1;
  pl.pos.assign((size_t)F, 0);
  for (int p = 0; p < F; ++p) pl.pos[(size_t)pl.perm[(size_t)p]] = p;
  std::vector<int> owner((size_t)F);
  for (int s = 0; s < S; ++s)
    for (int p = pl.first[(size_t)s]; p < pl.first[(size_t)s + 1]; ++p) owner[(size_t)p] = s;

  // ---- symbolic factorisation: struct(s) = s's adjacency after it, plus its children's structs
  // minus s; parent = the owner of struct(s)'s first position
  std::vector<std::vector<int>> children((size_t)S);
  std::vector<int> mark((size_t)F, -1);
  pl.parent.assign((size_t)S, -1);
  pl.level.assign((size_t)S, 0);
  pl.st_off.push_back(0);
  for (int s = 0; s < S; ++s) {
    const int lo = pl.first[(size_t)s], hi = pl.first[(size_t)s + 1];
    std::vector<int> rows;
    auto add = [&](int p) {
      if (p >= hi && mark[(size_t)p] != s) {
        mark[(size_t)p] = s;
        rows.push_back(p);
      }
    };
    for (int p = lo; p < hi; ++p)
      for (int u : adj[(size_t)pl.perm[(size_t)p]]) add(pl.pos[(size_t)u]);
    for (int ch : children[(size_t)s]) {
      for (int i = pl.st_off[(size_t)ch]; i < pl.st_off[(size_t)ch + 1]; ++i) add(pl.st[(size_t)i]);
      pl.level[(size_t)s] = std::max(pl.level[(size_t)s], pl.level[(size_t)ch] + 1);
    }
    std::sort(rows.begin(), rows.end());
    pl.st.insert(pl.st.end(), rows.begin(), rows.end());
    pl.st_off.push_back((int)pl.st.size());
    if (!rows.empty()) {
      pl.parent[(size_t)s] = owner[(size_t)rows[0]];
      children[(size_t)pl.parent[(size_t)s]].push_back(s);
    }
    pl.depth = std::max(pl.depth, pl.level[(size_t)s] + 1);
  }

  // ---- the updates of each supernode from its descendants, with their row maps
  std::vector<std::vector<int>> ups((size_t)S);
  for (int d = 0; d < S; ++d)
    for (int i = pl.st_off[(size_t)d]; i < pl.st_off[(size_t)d + 1];) {
      const int t = owner[(size_t)pl.st[(size_t)i]];
      int j = i;
      while (j < pl.st_off[(size_t)d + 1] && owner[(size_t)pl.st[(size_t)j]] == t) ++j;
      ups[(size_t)t].push_back(d);
      ups[(size_t)t].push_back(i - pl.st_off[(size_t)d]);
      ups[(size_t)t].push_back(j - i);
      i = j;
    }
  pl.up_off.push_back(0);
  for (int s = 0; s < S; ++s) {
    const int* sb = pl.st.data() + pl.st_off[(size_t)s];
    const int* se = pl.st.data() + pl.st_off[(size_t)s + 1];
    for (size_t u = 0; u < ups[(size_t)s].size(); u += 3) {
      const int d = ups[(size_t)s][u], i0 = ups[(size_t)s][u + 1];
      pl.up.push_back(d);
      pl.up_i0.push_back(i0);
      pl.up_nj.push_back(ups[(size_t)s][u + 2]);
      pl.up_map.push_back((int)pl.map.size());
      for (int i = pl.st_off[(size_t)d] + i0; i < pl.st_off[(size_t)d + 1]; ++i) {
        const int p = pl.st[(size_t)i];
        // struct(d) past s lies in struct(s) by the union rule: lower_bound finds it
        pl.map.push_back(owner[(size_t)p] == s ? p - pl.first[(size_t)s]
                                               : pl.ns(s) + (int)(std::lower_bound(sb, se, p) - sb));
      }
    }
    pl.up_off.push_back((int)pl.up.size());
  }

  // ---- schedule: the supernodes by level, and the panels
  pl.lv_off.assign((size_t)pl.depth + 1, 0);
  for (int s = 0; s < S; ++s) ++pl.lv_off[(size_t)pl.level[(size_t)s] + 1];
  for (int l = 0; l < pl.depth; ++l) pl.lv_off[(size_t)l + 1] += pl.lv_off[(size_t)l];
  pl.lv.assign((size_t)S, 0);
  std::vector<int> fill(pl.lv_off.begin(), pl.lv_off.end() - 1);
  for (int s = 0; s < S; ++s) pl.lv[(size_t)fill[(size_t)pl.level[(size_t)s]]++] = s;
  pl.panel.assign((size_t)S + 1, 0);
  for (int s = 0; s < S; ++s)
    pl.panel[(size_t)s + 1] = pl.panel[(size_t)s] + (6ll * (pl.ns(s) + pl.nt(s)) + 1) * (6ll * pl.ns(s));
  return pl;
}

}  // namespace sicp
