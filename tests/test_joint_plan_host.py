"""The plan of the sparse joint solve (csrc/joint_plan.h) and simpleicp_joint's solver argument.

CPU: joint_plan.h compiled with g++.  On paths, rings, strips with closures, a 2-D grid, a star, a
complete graph, disconnected pieces with singletons and duplicated pairs: the ordering is a
permutation; NumPy's Cholesky of a random diagonally dominant SPD matrix with the graph's 6 x 6
block pattern, in the plan's order, is exactly zero outside the symbolic pattern; every child and
every updating descendant sits at a lower level than its ancestor; the row maps land where the
union rule says; two builds are identical.  A NumPy statement of k_joint_sparse_solve's arithmetic
on the plan (assembly, left-looking updates, the column Cholesky with the right-hand side as the
last row, back substitution by level) solves the system as np.linalg.solve does.  Also the
wrapper's checks of `solver` and the header's documentation of the option joint_solver."""
import ctypes as C
import re
import subprocess

import numpy as np
import pytest

import simpleicp_b200 as sb
from conftest import REPO

JOINT_PLAN_FIELDS = ["perm", "first", "parent", "level", "st_off", "st", "up_off", "up", "up_i0", "up_nj", "up_map",
                     "map", "lv_off", "lv", "panel"]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("joint_plan") / "libjoint_plan_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", str(REPO / "tests" / "native" / "joint_plan_host.cpp"),
                    "-o", str(out)], check=True)
    lib = C.CDLL(str(out))
    lib.joint_plan_build.restype = C.c_longlong
    lib.joint_plan_limits.restype = C.c_longlong
    return lib


def make_plan(lib, F, pairs):
    p = np.ascontiguousarray(np.asarray(pairs, dtype=np.int32).reshape(-1, 2))
    n = lib.joint_plan_build(F, len(p), p.ctypes.data_as(C.c_void_p), None, C.c_longlong(0))
    buf = np.zeros(n, dtype=np.int64)
    lib.joint_plan_build(F, len(p), p.ctypes.data_as(C.c_void_p), buf.ctypes.data_as(C.c_void_p), C.c_longlong(n))
    pl = {"F": int(buf[0]), "n_super": int(buf[1]), "depth": int(buf[2])}
    at = 3
    for f in JOINT_PLAN_FIELDS:
        k = int(buf[at])
        pl[f] = buf[at + 1:at + 1 + k].copy()
        at += 1 + k
    return pl


# --------------------------------------------------------------------------- graphs (free indices)
def strip_pairs(n, n_edges, seed=11):
    """The free-free pairs of tests/test_gpu_joint.py's strip(n, ., n_edges) with cloud 0 fixed:
    (i, i + 1), (i, i + 2) and random closures 3 <= j - i <= 10, shifted to free indices."""
    rng = np.random.default_rng(seed)
    edges = [(i, i + 1) for i in range(n - 1)] + [(i, i + 2) for i in range(n - 2)]
    seen = set(edges)
    while len(edges) < n_edges:
        i = int(rng.integers(0, n - 3))
        j = i + int(rng.integers(3, 11))
        if j < n and (i, j) not in seen:
            seen.add((i, j))
            edges.append((i, j))
    return n - 1, [(a - 1, b - 1) for a, b in edges if a > 0 and b > 0]


def graph(name):
    if name == "path":
        return 60, [(i, i + 1) for i in range(59)]
    if name == "ring":
        return 70, [(i, (i + 1) % 70) for i in range(70)]
    if name == "strip_128":
        return strip_pairs(128, 400)
    if name == "strip_256":
        return strip_pairs(256, 800)
    if name == "grid_2d":
        return 256, [(16 * r + c, 16 * r + c + 1) for r in range(16) for c in range(15)] + \
                    [(16 * r + c, 16 * (r + 1) + c) for r in range(15) for c in range(16)]
    if name == "star":
        return 100, [(0, i) for i in range(1, 100)]
    if name == "complete_40":
        return 40, [(i, j) for i in range(40) for j in range(i + 1, 40)]
    if name == "pieces":
        # a path of 30, a ring of 25, a strip of 40, singletons 95..99 (every edge to a fixed cloud)
        return 100, [(i, i + 1) for i in range(29)] + [(30 + i, 30 + (i + 1) % 25) for i in range(25)] + \
                    [(55 + a, 55 + b) for a, b in strip_pairs(41, 120, seed=3)[1]]
    if name == "duplicates":
        F, p = strip_pairs(64, 200, seed=5)
        return F, p + [(b, a) for a, b in p[::3]] + p[::7] + [(3, 3)]
    raise KeyError(name)


GRAPHS = ["path", "ring", "strip_128", "strip_256", "grid_2d", "star", "complete_40", "pieces", "duplicates"]


def owner_of(pl):
    own = np.zeros(pl["F"], dtype=np.int64)
    for s in range(pl["n_super"]):
        own[pl["first"][s]:pl["first"][s + 1]] = s
    return own


def struct(pl, s):
    return pl["st"][pl["st_off"][s]:pl["st_off"][s + 1]]


def spd_matrix(F, pairs, seed=0):
    """A random diagonally dominant SPD matrix with one 6 x 6 block per pair and on the diagonal."""
    rng = np.random.default_rng(seed)
    N = np.zeros((6 * F, 6 * F))
    for a, b in sorted({(min(a, b), max(a, b)) for a, b in pairs if a != b}):
        B = rng.uniform(-1.0, 1.0, (6, 6))
        N[6 * a:6 * a + 6, 6 * b:6 * b + 6] = B
        N[6 * b:6 * b + 6, 6 * a:6 * a + 6] = B.T
    N += np.diag(np.abs(N).sum(1) + rng.uniform(1.0, 2.0, 6 * F))
    return N


def expand(clouds):
    return (6 * np.asarray(clouds, dtype=np.int64)[:, None] + np.arange(6)).ravel()


# --------------------------------------------------------------------------- the plan
@pytest.mark.parametrize("name", GRAPHS)
def test_plan_structure(lib, name):
    F, pairs = graph(name)
    pl = make_plan(lib, F, pairs)
    perm, S = pl["perm"], pl["n_super"]
    assert np.array_equal(np.sort(perm), np.arange(F))
    assert pl["first"][0] == 0 and pl["first"][-1] == F and np.all(np.diff(pl["first"]) > 0)
    # leaves of the dissection hold at most L clouds; a separator or a component without a
    # separating level may hold more
    own = owner_of(pl)
    pos = np.empty(F, dtype=np.int64)
    pos[perm] = np.arange(F)
    level, parent = pl["level"], pl["parent"]
    for s in range(S):
        t = struct(pl, s)
        assert np.all(np.diff(t) > 0) and (t.size == 0 or t[0] >= pl["first"][s + 1])
        if t.size:
            assert parent[s] == own[t[0]] and level[parent[s]] > level[s]
        else:
            assert parent[s] == -1
        kids = np.flatnonzero(parent == s)
        assert level[s] == (0 if kids.size == 0 else 1 + level[kids].max())
        # the updates of s: descendants in ascending order, at lower levels, with their row maps
        cols = np.arange(pl["first"][s], pl["first"][s + 1])
        ds = []
        for u in range(pl["up_off"][s], pl["up_off"][s + 1]):
            d, i0, nj, mo = (int(pl[f][u]) for f in ("up", "up_i0", "up_nj", "up_map"))
            ds.append(d)
            assert d < s and level[d] < level[s]
            td = struct(pl, d)
            assert (i0 == 0 or td[i0 - 1] < cols[0]) and nj >= 1
            assert np.all(np.isin(td[i0:i0 + nj], cols)) and not np.any(np.isin(td[i0 + nj:], cols))
            rows = np.concatenate((cols, t))
            assert np.array_equal(rows[pl["map"][mo:mo + td.size - i0]], td[i0:])
        want = [d for d in range(s) if np.any(np.isin(struct(pl, d), cols))]
        assert ds == want
    assert np.array_equal(np.sort(pl["lv"]), np.arange(S))
    for l in range(pl["depth"]):
        assert np.all(level[pl["lv"][pl["lv_off"][l]:pl["lv_off"][l + 1]]] == l)
    ns, nt = np.diff(pl["first"]), np.diff(pl["st_off"])
    assert np.array_equal(np.diff(pl["panel"]), (6 * (ns + nt) + 1) * 6 * ns)
    # two builds
    again = make_plan(lib, F, pairs)
    assert all(np.array_equal(pl[f], again[f]) for f in JOINT_PLAN_FIELDS) and pl["depth"] == again["depth"]


@pytest.mark.parametrize("name", GRAPHS)
def test_cholesky_stays_inside_the_symbolic_pattern(lib, name):
    F, pairs = graph(name)
    pl = make_plan(lib, F, pairs)
    N = spd_matrix(F, pairs)
    Lc = np.linalg.cholesky(N[np.ix_(expand(pl["perm"]), expand(pl["perm"]))])
    allowed = np.zeros((F, F), dtype=bool)
    for s in range(pl["n_super"]):
        cols = np.arange(pl["first"][s], pl["first"][s + 1])
        rows = np.concatenate((cols, struct(pl, s)))
        allowed[np.ix_(rows, cols)] = True
    nz = np.abs(Lc).reshape(F, 6, F, 6).max(axis=(1, 3)) > 0
    assert not np.any(nz & ~allowed), np.argwhere(nz & ~allowed)[:5]


def supernodal_solve(pl, N, b, fault=None):
    """k_joint_sparse_solve's arithmetic on the plan: the panels assembled from N (free-cloud order)
    and b as their last row, the descendants' updates, the column Cholesky, and the back
    substitution from the top level down.  Returns x in free-cloud order.  `fault` = (kind, s, u)
    makes one deliberate mistake in supernode s, as a wrong kernel would: "drop" skips update u,
    "flip" negates the off-diagonal 6 x 6 block u = (row block, column block) of its panel,
    "stale" sends the last row of update u's map to the panel row block that precedes it."""
    perm, S = pl["perm"], pl["n_super"]
    panels = []
    for s in range(S):
        cols = np.arange(pl["first"][s], pl["first"][s + 1])
        rows = np.concatenate((cols, struct(pl, s)))
        Cn, R = 6 * cols.size, 6 * rows.size + 1
        P = np.zeros((R, Cn))
        P[:R - 1] = N[np.ix_(expand(perm[rows]), expand(perm[cols]))]
        P[R - 1] = b[expand(perm[cols])]
        if fault and fault[0] == "flip" and fault[1] == s:
            i, j = fault[2]
            P[6 * i:6 * i + 6, 6 * j:6 * j + 6] *= -1.0
        for u in range(pl["up_off"][s], pl["up_off"][s + 1]):
            if fault and fault[0] == "drop" and fault[1:] == (s, u):
                continue
            d, i0, nj, mo = (int(pl[f][u]) for f in ("up", "up_i0", "up_nj", "up_map"))
            Pd = panels[d]
            r0 = 6 * (pl["first"][d + 1] - pl["first"][d]) + 6 * i0
            m = pl["map"][mo:mo + (Pd.shape[0] - 1 - r0) // 6]
            if fault and fault[0] == "stale" and fault[1:] == (s, u):
                m = m.copy()
                m[-1] -= 1
            ti = np.concatenate((expand(m), [R - 1]))
            tj = expand(m[:nj])
            P[np.ix_(ti, tj)] -= Pd[r0:] @ Pd[r0:r0 + 6 * nj].T
        for j in range(Cn):
            piv = np.sqrt(P[j, j])
            P[j + 1:, j] /= piv
            P[j, j] = piv
            P[j + 1:, j + 1:] -= np.outer(P[j + 1:, j], P[j + 1:Cn, j])
        panels.append(P)
    x = np.zeros(6 * pl["F"])
    for l in range(pl["depth"] - 1, -1, -1):
        for s in pl["lv"][pl["lv_off"][l]:pl["lv_off"][l + 1]]:
            P = panels[s]
            Cn = P.shape[1]
            t = P[-1] - P[Cn:-1].T @ x[expand(perm[struct(pl, s)])]
            Lss = np.tril(P[:Cn])
            x[expand(perm[np.arange(pl["first"][s], pl["first"][s + 1])])] = np.linalg.solve(Lss.T, t)
    return x


@pytest.mark.parametrize("name", GRAPHS)
def test_supernodal_solve_equals_the_dense_solve(lib, name):
    F, pairs = graph(name)
    pl = make_plan(lib, F, pairs)
    N = spd_matrix(F, pairs, seed=1)
    b = np.random.default_rng(2).normal(size=6 * F)
    x = supernodal_solve(pl, N, b)
    ref = np.linalg.solve(N, b)
    assert np.abs(x - ref).max() <= 1e-11 * np.abs(ref).max()


def backward_error(N, b, x):
    """eta = |b - N x|_inf / (|N|_inf |x|_inf + |b|_inf), the residual in extended precision: the
    normwise backward error of x as a solution of N x = b (DESIGN.md §6.11)."""
    r = np.asarray(b, dtype=np.longdouble) - np.asarray(N, dtype=np.longdouble) @ np.asarray(x, dtype=np.longdouble)
    return float(np.abs(r).max() / (np.abs(N).sum(1).max() * np.abs(x).max() + np.abs(b).max()))


def test_backward_error_catches_a_wrong_update_sign_or_row_map(lib):
    """The metric of the GPU backward-error tests (tests/test_gpu_joint_graphs.py) on the 2-D grid,
    against the restatement above with one mistake at a time: the last update of the supernode
    with the most updates dropped, the sign of one off-diagonal block, one stale row of a
    map.  The correct solve is at rounding level (measured 1.6e-16); each mistake is at least 1e-8."""
    F, pairs = graph("grid_2d")
    pl = make_plan(lib, F, pairs)
    N = spd_matrix(F, pairs, seed=1)
    b = np.random.default_rng(2).normal(size=6 * F)
    assert backward_error(N, b, supernodal_solve(pl, N, b)) <= 1e-14
    n_up = np.diff(pl["up_off"])
    s = int(np.argmax(n_up))
    assert n_up[s] >= 2
    u_last = int(pl["up_off"][s + 1]) - 1
    # the first supernode with an off-diagonal block that N holds; the first update whose map has
    # rows below the columns it updates
    def rows(t):
        return pl["perm"][np.concatenate((np.arange(pl["first"][t], pl["first"][t + 1]), struct(pl, t)))]

    s_fl, flip = next((t, (i, j)) for t in range(pl["n_super"]) for j in range(pl["first"][t + 1] - pl["first"][t])
                      for i in range(j + 1, rows(t).size)
                      if np.any(N[6 * rows(t)[i]:6 * rows(t)[i] + 6, 6 * rows(t)[j]:6 * rows(t)[j] + 6]))
    s_st, stale = next((t, u) for t in range(pl["n_super"]) for u in range(pl["up_off"][t], pl["up_off"][t + 1])
                       if struct(pl, int(pl["up"][u])).size - int(pl["up_i0"][u]) > int(pl["up_nj"][u]))
    for fault in (("drop", s, u_last), ("flip", s_fl, flip), ("stale", s_st, stale)):
        eta = backward_error(N, b, supernodal_solve(pl, N, b, fault))
        assert eta >= 1e-8, (fault, eta)


def test_strip_of_4096_clouds_has_a_shallow_tree(lib):
    """The §6.10 strip: 4095 free clouds, about 3 edges per cloud.  Nested dissection halves it at
    every level, so the tree is about log2(4095 / 16) + 1 levels deep."""
    F, pairs = strip_pairs(4096, 12_800)
    pl = make_plan(lib, F, pairs)
    sizes = np.diff(pl["first"])
    print(f"strip 4096: supernodes {pl['n_super']}, depth {pl['depth']}, largest {sizes.max()} clouds, "
          f"factor {8 * pl['panel'][-1] / 2**20:.1f} MiB")
    assert pl["depth"] <= 16
    assert 8 * pl["panel"][-1] < 1 << 30


def test_limits(lib):
    assert lib.joint_plan_limits(0) == 16384 and lib.joint_plan_limits(2) == 4 << 30
    assert 8 <= lib.joint_plan_limits(1) <= 16


# --------------------------------------------------------------------------- simpleicp_joint(solver=)
def _clouds(n=3, m=200):
    rng = np.random.default_rng(1)
    return [rng.normal(size=(m, 3)) for _ in range(n)]


@pytest.mark.parametrize("solver", ["Sparse", "cholesky", "", None, 1])
def test_solver_must_be_dense_or_sparse(solver):
    with pytest.raises(ValueError, match="solver must be 'dense' or 'sparse'"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], solver=solver)


def test_covariances_need_the_dense_solver():
    with pytest.raises(ValueError, match="covariances=True needs solver='dense'"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], solver="sparse", covariances=True)


def test_more_than_16384_free_clouds_are_refused_by_the_sparse_solver():
    clouds = [np.zeros((20, 3))] * 16386
    edges = [(0, i) for i in range(1, 16386)]
    with pytest.raises(ValueError, match="between 1 and 16384 free clouds under solver=sparse"):
        sb.simpleicp_joint(clouds, edges, solver="sparse")


def test_header_documents_joint_solver():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    entry = header[:header.index("int32_t sicp_register_joint(")]
    doc = entry[entry.rindex("/* ----"):]
    assert '"joint_solver"' in doc and "16 384" in doc and "SICP_ERR_STATE" in doc
    keys = re.search(r"/\*  keys:(.*?)\*/", header, re.S).group(1)
    assert '"joint_solver"' in keys
