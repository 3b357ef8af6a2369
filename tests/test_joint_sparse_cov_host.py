"""The selected inversion of the sparse joint solve's factor (DESIGN.md §6.14) and the bindings of
sicp_get_joint_selected_covariances, without a GPU.

A NumPy statement of k_joint_selinv's recurrence runs over the plan that joint_plan.h builds
(compiled with g++ as test_joint_plan_host does): per supernode from the roots down, X = Z_TT L_TJ
with Z_TT gathered from the ancestors' blocks through the plan's own update lists and row maps
(up, map), Z_TJ = -X L_JJ^-1 row by row, and Z_JJ column by column from Z_JJ L_JJ = L_JJ^-T -
Z_TJ^T L_TJ.  On random SPD matrices with the plan's block pattern (a strip, a 2-D block, a star,
a complete graph, several components, a relabelled block) every block of the pattern matches
np.linalg.inv.  A pair outside the pattern is chosen from the plan, and w_a^T w_b of the forward
solves along the elimination-tree paths (k_joint_sel_parked) gives its block.  Also the argument
handling of simpleicp_joint(covariances=), the header and the ctypes declaration."""
import re

import numpy as np
import pytest

import simpleicp_b200 as sb
from conftest import REPO
from simpleicp_b200 import _capi
from test_joint_plan_host import expand, graph, lib, make_plan, owner_of, spd_matrix, struct  # noqa: F401


def factor_panels(pl, N):
    """The supernodal factor in the kernel's layout: per supernode the rows of its columns and
    struct, its columns; L from NumPy's Cholesky in the plan's order (exactly the supernodal one on
    the pattern, test_joint_plan_host)."""
    perm = pl["perm"]
    L = np.linalg.cholesky(N[np.ix_(expand(perm), expand(perm))])
    panels = []
    for s in range(pl["n_super"]):
        cols = np.arange(pl["first"][s], pl["first"][s + 1])
        rows = np.concatenate((cols, struct(pl, s)))
        panels.append(L[np.ix_(expand(rows), expand(cols))])
    return panels


def selected_inverse(pl, panels):
    """k_joint_selinv's arithmetic: per supernode k, from level depth - 1 down, the block of Z with
    the rows of its panel.  Z_TT's block (ca, cb), ca >= cb, lies in the column of cb in the block
    of cb's supernode t, at ca's row there: map[mo + ca - b0] with (b0, mo) of the update of t from k."""
    own = owner_of(pl)
    Z = [None] * pl["n_super"]
    for lvl in range(pl["depth"] - 1, -1, -1):
        for k in pl["lv"][pl["lv_off"][lvl]:pl["lv_off"][lvl + 1]]:
            st = struct(pl, k)
            ns, nt = pl["first"][k + 1] - pl["first"][k], st.size
            C, T = 6 * ns, 6 * nt
            P = panels[k]
            Ljj, Ltj = P[:C], P[C:]
            runs, b = [], 0
            while b < nt:  # the ancestors struct(k) falls in, by the update lists
                t = own[st[b]]
                us = [u for u in range(pl["up_off"][t], pl["up_off"][t + 1]) if pl["up"][u] == k]
                assert len(us) == 1 and pl["up_i0"][us[0]] == b
                runs.append((t, b, int(pl["up_map"][us[0]])))
                b += int(pl["up_nj"][us[0]])
            run_of = np.zeros(nt, dtype=np.int64)
            for i, (t, b0, mo) in enumerate(runs):
                run_of[b0:] = i
            Ztt = np.zeros((T, T))
            for ca in range(nt):
                for cb in range(ca + 1):
                    t, b0, mo = runs[run_of[cb]]
                    col, row = 6 * pl["map"][mo + cb - b0], 6 * pl["map"][mo + ca - b0]
                    blk = Z[t][row:row + 6, col:col + 6]
                    Ztt[6 * ca:6 * ca + 6, 6 * cb:6 * cb + 6] = blk
                    Ztt[6 * cb:6 * cb + 6, 6 * ca:6 * ca + 6] = blk.T
            X = Ztt @ Ltj
            Ztj = np.zeros((T, C))
            for j in range(C - 1, -1, -1):  # Z_TJ L_JJ = -X, each row
                Ztj[:, j] = (-X[:, j] - Ztj[:, j + 1:] @ Ljj[j + 1:, j]) / Ljj[j, j]
            B = -Ztj.T @ Ltj
            Zjj = np.zeros((C, C))
            for j in range(C - 1, -1, -1):
                i = np.arange(j + 1, C)
                Zjj[i, j] = (B[i, j] - Zjj[np.ix_(i, i)] @ Ljj[i, j]) / Ljj[j, j]
                Zjj[j, i] = Zjj[i, j]
                Zjj[j, j] = (1.0 / Ljj[j, j] + B[j, j] - Zjj[i, j] @ Ljj[i, j]) / Ljj[j, j]
            Z[k] = np.vstack((Zjj, Ztj))
    return Z


def in_pattern(pl, own, p, q):
    lo, hi = min(p, q), max(p, q)
    k = own[lo]
    return hi < pl["first"][k + 1] or hi in set(struct(pl, k).tolist())


def path_solve(pl, panels, own, p):
    """w = L^-1 E_p on the supernodes from p's to its root, as k_joint_sel_parked: {supernode: rows}."""
    path, k = [], own[p]
    while k >= 0:
        path.append(k)
        k = pl["parent"][k]
    w = {k: np.zeros((6 * (pl["first"][k + 1] - pl["first"][k]), 6)) for k in path}
    w[path[0]][6 * (p - pl["first"][path[0]]):6 * (p - pl["first"][path[0]]) + 6] = np.eye(6)
    for k in path:
        C = w[k].shape[0]
        P = panels[k]
        for j in range(C):
            w[k][j] /= P[j, j]
            w[k][j + 1:] -= np.outer(P[j + 1:C, j], w[k][j])
        upd = P[C:] @ w[k]
        for i, q in enumerate(struct(pl, k)):
            t = own[q]
            r = 6 * (q - pl["first"][t])
            w[t][r:r + 6] -= upd[6 * i:6 * i + 6]
    return w


def relabelled_block():
    F, pairs = graph("grid_2d")
    relabel = np.random.default_rng(9).permutation(F)
    return F, [(int(relabel[a]), int(relabel[b])) for a, b in pairs]


def components():
    F1, p1 = graph("strip_128")
    F2, p2 = graph("grid_2d")
    return F1 + F2 + 40, p1 + [(F1 + a, F1 + b) for a, b in p2] + \
        [(F1 + F2 + i, F1 + F2 + j) for i in range(40) for j in range(i + 1, 40)]


PATTERNS = {"strip_128": lambda: graph("strip_128"), "grid_2d": lambda: graph("grid_2d"),
            "star": lambda: graph("star"), "complete_40": lambda: graph("complete_40"),
            "components": components, "relabelled_grid": relabelled_block}


@pytest.mark.parametrize("name", list(PATTERNS))
def test_selected_inverse_matches_the_inverse_on_the_pattern(lib, name):  # noqa: F811
    F, pairs = PATTERNS[name]()
    pl = make_plan(lib, F, pairs)
    N = spd_matrix(F, pairs, seed=4)
    perm = pl["perm"]
    Ninv = np.linalg.inv(N[np.ix_(expand(perm), expand(perm))])
    panels = factor_panels(pl, N)
    Z = selected_inverse(pl, panels)
    worst, n = 0.0, 0
    for k in range(pl["n_super"]):
        cols = np.arange(pl["first"][k], pl["first"][k + 1])
        rows = np.concatenate((cols, struct(pl, k)))
        ref = Ninv[np.ix_(expand(rows), expand(cols))]
        worst = max(worst, np.abs(Z[k] - ref).max() / np.abs(Ninv).max())
        n += rows.size * cols.size
        assert np.array_equal(Z[k][:6 * cols.size], Z[k][:6 * cols.size].T)
    print(f"{name}: F={F}, {pl['n_super']} supernodes, {n} blocks, max error {worst:.1e}")
    assert worst < 1e-12


@pytest.mark.parametrize("name", ["strip_128", "grid_2d", "components"])
def test_a_pair_outside_the_pattern_from_the_forward_solves(lib, name):  # noqa: F811
    F, pairs = PATTERNS[name]()
    pl = make_plan(lib, F, pairs)
    own = owner_of(pl)
    N = spd_matrix(F, pairs, seed=6)
    perm = pl["perm"]
    Ninv = np.linalg.inv(N[np.ix_(expand(perm), expand(perm))])
    panels = factor_panels(pl, N)
    rng = np.random.default_rng(1)
    outside = []
    while len(outside) < 8:
        p, q = (int(x) for x in rng.integers(0, F, 2))
        if p != q and not in_pattern(pl, own, p, q):
            outside.append((p, q))
    for p, q in outside:
        wp, wq = path_solve(pl, panels, own, p), path_solve(pl, panels, own, q)
        G = sum((wp[k].T @ wq[k] for k in wp if k in wq), np.zeros((6, 6)))
        ref = Ninv[6 * p:6 * p + 6, 6 * q:6 * q + 6]
        assert np.abs(G - ref).max() <= 1e-12 * np.abs(Ninv).max(), (p, q)
        if name == "components" and (p < 128) != (q < 128):  # different trees: exactly zero
            assert not set(wp) & set(wq) and not G.any()


def test_the_parked_pairs_of_the_gpu_test_lie_outside_the_pattern(lib):  # noqa: F811
    """test_gpu_joint_sparse_cov's parked pairs: the 127-cloud strip's edges give the plan; free
    clouds 1 -> 0, 100 -> 99, ... (cloud 0 is fixed).  At least one of its three parked pairs lies
    outside the pattern, so the forward-solve path is exercised on the device."""
    F, pairs = graph("strip_128")
    pl = make_plan(lib, F, pairs)
    own = owner_of(pl)
    pos = np.argsort(pl["perm"])
    outside = [not in_pattern(pl, own, pos[a - 1], pos[b - 1]) for a, b in ((1, 100), (5, 60), (30, 120))]
    assert any(outside), outside


# --------------------------------------------------------------------------- bindings
def _clouds(n=3, m=200):
    rng = np.random.default_rng(0)
    return [rng.normal(0, 1, (m, 3)) for _ in range(n)]


@pytest.mark.parametrize("value", [1, 0, "yes", "Selected", None, 1.0, np.array([True])])
def test_covariances_takes_a_bool_or_selected(value):
    with pytest.raises(TypeError, match="covariances"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], covariances=value)
    with pytest.raises(TypeError, match="covariances"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], covariances=value, solver="sparse")


def test_true_is_still_refused_under_the_sparse_solver_and_names_selected():
    with pytest.raises(ValueError, match="covariances=True needs solver='dense'.*'selected'"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], solver="sparse", covariances=True)


@pytest.mark.parametrize("solver", ["dense", "sparse"])
def test_selected_passes_the_argument_checks_under_both_solvers(solver):
    """'selected' gets past the checks of covariances= to the run's own: a bad run argument is
    then the TypeError that simpleicp_joint raises for it, whichever solver."""
    with pytest.raises(TypeError, match="unsupported"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], solver=solver, covariances="selected", mov_neighbors=10)


def test_header_and_ctypes_declare_the_entry_point():
    h = (REPO / "include" / "sicp_b200.h").read_text()
    m = re.search(r"int32_t sicp_get_joint_selected_covariances\(([^)]*)\);", h)
    assert m, "declaration missing"
    args = [a.strip() for a in re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")]
    assert args == ["sicp_ctx* ctx", "int32_t n_clouds", "double* cloud_cov", "int32_t n_edges", "double* edge_cov",
                    "double* s0"]
    doc = h[h.index("the same covariances under either solver"):m.start()]
    for word in ("Takahashi", "pattern", "parked", "w_a^T w_b", "J'_c", "o_c^0", "SICP_ERR_STATE",
                 "sicp_get_joint_covariances keeps refusing"):
        assert word in doc, word
    assert "sicp_get_joint_selected_covariances" in _capi.SYMBOLS
    lib = _capi.load_library(build_if_missing=False)
    assert lib.sicp_get_joint_selected_covariances.argtypes == lib.sicp_get_joint_covariances.argtypes
    assert lib.sicp_get_joint_selected_covariances.restype == lib.sicp_get_joint_covariances.restype
    assert _capi.ABI_VERSION == 5 and lib.sicp_abi_version() == 5
