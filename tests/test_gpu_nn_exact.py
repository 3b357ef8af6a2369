"""Exact nearest neighbours of every search path, on adversarial and georeferenced geometry.

The correspondence search (nn.cu) and the k-NN of the normals (normals.cu) promise the exact
nearest neighbour(s), ties broken towards the lower original index, whichever engine, lane
count, warm start, ring limit or cell size runs.  Their exactness rests on slack arguments (row
bounds in float32 cell units, the ring guard shrunk by 1e-9 h, the ring-1 prunes with a relative
1e-12 on the best distance, the brute-force engine's float32 filter margin, the hand-off of
unresolved queries to the brute-force engine).  This file checks the promise against an exact
host reference.

Dyadic design.  Every coordinate is O + k * 2^-10 with an integer k, and within one case every
coordinate difference stays below 2^25 units.  Then each difference, each square and each sum of
three squares is exact in float64, with or without the FMA contraction nvcc applies to
dx*dx + dy*dy + dz*dz, so the device's squared distance is U^2 times an integer and the nearest
neighbour is the lexicographic minimum of (integer d^2, original index).  The host decides that
in integer arithmetic (cKDTree only shortlists candidates).  The transforms are signed axis
permutations with dyadic translations, so rigid_apply (common.cuh) is exact too; the host
asserts both facts before any device result is compared.

Origins: 0 and the UTM-scale O_UTM below, where coordinate ulps are 2^-30 m and a cell face
computed as fma(c, h, o) can be rounded by far more than the guard's 1e-9 h slack.  The
face-sliver tests put the true neighbour on the last representable coordinate before such a
face; see test_face_slivers for why the slack still holds there.
"""
from __future__ import annotations

import functools
import itertools
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import simpleicp_oracle as O

from simpleicp_b200 import _capi
from test_grid_plan import first_plan

U = 2.0 ** -10                                  # lattice unit (m)
KMAX = 2 ** 25                                  # bound on every coordinate difference, in units
O_UTM = (612345.25, 5432109.87, 310.5)
ORIGINS = {"origin": (0.0, 0.0, 0.0), "utm": O_UTM}
OCCUPANCIES = (0.25, 3.0, 64.0)

# A covering set of the search options (not the full product): every value of every option
# appears, the hand-off configurations (grid_max_rings 1 without the sphere scan) on both kernels.
PATHS = [
    dict(nn_engine=_capi.NN_AUTO),
    dict(nn_engine=_capi.NN_GRID),
    dict(nn_engine=_capi.NN_BRUTE),
    dict(nn_engine=_capi.NN_AUTO, match_group=1),
    dict(nn_engine=_capi.NN_AUTO, match_group=1, grid_max_rings=1),
    dict(nn_engine=_capi.NN_AUTO, match_group=2, sphere_scan=0),
    dict(nn_engine=_capi.NN_GRID, match_group=4, warm_start=0),
    dict(nn_engine=_capi.NN_AUTO, match_group=8, grid_max_rings=1),
    dict(nn_engine=_capi.NN_AUTO, match_group=16, sphere_scan=0, grid_max_rings=1),
    dict(nn_engine=_capi.NN_GRID, match_group=16, sphere_scan=1, warm_start=1),
]
HANDOFF = [p for p in PATHS if p.get("grid_max_rings") == 1 and p["nn_engine"] == _capi.NN_AUTO
           and (p.get("match_group") == 1 or p.get("sphere_scan") == 0)]
DEFAULTS = dict(nn_engine=_capi.NN_AUTO, match_group=0, sphere_scan=1, warm_start=1, grid_max_rings=8)


# ------------------------------------------------------------------------------ host reference
def to_xyz(k, origin):
    """Coordinates O + k U (exact: k U is dyadic and the sum lies on O's ulp grid)."""
    X = np.asarray(origin, dtype=np.float64)[None, :] + np.asarray(k, dtype=np.int64) * U
    assert np.array_equal(np.rint((X - np.asarray(origin)) / U).astype(np.int64), k), "not exact"
    return X


def exact_knn(P, Q, k):
    """The k first (integer d^2, index) pairs of every query: the lexicographic order the device
    promises.  P, Q are integer lattice coordinates (exact as float64 in the tree)."""
    P = np.asarray(P, dtype=np.int64)
    Q = np.asarray(Q, dtype=np.int64)
    tree = cKDTree(P.astype(np.float64))
    dk, _ = tree.query(Q.astype(np.float64), k=k)
    dk = np.asarray(dk).reshape(len(Q), -1)[:, -1]
    cand = tree.query_ball_point(Q.astype(np.float64), r=dk * (1 + 1e-9) + 1e-6)
    idx = np.empty((len(Q), k), dtype=np.int64)
    d2 = np.empty((len(Q), k), dtype=np.int64)
    for i, c in enumerate(cand):
        c = np.asarray(c, dtype=np.int64)
        dd = ((P[c] - Q[i]) ** 2).sum(axis=1)
        o = np.lexsort((c, dd))[:k]
        assert len(o) == k
        idx[i], d2[i] = c[o], dd[o]
    assert d2.max() < 2 ** 52
    return idx, d2


def n_ties(P, Q):
    """Queries whose nearest distance is shared by two or more points."""
    idx, d2 = exact_knn(P, Q, 2)
    return int((d2[:, 0] == d2[:, 1]).sum())


def perm_H(R, s, origin):
    """H = [R | t] with R a signed permutation and t = O - R O + s U: maps O + k U to
    O + (R k + s) U."""
    H = np.eye(4)
    H[:3, :3] = R
    H[:3, 3] = (np.asarray(origin) - R @ np.asarray(origin)) + np.asarray(s) * U
    return H


def rigid_apply(H, X):
    """common.cuh: rigid_apply, term by term as the device evaluates it (with R in {0, +-1} the
    products are exact, so fma and plain evaluation agree)."""
    R, t = H[:3, :3], H[:3, 3]
    return np.column_stack([((R[i, 0] * X[:, 0] + R[i, 1] * X[:, 1]) + R[i, 2] * X[:, 2]) + t[i]
                            for i in range(3)])


def inverse(H):
    R = H[:3, :3].T
    Hi = np.eye(4)
    Hi[:3, :3] = R
    Hi[:3, 3] = -(R[:, 0] * H[0, 3] + R[:, 1] * H[1, 3] + R[:, 2] * H[2, 3])
    return Hi


# ------------------------------------------------------------------------------ case catalogue
@dataclass
class Case:
    name: str
    mk: np.ndarray                 # movable cloud, lattice units
    qk: np.ndarray                 # queries in the MOVABLE frame, lattice units
    R: np.ndarray = field(default_factory=lambda: np.eye(3, dtype=np.int64))
    far: bool = False              # some queries need more rings than grid_max_rings = 1

    S0 = np.array([3, -5, 7])

    def H(self, origin, shift=(0, 0, 0)):
        """H and the fixed points p (lattice units, the same for every shift) with H^-1 p = the
        queries moved by -shift."""
        H = perm_H(self.R, self.S0 + self.R @ np.asarray(shift), origin)
        return H, self.qk @ self.R.T + self.S0


def _rng(name):
    return np.random.default_rng(sum(map(ord, name)) * 7919)


def sheet(n=6000, side=2 ** 14):
    """Scan-like sheet: jittered, tilted, ~3 points per cell at the default occupancy."""
    rng = _rng("sheet")
    xy = rng.integers(0, side, size=(n, 2))
    z = (xy[:, 0] // 8 + xy[:, 1] // 16) + rng.integers(-20, 21, n)
    mk = np.column_stack((xy, z))
    qxy = rng.integers(-200, side + 200, size=(3000, 2))
    qk = np.column_stack((qxy, qxy[:, 0] // 8 + qxy[:, 1] // 16 + rng.integers(-600, 601, 3000)))
    return Case("sheet", mk, qk)


def ties(L=64, dims=(20, 16, 10)):
    """Lattice queries equidistant from 2, 4, 6 or 8 points, plus duplicates.  Indices run
    against the scan order (the last point of a row has the lowest index) and every duplicate's
    copy sits 2048+ indices away, so tie partners straddle lanes, rows, brute-force tiles and
    chunks."""
    g = np.stack(np.meshgrid(*[np.arange(d) for d in dims], indexing="ij"), -1).reshape(-1, 3) * L
    g = g[np.lexsort((g[:, 0], g[:, 1], g[:, 2]))][::-1]     # descending scan order
    rng = _rng("ties")
    hole = g[rng.choice(len(g), 40, replace=False)]
    keep = ~(g[:, None, :] == hole[None, :, :]).all(-1).any(-1)
    base = g[keep]
    dup_src = base[rng.choice(len(base), 300, replace=False)]
    mk = np.concatenate((dup_src, base, dup_src[::-1]))   # copies far apart in index
    h = L // 2
    c = base[rng.choice(len(base), 400, replace=False)]
    qk = np.concatenate((c + [h, 0, 0], c + [h, h, 0], c + [0, h, h], c + [h, h, h],   # 2, 4, 4, 8
                         hole,                                                         # 6
                         dup_src[:200] + [1, 2, 0], dup_src[:100]))                    # duplicates
    R = np.array([[0, 1, 0], [-1, 0, 0], [0, 0, 1]], dtype=np.int64)
    return Case("ties", mk, qk, R=R)


def far_queries():
    """A sheet with clusters separated by empty cells; queries behind every face of the box, on
    an axis 50 and 150 cells from the sheet (the axis probes stop after 96 steps), diagonal to it
    (the probes miss), and behind the clusters."""
    rng = _rng("far")
    n = 4000
    xy = rng.integers(0, 2 ** 13, size=(n, 2))
    mk = np.column_stack((xy, rng.integers(0, 8, n)))
    clusters = np.concatenate([rng.integers(0, 40, size=(60, 3)) + c for c in
                               ([-3000, 4000, 5000], [12000, 12000, -4000])])
    mk = np.concatenate((mk, clusters))
    h = int(np.sqrt(3 * 2 ** 26 / n))          # ~ the default cell size in units
    mid = 2 ** 12
    q = [[mid, mid, 50 * h], [mid, mid, 150 * h], [mid, mid, -50 * h], [mid, mid, -150 * h],
         [-40 * h, mid, 3], [2 ** 13 + 40 * h, mid, 3], [mid, -60 * h, 3], [mid, 2 ** 13 + 60 * h, 3],
         [-30 * h, -30 * h, 30 * h], [2 ** 13 + 30 * h, 2 ** 13 + 30 * h, -30 * h],
         [-3000 - 20 * h, 4000, 5000], [12000 + 20 * h, 12000 + 20 * h, -4000 - 20 * h]]
    q = np.array(q, dtype=np.int64)
    qk = np.concatenate([q + rng.integers(-30, 31, size=q.shape) for _ in range(20)])
    return Case("far", mk, qk, far=True)


def degenerate(kind):
    rng = _rng("deg" + kind)
    if kind == "plane":                       # nz = 1
        xy = rng.integers(0, 5000, size=(3000, 2))
        mk = np.column_stack((xy, np.zeros(3000, dtype=np.int64)))
    elif kind == "line":
        mk = np.column_stack((rng.integers(0, 200000, 2000), np.zeros((2000, 2), dtype=np.int64)))
    elif kind == "one_cell":
        mk = rng.integers(0, 4, size=(500, 3))
    elif kind == "one_point":
        mk = np.array([[5, -3, 2]])
    elif kind == "two_points":
        mk = np.array([[0, 0, 0], [64, 0, 0]])
    else:                                     # movable sizes around the 2048-point tile
        n = int(kind.split("_")[1])
        mk = rng.integers(0, 3000, size=(n, 3))
    lo, hi = mk.min(0), mk.max(0)
    qk = rng.integers(lo - 100, hi + 101, size=(600, 3))
    if kind == "two_points":
        qk = np.concatenate((qk, [[32, 0, 0], [32, 5, -5]]))   # equidistant
    return Case(kind, mk, qk)


def cube(n_side=100):
    """A volumetric cube of n_side^3 points: its first cell size assumes a surface, so the 2^25
    cell cap forces the h *= 1.26 growth of grid.cu."""
    g = np.stack(np.meshgrid(*[np.arange(n_side)] * 3, indexing="ij"), -1).reshape(-1, 3) * 8
    rng = _rng("cube")
    qk = rng.integers(-40, 8 * n_side + 40, size=(3000, 3))
    qk[:500] = g[rng.choice(len(g), 500, replace=False)] + 4          # 8-way ties
    return Case("cube", g, qk)


F32_BASE = 3008   # a multiple of 64: no 64-point block of pairs straddles a 2048-point tile


def f32_near_ties():
    """Near-ties for the brute-force engine's float32 filter: each query is 2^16..2^17 units
    (64-128 m) above its own pair of candidates, whose squared distances differ by exactly one
    unit^2.  The pairs sit in a row 2048 units
    apart beside and above a compact cloud that lies behind them, so the pair holds the first
    and second exact neighbours of its query, while the centred float32 copy orders the pair by
    rounding of their centred coordinates (test_f32_filter_cases_reverse_order).  Each pair's farther point comes 32 indices
    before its nearer one in the same tile: the same lane of k_bf_nn meets the farther point
    first, so where float32 reverses the pair only the filter margin sends the nearer one to
    the float64 re-evaluation."""
    rng = _rng("f32")
    base = np.column_stack((rng.integers(-2000, 2000, (F32_BASE, 2)), rng.integers(-2000, 1, F32_BASE)))
    # a few points 23 km away move the centre of the float32 copy ~12 km from the pairs, where a
    # float32 ulp is one unit: the pairs' centred coordinates round, each pair differently
    base[:8] = [-24_000_001, 0, -1000] + np.arange(8)[:, None] * [0, 0, -3]
    qk, near, far = [], [], []
    for i in range(169):
        # m and m + e, e = (-E, 0, 2), E odd: d^2(m + e) - d^2(m) = 2 E d_x - 4 d_z + E^2 + 4 =
        # delta = +-1.  The pair differs along the large components of d and its x coordinates
        # differ by an odd number of units, so float32 rounds the two apart.
        while True:
            dz, E, delta = int(rng.integers(2 ** 16, 2 ** 17)), 2 * int(rng.integers(0, 8)) + 1, int(rng.choice([-1, 1]))
            if (4 * dz - E * E - 4 + delta) % (2 * E) == 0:
                break
        dx = (4 * dz - E * E - 4 + delta) // (2 * E)
        m = np.array([2100, 2048 * (i - 84), 64])   # a row along y, beside and above the cloud
        m2 = m + [-E, 0, 2]
        a, b = (m, m2) if delta == 1 else (m2, m)
        near.append(a)
        far.append(b)
        qk.append(m + [dx, int(rng.integers(-20, 21)), dz])
    n = len(qk)
    pts = np.zeros((2 * ((n + 31) // 32) * 32, 3), dtype=np.int64)
    pts[:] = [-24_000_001, 0, -2000]            # filler behind the pairs
    fi, ni = f32_pair_slots(n)
    pts[fi - F32_BASE], pts[ni - F32_BASE] = far, near
    return Case("f32", np.concatenate((base, pts)), np.array(qk))


def f32_pair_slots(n):
    """Indices of the farther and the nearer point of each pair: blocks of 64, farther first."""
    i = np.arange(n)
    fi = F32_BASE + 64 * (i // 32) + i % 32
    return fi, fi + 32


def catalogue():
    cases = [sheet(), ties(), far_queries(), cube(), f32_near_ties()]
    cases += [degenerate(k) for k in ("plane", "line", "one_cell", "one_point", "two_points",
                                      "size_40", "size_2047", "size_2048", "size_2049")]
    return cases


@functools.lru_cache(maxsize=None)
def cases():
    return {c.name: c for c in catalogue()}


@functools.lru_cache(maxsize=None)
def reference(name, shift=(0, 0, 0)):
    c = cases()[name]
    qk = c.qk - np.asarray(shift)
    return exact_knn(c.mk, qk, 1)


# --------------------------------------------------------------------------- host self-checks
@pytest.mark.parametrize("name", [c.name for c in catalogue()])
@pytest.mark.parametrize("where", list(ORIGINS))
def test_case_design_is_exact(name, where):
    """Every d^2 fits the exactness bound, the transforms are exact, and H^-1 p gives back the
    designed queries bit for bit (rigid_apply as the device evaluates it)."""
    c = cases()[name]
    origin = ORIGINS[where]
    span = np.ptp(np.concatenate((c.mk, c.qk)), axis=0)
    assert span.max() < KMAX and 3 * int(span.max()) ** 2 < 2 ** 52
    for shift in ((0, 0, 0), (1, 0, 0), (0, 0, 40)):
        H, pk = c.H(origin, shift)
        P = to_xyz(pk, origin)
        Q = rigid_apply(inverse(H), P)
        assert np.array_equal(Q, to_xyz(c.qk - np.asarray(shift), origin))
        # the matched point moved by H (point-to-plane distance) is exact too
        M = to_xyz(c.mk, origin)
        s = c.S0 + c.R @ np.asarray(shift)
        assert np.array_equal(rigid_apply(H, M), to_xyz(c.mk @ c.R.T + s, origin))


def test_case_design_has_ties():
    assert n_ties(cases()["ties"].mk, cases()["ties"].qk) >= 1000
    assert n_ties(cases()["cube"].mk, cases()["cube"].qk) >= 500
    assert n_ties(cases()["two_points"].mk, cases()["two_points"].qk) >= 1
    # the duplicates really straddle brute-force tiles (2048 points) and chunks
    mk = cases()["ties"].mk
    _, first = np.unique(mk, axis=0, return_index=True)
    dup = {tuple(v) for v in mk[:300]}
    far_apart = [i for i, v in enumerate(mk[-300:]) if tuple(v) in dup]
    assert len(far_apart) == 300 and len(mk) - 300 > 2048


def test_reference_agrees_with_ckdtree_without_ties():
    for c in catalogue():
        idx, d2 = reference(c.name)
        dd, ii = cKDTree(c.mk.astype(np.float64)).query(c.qk.astype(np.float64), k=1)
        if len(c.mk) >= 2:
            _, d2b = exact_knn(c.mk, c.qk, 2)
            unique = d2b[:, 0] != d2b[:, 1]
        else:
            unique = np.ones(len(c.qk), dtype=bool)
        assert np.array_equal(ii[unique], idx[unique, 0]), c.name
        assert np.array_equal(dd, np.sqrt(d2[:, 0].astype(np.float64))), c.name


def f32_d2(Mf, a):
    """k_bf_nn's filter distance: float32 differences, fmaf(dz, dz, fmaf(dy, dy, dx * dx))."""
    f = np.float32
    dx, dy, dz = (f(Mf[:, i] - f(a[i])) for i in range(3))
    t = (dx.astype(np.float64) * dx).astype(f)
    t = (dy.astype(np.float64) * dy + t).astype(f)
    return (dz.astype(np.float64) * dz + t).astype(f)


def test_f32_filter_cases_reverse_order():
    """In f32_near_ties the designed pair holds the exact first and second neighbours of every
    query, one unit^2 apart, and in the centred float32 copy the filter sees the pair in reversed
    order for a good share of the queries.  The centre here is the cloud's box centre;
    the device centres on its grid's box, which rounds the same way in distribution."""
    c = cases()["f32"]
    n_pairs = len(c.qk)
    far, near = f32_pair_slots(n_pairs)
    idx, d2 = exact_knn(c.mk, c.qk, 2)
    assert np.array_equal(idx, np.column_stack((near, far)))
    assert (d2[:, 1] - d2[:, 0] == 1).all()
    assert ((far // 2048) == (near // 2048)).all()
    for origin in ORIGINS.values():
        M = to_xyz(c.mk, origin)
        ctr = 0.5 * (M.min(0) + M.max(0))
        Mf = (M - ctr).astype(np.float32)
        Q = to_xyz(c.qk, origin)
        reversed_ = 0
        for i in range(n_pairs):
            d32 = f32_d2(Mf[idx[i]], (Q[i] - ctr).astype(np.float32))
            reversed_ += bool(d32[0] > d32[1])
        assert reversed_ >= n_pairs // 5, reversed_


# ------------------------------------------------------------------------------ device helpers
def set_paths(e, opts):
    for k, v in {**DEFAULTS, **opts}.items():
        e.set_option(k, v)


@functools.lru_cache(maxsize=None)
def _engine_cache():
    return {}


def engine_for(name, where, occ):
    """One engine per (case, origin, occupancy): the grid is built by set_clouds."""
    key = (name, where, occ)
    cache = _engine_cache()
    if key not in cache:
        c = cases()[name]
        origin = ORIGINS[where]
        e = _capi.Engine()
        e.set_option("grid_target_occupancy", occ)
        _, pk = c.H(origin)
        e.set_clouds(to_xyz(pk, origin), to_xyz(c.mk, origin))
        e.set_selected(None)
        K = len(c.qk)
        z = np.zeros(K, dtype=np.float32)
        e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
        cache[key] = e
    return cache[key]


def check_match(e, c, origin, shift, what):
    """match(H) against the exact reference; the point-to-plane distance through the normal
    (0, 0, 1) is one coordinate difference and must equal the host's with ==."""
    H, pk = c.H(origin, shift)
    idx, d = e.match(H)
    ref, _ = reference(c.name, tuple(shift))
    bad = np.flatnonzero(idx != ref[:, 0])
    assert bad.size == 0, f"{what}: {bad.size} of {len(idx)} queries differ, first {bad[:5]}: " \
                          f"{idx[bad[:5]]} vs {ref[bad[:5], 0]}"
    M = to_xyz(c.mk, origin)
    Mt = rigid_apply(H, M)
    d_host = Mt[ref[:, 0], 2] - to_xyz(pk, origin)[:, 2]
    assert np.array_equal(d, d_host), what
    return len(idx)


RUN_COUNTS: dict = {}


@pytest.mark.gpu
@pytest.mark.parametrize("occ", OCCUPANCIES)
@pytest.mark.parametrize("where", list(ORIGINS))
@pytest.mark.parametrize("name", [c.name for c in catalogue()])
def test_match_exact_on_every_path(gpu, name, where, occ):
    """Every path of the covering set returns the exact reference indices.  Each configuration
    runs three consecutive matches with the same K (a large move, then back, then a one-unit move)
    so the warm start sees both a poor bound (ring 1 first) and a good one (sphere scan)."""
    c = cases()[name]
    origin = ORIGINS[where]
    e = engine_for(name, where, occ)
    moves = [(0, 0, 2000), (0, 0, 0), (1, 0, 0)]
    for opts in PATHS:
        set_paths(e, opts)
        for shift in moves:
            n = check_match(e, c, origin, shift, f"{name}@{where} occ {occ} {opts} shift {shift}")
            RUN_COUNTS[str(opts)] = RUN_COUNTS.get(str(opts), 0) + n


@pytest.mark.gpu
@pytest.mark.parametrize("where", list(ORIGINS))
@pytest.mark.parametrize("name", ["far", "sheet", "ties"])
def test_bruteforce_handoff_runs_and_is_exact(gpu, name, where):
    """With grid_max_rings = 1 and no sphere scan the far queries are handed to the brute-force
    engine: the iteration record counts them (n_bruteforce > 0) and match() returns the exact
    neighbours for them."""
    c = cases()[name]
    origin = ORIGINS[where]
    e = engine_for(name, where, 3.0)
    lsq = e.lsq_params(np.zeros(6), np.zeros(6), [np.inf] * 5 + [0.0], 1.0)
    params = e.run_params(0.0, 1.0, 1, lsq)
    for opts in HANDOFF:
        set_paths(e, opts)
        H, _ = c.H(origin)
        check_match(e, c, origin, (0, 0, 0), f"{name}@{where} {opts}")
        if np.array_equal(c.R, np.eye(3)):
            # iterate moves the queries by the rbp parameters: zero angles are exact
            rec = e.iterate(params, x_in=list(np.zeros(3)) + list(H[:3, 3]), want_record=True)
            print(f"{name}@{where} {opts}: n_bruteforce = {rec.n_bruteforce}")
            if c.far:
                assert rec.n_bruteforce > 0


# --------------------------------------------------------------------------- face slivers
def cell_of(v, o, h):
    """cell_coord (common.cuh) without the clamp: floor(fl(v - o) * fl(1 / h))."""
    return np.floor((np.float64(v) - o) * (1.0 / h))


def computed_faces(c, o, h):
    """fl(o + c h) as an fma (one rounding) and unfused (two roundings)."""
    return float(Fraction(o) + c * Fraction(h)), float(o + float(c * Fraction(h)))


def last_below_face(c, o, h):
    """The largest double that cell_coord puts below face c."""
    v = computed_faces(c, o, h)[0]
    while cell_of(v, o, h) >= c:
        v = float(np.nextafter(v, -np.inf))
    while cell_of(np.nextafter(v, np.inf), o, h) < c:
        v = float(np.nextafter(v, np.inf))
    return v


SLIVER_GAP = 0.25e-9   # the competitor is farther than the true neighbour by at most this x h

# The ring-1 prunes of the cooperative match carry a relative slack of 1e-12 on `best`.
#   * Own-row side cells (nn.cu: `bx * bx > best * (1 + 1e-12)`): the slack is not needed.  Every
#     double in the side cell is at least bx from the query along x (see slivers() for why no
#     point lies between the computed and the true face), so |dx| >= bx exactly, and every
#     operation of the point's d^2 (an fma chain that adds dy^2, dz^2 >= 0 to dx^2) is monotone:
#     computed d^2 >= fl(dx^2) >= fl(bx^2).  A pruned cell therefore holds nothing at or below
#     best, ties included.  Dropping the slack leaves the search exact, and the tests agree.
#   * Neighbour rows (`lim = best * (1 + 1e-12)`, compared with lb = by^2 + bz^2): here the
#     slack is needed.  lb and a point's d^2 are sums of different terms in a different order,
#     so for a point exactly on both row faces (dy = by, dz = bz, dx = 0) they can round one ulp
#     apart, and a tie partner or a point within that ulp in the own row would then hide it.
#     The dyadic cases cannot produce that (every sum is exact) and the slivers do not put a
#     point on two faces at once, so no test here fails without this slack.  A case for it needs
#     the contraction nvcc chose for the two sums and an own-row competitor whose d^2 matches to
#     the last bit.


def slivers(o, h, axis, row, faces):
    """Query q, true neighbour p and competitor c for every face in `faces` along `axis`.
    p is the last double below the face; q lies 0.25 h above the face (p is in a side cell of
    ring 1: own-row cells for x faces, neighbour rows for y faces) or 1.25 h above it (p is one
    cell beyond ring 1: the guard decides).  c is p mirrored through q (exact: all three lie on
    one binade's ulp grid) and lifted in z by eps, where the z ulp is 2^-44 m: it is strictly
    farther than p, by less than SLIVER_GAP * h, a quarter of the guard's 1e-9 h slack, inside
    the block ring 1 explores.  `row` gives the other two coordinates."""
    Q, P, C = [], [], []
    for j, cf in enumerate(faces):
        v = last_below_face(cf, o[axis], h)
        F = computed_faces(cf, o[axis], h)[0]
        # why the 1e-9 h slack holds although |F - (o + c h)| can exceed it: every double below
        # the face is <= F, so no point can sit between the computed and the true face.  For a
        # face rounded away from the query F itself is the last double below the face.
        assert v == F
        qa = F + (0.25 if j % 2 == 0 else 1.25) * h
        dist = qa - v
        ca = qa + dist
        assert ca - qa == dist and qa - v == dist
        eps = float(np.sqrt(2.0 * dist * 0.5 * SLIVER_GAP * h))
        zc = row[2]
        dz = (zc + eps) - zc
        # d(c) - d(p) ~ dz^2 / (2 dist): positive after rounding (dz^2 >> ulp(dist^2)) and small
        assert dz * dz > 16 * np.spacing(dist * dist) and dz * dz / (2 * dist) <= SLIVER_GAP * h
        for a, z, lst in ((qa, zc, Q), (v, zc, P), (ca, zc + eps, C)):
            x = np.array(row, dtype=np.float64)
            x[axis] = a
            x[2] = z
            lst.append(x)
    return np.array(Q), np.array(P), np.array(C)


def faces_rounded_away(o_a, h, lo, hi, step):
    """Faces c in [lo, hi) whose computed value lies below the true one (a bound measured from a
    query above the face comes out too large), at least `step` apart.  Only faces where the
    fused and the unfused evaluation of o + c h give the same double are used, so the test does
    not depend on whether nvcc contracts g.ox + x0 * g.h into an fma."""
    out, c = [], lo
    while c < hi:
        F, F2 = computed_faces(c, o_a, h)
        if F == F2 and Fraction(F) < Fraction(o_a) + c * Fraction(h):
            out.append(c)
            c += step
        else:
            c += 1
    return out


def sliver_cloud(n_base, with_queries):
    """A dense sheet (~3 points per 4 cm cell, 2 m x 4 m at the UTM origin) and, ten cells above
    it, 8 slivers across y faces (neighbour rows of ring 1, or the guard) and 4 across x faces
    (own-row side cells, or the guard).  The grid depends on the box and the point count only,
    and the slivers stay inside the sheet's x, y extent (z does not enter the cell size), so the
    layout can be planned before the cloud exists.  Returns the cloud, the queries, the plan."""
    rng = np.random.default_rng(5)
    base = to_xyz(np.column_stack((rng.integers(0, 2048, n_base), rng.integers(0, 4096, n_base),
                                   rng.integers(0, 5, n_base))), O_UTM)
    nq = 12
    n = n_base + (3 if with_queries else 2) * nq
    o = base.min(0)
    _, h, _, _ = first_plan(np.concatenate((base, np.tile(o, (n - n_base, 1)))))
    dims = tuple(int(np.floor((base[:, a].max() - o[a]) / h) + 1) for a in range(2))
    zc = o[2] + 10.5 * h
    xmid = o[0] + (dims[0] // 2 + 0.5) * h
    fy = faces_rounded_away(o[1], h, 4, dims[1] - 24, 7)[:8]
    Qy, Py, Cy = slivers(o, h, 1, (xmid, 0.0, zc), fy)
    fx = faces_rounded_away(o[0], h, 6, dims[0] - 6, 7)[:4]
    Qx, Px, Cx = slivers(o, h, 0, (0.0, o[1] + (dims[1] - 10 + 0.5) * h, zc), fx)
    assert len(fy) == 8 and len(fx) == 4
    Q, P, C = np.concatenate((Qy, Qx)), np.concatenate((Py, Px)), np.concatenate((Cy, Cx))
    X = np.concatenate(((Q,) if with_queries else ()) + (P, C, base))
    plan = first_plan(X)[:3]  # the first attempt's plan, kept: its occupancy is in the band
    assert plan[1] == h and np.array_equal(plan[0], o), "the slivers changed the planned grid"
    return X, Q, plan


@pytest.mark.gpu
@pytest.mark.parametrize("side", ["mov", "fix"])
def test_face_slivers(gpu, side):
    """UTM-scale cell faces (ulp 2^-30 m in y, 2^-33 m in x) with 4 cm cells, so that rounding a
    face exceeds the guard's 1e-9 h slack; the true neighbour on the last double below a face
    rounded away from the query, a competitor strictly farther inside the explored block but by
    less than the slack (so a guard that added the slack instead of subtracting it would stop
    with the competitor: match_group 1 and the paths without the sphere scan, every k-NN body).  The
    match paths (side "mov") and every k-NN body (side "fix", k = 2: the query itself, then the
    sliver neighbour) must find the sliver neighbour.

    Result: exact at the parent commit; no library change was needed.  The slack holds for a
    reason other than its size: the face is F = fl(T) with T = o + c h, and cell_coord's face
    differs from T by a few ulps of (c h) only, far below half an ulp of the coordinates.  When
    F < T no double lies between F and the face, so every point of the cells below it has v <= F
    and lies at least q - F from the query, which is exactly the computed bound (the host asserts
    v <= F for every face used).  The 1e-9 h slack only has to cover the relative rounding of the
    subtraction and the squares."""
    n_base = 15000
    with _capi.Engine() as e:
        e.set_option("keep_knn", 1)
        if side == "mov":
            Xm, Q, plan = sliver_cloud(n_base, with_queries=False)
            nq = len(Q)
            e.set_clouds(Q, Xm)
            got = e.grid_params("mov")
            e.set_selected(None)
            z = np.zeros(nq, dtype=np.float32)
            e.set_normals(z, z, np.ones(nq, dtype=np.float32), np.full(nq, 0.9, dtype=np.float32))
            for opts in PATHS:
                set_paths(e, opts)
                for _ in range(2):   # the second one warm-started
                    idx, _d = e.match(np.eye(4))
                    assert np.array_equal(idx, np.arange(nq)), (opts, np.flatnonzero(idx != np.arange(nq)))
        else:
            Xf, Q, plan = sliver_cloud(n_base, with_queries=True)
            nq = len(Q)
            e.set_clouds(Xf, Xf[nq:])
            e.set_selected(np.arange(nq))
            for coop in (-1, 0, 1, 2):
                e.set_option("knn_coop", coop)
                e.estimate_normals(2)
                idx, _d2 = e.get_knn(2)
                assert np.array_equal(idx[:, 0], np.arange(nq))
                assert np.array_equal(idx[:, 1], nq + np.arange(nq)), coop
            got = e.grid_params("fix")
        assert np.array_equal(got[0], plan[0]) and got[1] == plan[1] and got[2] == plan[2], (got, plan)
        assert plan[1] < 0.05 and 1e-9 * plan[1] < 2.0 ** -33


# ------------------------------------------------------------------------------ k-NN
KNN_CASES = [("ties", 3), ("ties", 10), ("ties", 16), ("ties", 17), ("ties", 40), ("sheet", 10),
             ("sheet", 16), ("cube", 17), ("cube", 40), ("one_cell", 64), ("two_points", 2),
             ("size_40", 40)]


def pca(pts):
    """The oracle's normal / planarity on a given neighbour set (simpleicp_oracle.estimate_normals)."""
    C = np.cov(pts.T, bias=False)
    w, v = np.linalg.eig(C)
    o = w.argsort()[::-1]
    w, v = w[o], v[:, o]
    return v[:, 2].astype(np.float32), np.float32((w[1] - w[2]) / w[0])


@pytest.mark.gpu
@pytest.mark.parametrize("where", list(ORIGINS))
@pytest.mark.parametrize("name,k", KNN_CASES)
def test_knn_exact(gpu, name, k, where):
    """get_knn equals the exact (d^2, index) order, every knn_coop value; dist2 equals the
    integer d^2 with ==; normals and planarity match the oracle's np.cov / eig on that set."""
    c = cases()[name]
    origin = ORIGINS[where]
    P = to_xyz(c.mk, origin)
    sel = np.unique(np.linspace(0, len(P) - 1, min(len(P), 800)).astype(np.int64))
    k = min(k, len(P))
    ref_idx, ref_d2 = exact_knn(c.mk, c.mk[sel], k)
    with _capi.Engine() as e:
        e.set_option("keep_knn", 1)
        e.set_option("sign_mode", _capi.SIGN_CANONICAL)
        e.set_clouds(P, P)
        e.set_selected(sel)
        for coop in (-1, 0, 1, 2):
            e.set_option("knn_coop", coop)
            nx, ny, nz, pl = e.estimate_normals(k)
            idx, d2 = e.get_knn(k)
            assert np.array_equal(idx, ref_idx), f"coop {coop}: {(idx != ref_idx).any(1).sum()} rows differ"
            assert np.array_equal(d2, ref_d2 * U * U)
            n_gpu = np.column_stack((nx, ny, nz)).astype(np.float64)
            for i in range(0, len(sel), 7):
                n_ref, pl_ref = pca(P[ref_idx[i]])
                if not np.isfinite(pl_ref) or pl_ref <= 0.05:
                    continue
                s = np.sign(np.dot(n_gpu[i], n_ref))
                assert np.abs(s * n_gpu[i] - n_ref).max() < 5e-6
                assert abs(pl[i] - pl_ref) <= 1e-6


# --------------------------------------------------------------------------- overlap filter
@pytest.mark.gpu
@pytest.mark.parametrize("where", list(ORIGINS))
def test_overlap_filter_boundary(gpu, where):
    """A neighbour at exactly max_range is dropped, one at the next representable d^2 inside is
    kept; queries far from everything are decided by the guard alone.  Bit for bit against the
    oracle's select_in_range and against the integer reference."""
    origin = ORIGINS[where]
    rng = np.random.default_rng(11)
    r = 300                                      # max_range = r U: r^2 U^2 is exact
    mk = np.stack(np.meshgrid(*[np.arange(0, 20 * 1024, 1024)] * 2, [0], indexing="ij"), -1).reshape(-1, 3)
    offs = []
    for target in range(r * r - 40, r * r + 41):
        a = rng.integers(0, r + 1)
        b2 = target - a * a
        if b2 < 0:
            continue
        b = int(np.sqrt(b2))
        c2 = b2 - b * b
        cc = int(np.sqrt(c2))
        if cc * cc == c2:
            offs.append([a, b, cc])
    offs += [[r, 0, 0], [0, r, 0], [0, 0, r], [0, 0, r - 1], [r - 1, 1, 0]]
    # the largest d^2 below r^2 that three integer squares reach (r^2 - 1 is 7 mod 8 here)
    inside = max(a * a + b * b + c * c for a in range(r) for b in range(0, 40) for c in range(0, 40)
                 if a * a + b * b + c * c < r * r)
    offs += [[a, b, c] for a in range(r - 2, r) for b in range(40) for c in range(40)
             if a * a + b * b + c * c == inside][:4]
    offs = np.array(offs)
    base = mk[rng.integers(0, len(mk), len(offs))]
    far = np.array([[-40 * 1024, 5000, 0], [5000, 30 * 1024, 9000], [3000, 3000, 60 * 1024]])
    qk = np.concatenate((base + offs * rng.choice([-1, 1], offs.shape), far))
    _, d2 = exact_knn(mk, qk, 1)
    assert (d2[:, 0] == r * r).any() and (d2[:, 0] == inside).any() and (d2[:, 0] > r * r).any()
    keep_ref = d2[:, 0] < r * r
    H0 = perm_H(np.eye(3), (5, -3, 2), origin)      # a dyadic translation
    Xf = to_xyz(qk + [5, -3, 2], origin)
    Xm = to_xyz(mk, origin)
    assert np.array_equal(rigid_apply(H0, Xm), to_xyz(mk + [5, -3, 2], origin))
    sel = np.arange(len(qk))
    oracle = O.select_in_range(Xf, sel, rigid_apply(H0, Xm), r * U)
    assert np.array_equal(sel[keep_ref], oracle)
    with _capi.Engine() as e:
        e.set_clouds(Xf, Xm)
        e.set_selected(None)
        for opts in PATHS:
            set_paths(e, opts)
            keep = e.select_in_range(H0, r * U)
            assert np.array_equal(np.flatnonzero(keep), oracle), opts


# --------------------------------------------------------------------------- whole runs
def _run(e, Xf, Xm, opts, occ):
    import simpleicp_b200 as sb

    e.reset_options()
    e.set_option("grid_target_occupancy", occ)
    set_paths(e, opts)
    r = sb.register(Xf, Xm, engine=e, want_normals=False)
    return (np.array(r.H), r.records, np.array(r.residuals), np.array(r.X_mov_transformed))


def _same_records(ra, rb, what):
    """Every field of every iteration record bit for bit; n_bruteforce counts the queries a path
    handed to the brute-force engine, a property of the path, not of the result."""
    assert len(ra) == len(rb), what
    for it, (a, b) in enumerate(zip(ra, rb)):
        assert a.keys() == b.keys(), what
        for k in a:
            if k == "n_bruteforce":
                continue
            va, vb = np.asarray(a[k]), np.asarray(b[k])
            assert va.dtype == vb.dtype and np.array_equal(va, vb, equal_nan=va.dtype.kind == "f"), \
                f"{what}: iteration {it} {k}: {a[k]} vs {b[k]}"


def _same(a, b, what):
    assert np.array_equal(a[0], b[0]), f"{what}: H"
    _same_records(a[1], b[1], what)
    assert np.array_equal(a[2], b[2]), f"{what}: residuals"
    assert np.array_equal(a[3], b[3]), f"{what}: transformed cloud"


def _utm_c3(n=200_000):
    Xf, Xm, _ = O.c3_pair(n)
    return tuple(np.round(X / U) * U + np.asarray(O_UTM) for X in (Xf, Xm))


@pytest.mark.gpu
@pytest.mark.parametrize("pair", ["dragon", "c3_utm"])
def test_whole_run_independent_of_search_path(gpu, pair):
    """The same neighbours, the same distance formula, exact order statistics: register returns
    bit-identical H, records, residuals and transformed cloud on every search path.

    grid_target_occupancy is the exception for H and the residuals: the solve centres its moments
    on the movable grid's box (make_float4_copy: mov_center), whose far corner o + n h moves with
    the cell size, so another cell size rounds the moment sums differently.  The neighbours and
    the kept sets stay identical there (n_kept of every record), H agrees to rounding."""
    if pair == "dragon":
        from conftest import load_pair

        Xf, Xm = load_pair("dragon")
    else:
        Xf, Xm = _utm_c3()
    with _capi.Engine() as e:
        ref = _run(e, Xf, Xm, PATHS[0], 3.0)
        for opts in PATHS[1:]:
            _same(_run(e, Xf, Xm, opts, 3.0), ref, f"{pair} {opts}")
        for occ in (0.25, 64.0):
            got = _run(e, Xf, Xm, PATHS[0], occ)
            assert [r["n_kept"] for r in got[1]] == [r["n_kept"] for r in ref[1]], f"{pair} occ {occ}"
            # rotations to rounding; translations to rounding times the lever arm of rotations
            # about the origin (5e6 m for the UTM pair)
            tol = np.full((4, 4), 1e-11)
            tol[:3, 3] = 1e-11 * max(1.0, np.abs(Xm).max())
            assert (np.abs(got[0] - ref[0]) <= tol).all(), f"{pair} occ {occ}: {np.abs(got[0] - ref[0]).max()}"


@pytest.mark.gpu
def test_batch_mixing_origins_equals_per_pair(gpu):
    """A batch mixing a pair at the origin, one at the UTM origin, a planar pair and a one-cell
    movable cloud: the same status and bit-identical H on every search path of the batched
    match, and per pair what register returns.

    The planar pair fails (its normals are all (0, 0, 1): tx, ty and the rotation about z are
    not determined) in the batch and in register alike.  The other three are compared with
    register to rounding: the batched reject/solve kernel is not bit-identical to the single-pair
    kernels (7e-17 at the origin, 7e-12 on the ill-conditioned one-cell pair), and with Euler
    angles about the origin a 5e6 m lever arm turns that into 5e-5 m in the UTM pair's
    translation.  Those are properties of the solve, not of the search."""
    import simpleicp_b200 as sb
    from simpleicp_b200.simpleicp import SimpleICPException

    rng = np.random.default_rng(3)

    def surf(seed, origin):
        X = O.surface(30_000, seed, extent=30.0)
        return np.round(X / U) * U + np.asarray(origin)

    plane = np.column_stack((rng.integers(0, 30 * 1024, (20_000, 2)) * U, np.zeros(20_000)))
    plane_m = plane + [3 * U, -2 * U, 5 * U]
    one_cell_m = np.round(rng.uniform(0, 1, (500, 3)) / U) * U * 0.001 + 2.0
    one_cell_f = np.round(rng.uniform(0, 1, (2000, 3)) / U) * U * 0.002 + 2.0
    pairs = [(surf(1, (0, 0, 0)), surf(2, (0, 0, 0)) + [0.05, -0.03, 0.02]),
             (surf(3, O_UTM), surf(4, O_UTM) + [0.05, -0.03, 0.02]),
             (plane, plane_m),
             (one_cell_f, one_cell_m)]
    ok = [True, True, False, True]
    results = {}
    with _capi.Engine() as e:
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        params = e.run_params(0.3, 1.0, 100, lsq)
        for opts in (PATHS[0], PATHS[5], PATHS[9]):
            e.reset_options()
            set_paths(e, opts)
            res = e.register_batch(pairs, 1000, 10, params)
            results[str(opts)] = [(b.status, np.array(b.H).reshape(4, 4)) for b in res]
        for i, (Xf, Xm) in enumerate(pairs):
            st, H_b = results[str(PATHS[0])][i]
            assert (st == 0) == ok[i], f"pair {i}: status {st}"
            for key, rs in results.items():
                assert rs[i][0] == st, f"pair {i} {key}: status"
                assert np.array_equal(rs[i][1], H_b), f"pair {i} {key}"
            e.reset_options()
            if not ok[i]:
                with pytest.raises(SimpleICPException):
                    sb.register(Xf, Xm, engine=e, want_normals=False)
                continue
            r = sb.register(Xf, Xm, engine=e, want_normals=False)
            tol = np.full((4, 4), 1e-12 if i == 0 else 1e-10)
            tol[:3, 3] *= max(1.0, np.abs(Xm).max())
            assert (np.abs(H_b - r.H) <= tol).all(), f"pair {i}: {np.abs(H_b - r.H).max()}"


def teardown_module(module):
    for e in _engine_cache().values():
        e.close()
    _engine_cache().clear()
    if RUN_COUNTS:
        print("queries checked per path:", RUN_COUNTS)
