"""The cell plans of the grid builder (csrc/grid_plan.h, grid.cu: grid_build) against a NumPy
statement of its two policies, with the exact occupancy of a cloud for a given cell size.

CPU: grid_plan.h compiled with g++ and stepped with NumPy's occupancies, on designed clouds that
reach every branch of both policies.  GPU: the one-pair grids sicp_set_clouds and
sicp_estimate_normals build (Engine.grid_params) equal the one-pair statement."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

from conftest import REPO

CAP = 1 << 25    # cells
ATTEMPTS = 4
O_UTM = np.array([612345.25, 5432109.875, 310.5])


# --------------------------------------------------------------------------- the statement
def cap_of(policy, n):
    return CAP if policy == "pair" else min(CAP, max(4096, 32 * n))


def fit(ext, h, cap):
    """Dims of h; h grows by 1.26 while they exceed the cap.  Returns (h, dims, capped)."""
    capped = False
    while True:
        d = tuple(max(1, int(np.floor(x / h)) + 1) for x in ext)
        if d[0] * d[1] * d[2] <= cap:
            return h, d, capped
        h *= 1.26
        capped = True


def first_plan(X, target=3.0, policy="pair"):
    """(origin, h, dims, capped) of the first attempt: h ~ sqrt(target A / n), A the product of
    the two largest extents (a 2-D manifold in 3-D), fitted under the policy's cap."""
    lo = X.min(0)
    ext = X.max(0) - lo
    e = np.sort(ext)
    emax = max(e[2], 1e-12)
    area = max(e[2] * max(e[1], 1e-3 * emax), 1e-300)
    h = max(math.sqrt(target * area / max(len(X), 1)), emax * 1e-6)
    return (lo,) + fit(ext, h, cap_of(policy, len(X)))


def occupied(X, o, h, d):
    """Occupied cells: floor((v - o) * (1 / h)) per axis, clamped to [0, dims - 1] as cell_coord
    clamps it."""
    c = np.floor((X - o) * (1.0 / h))
    c = np.minimum(np.maximum(c, 0), np.array(d) - 1).astype(np.int64)
    return len(np.unique((c[:, 2] * d[1] + c[:, 1]) * d[0] + c[:, 0]))


def plan(X, policy, target=3.0):
    """The final (origin, h, dims) of a policy and how it got there: the attempt it stopped at,
    the exit ("band", "exhausted", "cannot_refine" for the one pair, "capped" for the batch),
    the direction of every rescale and whether any fit hit the cap."""
    o, h, d, capped = first_plan(X, target, policy)
    n, ext = len(X), X.max(0) - o
    steps, hit_cap = [], capped
    for attempt in range(ATTEMPTS):
        occ = n / max(occupied(X, o, h, d), 1)
        if attempt == ATTEMPTS - 1:
            exit_ = "exhausted"
        elif target / 1.6 <= occ <= target * 1.6:
            exit_ = "band"
        elif policy == "pair" and occ > target and d[0] * d[1] * d[2] * 2 > CAP:
            exit_ = "cannot_refine"
        elif policy == "batch" and capped:
            exit_ = "capped"
        else:
            f = min(max((target / occ) ** (1 / 2.3), 0.25), 4.0)
            steps.append("coarsen" if f > 1 else "refine")
            h, d, capped = fit(ext, h * f, cap_of(policy, n))
            hit_cap = hit_cap or capped
            continue
        return dict(o=o, h=h, dims=d, attempt=attempt, exit=exit_, steps=steps, hit_cap=hit_cap)


# --------------------------------------------------------------------------- designed clouds
def _uniform(rng, n, size):
    return rng.uniform(0.0, 1.0, (n, 3)) * np.asarray(size, dtype=np.float64)


def cloud(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    base = name.removesuffix("_utm")
    if base == "sheet":          # ~3 points per cell at the first estimate: accepted at attempt 0
        X = _uniform(rng, 20000, (10.0, 20.0, 0.0))
    elif base == "slab":         # thicker than a sheet: too sparse, coarsened once
        X = _uniform(rng, 20000, (10.0, 10.0, 0.5))
    elif base == "rows":         # 40 lines 0.25 apart in a 2-D box: too full, refined once
        X = np.column_stack((rng.uniform(0.0, 10.0, 20000), rng.integers(0, 40, 20000) * 0.25, np.zeros(20000)))
    elif base == "cube":         # a 3-D cloud under the 2-D estimate: coarsened at every attempt
        X = _uniform(rng, 20000, (1.0, 1.0, 1.0))
    elif base == "diagonal":     # a line in a 2-D box: refined until the batch cap binds
        t = rng.uniform(0.0, 1.0, 20000)
        X = np.column_stack((8.0 * t, 5.0 * t, np.zeros_like(t)))
    elif base == "clusters":     # 10 coincident points per site: never in the band
        X = np.repeat(_uniform(rng, 1000, (10.0, 10.0, 0.0)), 10, axis=0)
    elif base == "dense_cube":   # the cap binds for both policies
        X = _uniform(rng, 400000, (1.0, 1.0, 1.0))
    elif base == "sparse_cube":  # the batch cap binds and the cells are too empty: the policies part
        X = _uniform(rng, 50000, (1.0, 1.0, 1.0))
    elif base == "dense_sites":  # 20 points per site in a cube: capped, too full, cannot refine
        X = np.repeat(_uniform(rng, 20000, (1.0, 1.0, 1.0)), 20, axis=0)
    elif base == "line":         # two zero extents
        X = np.zeros((5000, 3))
        X[:, 0] = rng.uniform(0.0, 30.0, 5000)
    elif base == "point":        # three zero extents
        X = np.zeros((7, 3)) + [1.5, -2.25, 0.125]
    elif base == "single":       # one point
        X = np.array([[0.5, 0.25, -0.75]])
    else:
        raise KeyError(name)
    return X + O_UTM if name.endswith("_utm") else X


# cloud: (exit, attempt, first rescale or None, first fit capped) of the one-pair and the batch policy
EXPECT = {
    "sheet": [("band", 0, None, False)] * 2,
    "slab": [("band", 1, "coarsen", False)] * 2,
    "rows": [("band", 1, "refine", False)] * 2,
    "cube": [("exhausted", 3, "coarsen", False)] * 2,
    "diagonal": [("exhausted", 3, "refine", False), ("capped", 2, "refine", False)],
    "clusters": [("exhausted", 3, "refine", False)] * 2,
    "dense_cube": [("exhausted", 3, "coarsen", True), ("capped", 0, None, True)],
    "sparse_cube": [("exhausted", 3, "coarsen", False), ("capped", 0, None, True)],
    "dense_sites": [("cannot_refine", 0, None, True), ("capped", 0, None, True)],
    "line": [("band", 0, None, False)] * 2,
    "point": [("exhausted", 3, "refine", False)] * 2,
    "single": [("exhausted", 3, "coarsen", False)] * 2,
}
CLOUDS = list(EXPECT) + [b + "_utm" for b in ("sheet", "slab", "rows", "cube", "diagonal", "line", "point")]


@pytest.mark.parametrize("name", list(EXPECT))
def test_designed_clouds_take_their_branch(name):
    """The statement on the designed clouds: between them they take every branch of both
    policies; sparse_cube is where the two part (the batch cap binds on cells that are too empty:
    the batch stops, the one pair coarsens)."""
    X = cloud(name)
    for policy, want in zip(("pair", "batch"), EXPECT[name]):
        r = plan(X, policy)
        got = (r["exit"], r["attempt"], (r["steps"] or [None])[0], first_plan(X, 3.0, policy)[3])
        assert got == want, (policy, got, want)


# --------------------------------------------------------------------------- CPU: grid_plan.h
@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("grid_plan") / "libgrid_plan_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                    str(REPO / "tests" / "native" / "grid_plan_host.cpp"), "-o", str(out)], check=True)
    lib = C.CDLL(str(out))
    lib.grid_plan_first.restype = None
    lib.grid_plan_next.restype = C.c_int
    return lib


def stepped(lib, X, policy, target=3.0):
    """grid_plan.h driven the way grid_build drives it, with NumPy's occupancies."""
    o = X.min(0)
    ext = np.ascontiguousarray(X.max(0) - o)
    one_pair, n = int(policy == "pair"), C.c_longlong(len(X))
    h, d, capped = C.c_double(), (C.c_longlong * 3)(), C.c_int()
    e = ext.ctypes.data_as(C.c_void_p)
    lib.grid_plan_first(one_pair, C.c_double(target), e, n, C.byref(h), d, C.byref(capped))
    for attempt in range(ATTEMPTS):
        nocc = occupied(X, o, h.value, tuple(d))
        if lib.grid_plan_next(one_pair, C.c_double(target), e, n, C.c_longlong(nocc), attempt, C.byref(h), d,
                              C.byref(capped)):
            return o, h.value, tuple(d), attempt
    raise AssertionError("no final plan after four attempts")


@pytest.mark.parametrize("policy", ["pair", "batch"])
@pytest.mark.parametrize("name", CLOUDS)
def test_header_equals_statement(lib, name, policy):
    X = cloud(name)
    want = plan(X, policy)
    o, h, d, attempt = stepped(lib, X, policy)
    assert np.array_equal(o, want["o"]) and h == want["h"] and d == want["dims"], ((h, d), want)
    assert attempt == want["attempt"], (attempt, want)


@pytest.mark.parametrize("target", [0.5, 8.0])
@pytest.mark.parametrize("policy", ["pair", "batch"])
def test_header_equals_statement_other_targets(lib, target, policy):
    """The option grid_target_occupancy moves the band and the estimate alike."""
    for name in ("sheet", "cube_utm", "diagonal"):
        X = cloud(name)
        want = plan(X, policy, target)
        o, h, d, attempt = stepped(lib, X, policy, target)
        assert h == want["h"] and d == want["dims"] and attempt == want["attempt"], (name, (h, d), want)


# --------------------------------------------------------------------------- GPU: the one-pair grids
@pytest.mark.gpu
@pytest.mark.parametrize("name", CLOUDS)
def test_pair_grids_follow_the_one_pair_policy(gpu, name):
    """The movable grid of sicp_set_clouds and the fixed grid of sicp_estimate_normals."""
    from simpleicp_b200 import _capi

    X = cloud(name)
    want = plan(X, "pair")
    with _capi.Engine() as e:
        e.set_clouds(X, X)
        got_mov = e.grid_params("mov")
        e.set_selected(np.arange(min(len(X), 16)))
        if len(X) >= 2:
            e.estimate_normals(2)
            got = [got_mov, e.grid_params("fix")]
        else:
            got = [got_mov]
    for o, h, d in got:
        assert np.array_equal(o, want["o"]) and h == want["h"] and d == want["dims"], ((o, h, d), want)
