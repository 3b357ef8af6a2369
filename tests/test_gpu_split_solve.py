"""The serial tail of the barrier-free reject/solve kernel (reduction of the per-block partials, the
Gauss-Newton solve, statistics, state and record stores) runs in the one-block kernel k_rs_solve
launched behind the select/accumulate grid.  With programmatic dependent launch (option pdl 1, the
default) k_rs_solve first rehearses the tail on the previous iteration's partials while the grid
runs; without it (pdl 0) it runs the tail once.  Nothing the rehearsal does may show in a result:
whole registrations must agree bit for bit."""
import numpy as np
import pytest

from conftest import load_pair

import simpleicp_b200 as sb
from simpleicp_b200 import _capi, synthetic


def bits(res):
    """Every output of a registration as raw 64-bit patterns (NaN-safe equality)."""
    recs = res.records[:res.iterations]
    rec = [np.hstack([np.ravel(np.asarray(r[k], dtype=np.float64)) for k in sorted(r)]) for r in recs]
    out = [np.asarray(res.H, dtype=np.float64), np.asarray(res.X_mov_transformed, dtype=np.float64),
           np.asarray(res.residuals, dtype=np.float64)] + rec
    return res.iterations, [np.ascontiguousarray(a).view(np.uint64) for a in out]


def assert_same(a, b, what):
    assert a[0] == b[0], f"{what}: {a[0]} vs {b[0]} iterations"
    assert len(a[1]) == len(b[1])
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        assert x.shape == y.shape and np.array_equal(x, y), f"{what}: output {i} differs"


def run(e, X_fix, X_mov, K, pdl):
    e.set_option("pdl", pdl)
    n0 = e.timings()["kernel_launches"]
    res = sb.register(X_fix, X_mov, correspondences=K, engine=e, want_normals=False)
    tm = e.timings()
    assert tm["fused_iterations"] > 0  # the barrier-free kernel served iterations
    return bits(res), tm["kernel_launches"] - n0, tm["fused_iterations"]


@pytest.fixture(scope="module")
def pairs():
    X_fix, X_mov, _ = synthetic.c3_pair(1_000_000, shift=0)
    A_fix, A_mov = load_pair("airborne")
    # C3: 131 blocks of one tile each; airborne at K = 200 000: several tiles per block and the
    # grid at its cap of one block per SM but one
    return {"c3": (X_fix, X_mov, 100_000), "airborne": (A_fix, A_mov, 200_000)}


def launches_per_iteration(e, p, fused):
    """Kernel launches of one steady-state iterate() call, and the selection path it took."""
    e.set_option("fused", fused)
    for _ in range(3):
        n0 = e.timings()["kernel_launches"]
        rec = e.iterate(p, want_record=True)
        n = e.timings()["kernel_launches"] - n0
    assert rec.n_bruteforce == 0
    return n, e.selection()["path"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c3", "airborne"])
def test_rehearsal_matches_plain_tail(gpu, pairs, name):
    X_fix, X_mov, K = pairs[name]
    with _capi.Engine() as e:
        # without PDL the solve kernel skips its rehearsal
        ref, launches_ref, fused_ref = run(e, X_fix, X_mov, K, pdl=0)
    with _capi.Engine() as e:
        new, launches_new, fused_new = run(e, X_fix, X_mov, K, pdl=1)
    assert_same(ref, new, f"{name} pdl 0 vs 1")
    assert (launches_new, fused_new) == (launches_ref, fused_ref)
    # k_rs_solve ran: a barrier-free iteration launches one kernel more than a cooperative one
    with _capi.Engine() as e:
        e.set_clouds(X_fix, X_mov)
        e.set_selected(sb.pointcloud.subsample_indices(X_fix.shape[0], K).astype(np.int64))
        e.estimate_normals(10)
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        p = e.run_params(0.3, 1.0, 100, lsq)
        e.iterate(p, x_in=np.zeros(6), want_record=True)
        n_fused, path_fused = launches_per_iteration(e, p, 1)
        n_coop, path_coop = launches_per_iteration(e, p, 0)
    assert (path_fused, path_coop) == (_capi.SEL_PATH_BINSTORE, _capi.SEL_PATH_RADIX)
    assert n_fused == n_coop + 1


@pytest.mark.gpu
def test_rehearsal_leaves_no_trace(gpu, pairs):
    """The rehearsal reads partials a different problem left (another pair, another grid size)
    and the loop state of the run in progress; what it computes goes to scratch memory only."""
    X_fix, X_mov, K = pairs["c3"]
    A_fix, A_mov, KA = pairs["airborne"]
    with _capi.Engine() as e:
        ref, _, _ = run(e, X_fix, X_mov, K, pdl=0)
    with _capi.Engine() as e:
        run(e, A_fix, A_mov, KA, pdl=1)
        again, _, _ = run(e, X_fix, X_mov, K, pdl=1)
        twice, _, _ = run(e, X_fix, X_mov, K, pdl=1)
    assert_same(ref, again, "c3 after airborne")
    assert_same(ref, twice, "c3 repeated")
