"""The serial tail of the barrier-free reject/solve kernel (reduction of the per-block partials, the
Gauss-Newton solve, statistics, state and record stores) runs either in the kernel's last block
(option split_solve 0) or in the one-block kernel k_rs_solve launched behind it (split_solve 1, the
default), which first rehearses the tail on the previous iteration's partials.  Both reduce the
same partials in the same order, so whole registrations must agree bit for bit, and nothing the
rehearsal does may show in a result."""
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


def run(e, X_fix, X_mov, K, split, pdl=1):
    e.set_option("split_solve", split)
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


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c3", "airborne"])
def test_split_solve_matches_last_block_tail(gpu, pairs, name):
    X_fix, X_mov, K = pairs[name]
    with _capi.Engine() as e:
        ref, launches_ticket, fused_ticket = run(e, X_fix, X_mov, K, split=0)
    with _capi.Engine() as e:
        new, launches_split, fused_split = run(e, X_fix, X_mov, K, split=1)
        # without PDL the solve kernel skips its rehearsal
        nopdl, _, _ = run(e, X_fix, X_mov, K, split=1, pdl=0)
    assert_same(ref, new, f"{name} split_solve 0 vs 1")
    assert_same(ref, nopdl, f"{name} split_solve 1 without PDL")
    # k_rs_solve ran: one more launch behind every launch of the select kernel
    assert fused_split == fused_ticket
    assert launches_split > launches_ticket


@pytest.mark.gpu
def test_rehearsal_leaves_no_trace(gpu, pairs):
    """The rehearsal reads partials a different problem left (another pair, another grid size)
    and the loop state of the run in progress; what it computes goes to scratch memory only."""
    X_fix, X_mov, K = pairs["c3"]
    A_fix, A_mov, KA = pairs["airborne"]
    with _capi.Engine() as e:
        ref, _, _ = run(e, X_fix, X_mov, K, split=0)
    with _capi.Engine() as e:
        run(e, A_fix, A_mov, KA, split=1)
        again, _, _ = run(e, X_fix, X_mov, K, split=1)
        twice, _, _ = run(e, X_fix, X_mov, K, split=1)
    assert_same(ref, again, "c3 after airborne")
    assert_same(ref, twice, "c3 repeated")
