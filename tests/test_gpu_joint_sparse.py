"""sicp_register_joint / simpleicp_joint under the sparse solve (option joint_solver 1, DESIGN.md
§6.11) on the GPU: against the dense solve on the ring and on strips of 127 and 255 free clouds;
lock-step with the NumPy restatement (oracle/joint_oracle.py) on the ring and on a strip of 1023
free clouds; four and sixteen independent strips in one call (F = 1020 and 4080) against each
strip through the dense solve; relabelled clouds; determinism; the failures and the call order;
memory kinds; and simpleicp_joint(solver="sparse")."""
import ctypes as C

import numpy as np
import pytest
import torch

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

from test_gpu_joint import _lockstep, _params, strip
from test_joint_host import ring

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _joint(eng, solver, scans, edges, fixed, H0, mod=1.0, **kw):
    """register_joint under joint_solver `solver`, with its batch outputs; the option is reset."""
    is_fixed = np.zeros(len(scans), dtype=bool)
    is_fixed[list(fixed)] = True
    eng.set_option("joint_solver", solver)
    try:
        H, out = eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, _params(eng, **kw), mod)
        return H, out, eng.batch_outputs(out)
    finally:
        eng.set_option("joint_solver", 0)


def _assert_agree(a, b, pose_tol=1e-9):
    """Two runs of one problem: iterations, convergence and every kept count exact; poses within
    pose_tol; every record's statistics and the batch outputs' residuals within 1e-9 m.  (A mean,
    median or MAD near zero carries the rounding of the poses, about 1e-12 rad times lever arms of
    tens of metres, so a relative bound would not fit it.)"""
    (Ha, outa, oa), (Hb, outb, ob) = a, b
    assert [(o.status, o.iterations, o.converged) for o in outa] == [(o.status, o.iterations, o.converged) for o in outb]
    assert np.abs(Ha - Hb).max() < pose_tol
    for o, (Xa, ra, la, Ta), (Xb, rb, lb, Tb) in zip(outa, oa, ob):
        if o.status != 0:
            continue
        for it in range(o.iterations):
            assert la[it].n_kept == lb[it].n_kept, it
            for f in ("mean_res", "std_res", "median", "mad"):
                u, v = getattr(la[it], f), getattr(lb[it], f)
                assert abs(u - v) <= 1e-9, (it, f, u, v)
        assert ra.size == rb.size
        assert np.abs(ra - rb).max() <= 1e-9


PROBLEMS = {"ring": lambda: ring(), "strip_128": lambda: strip(128, 50_000, 400),
            "strip_256": lambda: strip(256, 20_000, 800)}


@pytest.mark.parametrize("problem", list(PROBLEMS))
def test_sparse_equals_dense(eng, problem):
    scans, truth, H0, edges = PROBLEMS[problem]()
    dense = _joint(eng, 0, scans, edges, (0,), H0)
    sparse = _joint(eng, 1, scans, edges, (0,), H0)
    assert all(o.status == 0 for o in dense[1])
    _assert_agree(dense, sparse)


def test_ring_lockstep_with_the_oracle(eng):
    scans, truth, H0, edges = ring()
    eng.set_option("joint_solver", 1)
    try:
        H, out, logs, ref = _lockstep(eng, scans, H0, edges, (0,))
    finally:
        eng.set_option("joint_solver", 0)
    assert all(o.iterations == len(ref.log) for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row]
    assert np.abs(H - ref.H).max() < 1e-9


def _strips(k, n, n_points, n_edges):
    """k strips of n clouds, one problem: strip s is strip(n, ., seed 11 + s) with the first two
    clouds (scans, truth and start poses) of strip 0, so that every strip's first edge is strip 0's
    and the common centre c_w of the increments (the first edge's movable box centre, DESIGN.md
    §6.9) is the same in the joint call and in each strip's own call.  The strips share no edge."""
    parts = [strip(n, n_points, n_edges, seed=11 + s) for s in range(k)]
    scans, truth, H0, edges = [], [], [], []
    for s, (sc, tr, h0, ed) in enumerate(parts):
        sc, tr, h0 = list(sc), tr.copy(), h0.copy()
        sc[:2], tr[:2], h0[:2] = parts[0][0][:2], parts[0][1][:2], parts[0][2][:2]
        parts[s] = (sc, tr, h0, ed)
        scans += sc
        truth.append(tr)
        H0.append(h0)
        edges.append(ed + s * n)
    return parts, scans, np.concatenate(truth), np.concatenate(H0), np.concatenate(edges)


def test_four_strips_in_one_call_equal_each_strip_alone(eng):
    """F = 4 x 255 = 1020: the joint matrix is block diagonal, one block per strip.  Fixed
    iterations (min_change = 0 never stops) so that the iteration counts cannot part."""
    parts, scans, truth, H0, edges = _strips(4, 256, 10_000, 800)
    kw = dict(max_iterations=4, min_change=0.0)
    H, out, outputs = _joint(eng, 1, scans, edges, (0, 256, 512, 768), H0, **kw)
    for s, (sc, tr, h0, ed) in enumerate(parts):
        Hs, outs, os_ = _joint(eng, 0, sc, ed, (0,), h0, **kw)
        e = slice(s * len(ed), (s + 1) * len(ed))
        assert np.abs(H[256 * s:256 * (s + 1)] - Hs).max() < 1e-9, s
        for o, p, (_, _, la, _), (_, _, lb, _) in zip(out[e], outs, outputs[e], os_):
            assert (o.status, o.iterations) == (p.status, p.iterations) == (0, 4)
            assert [r.n_kept for r in la[:4]] == [r.n_kept for r in lb[:4]]


def test_strip_of_1023_free_clouds_lockstep_with_the_oracle(eng):
    """A connected problem past the dense solve's cap: 1024 clouds of 5 000 points, 3 000 edges,
    three iterations in lock-step with the oracle (whose dense solve of 6 138 unknowns is the
    reference).  Its far clouds sit 2 km from c_w, which the strips of the block-diagonal tests do
    not reach.  Kept counts exact.  The poses: the rule itself moves this strip's poses by metres
    in three iterations, and the gap between any two solves of it grows with that motion: on a strip
    of 255 free clouds of 5 000 points the established dense solve is already 3.6e-9 from the oracle
    after three iterations (the sparse one 3.6e-9 too), and here the sparse solve is 2.0e-6 from it
    (H100).  The bound is set above that, with the dense path's behaviour as the reference (DESIGN.md
    §6.11, Limits)."""
    scans, truth, H0, edges = strip(1024, 5_000, 3_000, seed=12)
    eng.set_option("joint_solver", 1)
    try:
        H, out, logs, ref = _lockstep(eng, scans, H0, edges, (0,), max_iterations=3)
    finally:
        eng.set_option("joint_solver", 0)
    assert all(o.status == 0 and o.iterations == len(ref.log) == 3 for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row], it
    assert np.abs(H - ref.H).max() < 1e-5


def test_relabelled_clouds_give_the_same_poses(eng):
    """A random permutation of the cloud indices and of the edges after the first (which fixes the
    common centre c_w): another ordering of the same system, so only rounding may differ."""
    scans, truth, H0, edges = strip(128, 20_000, 400)
    rng = np.random.default_rng(7)
    new = rng.permutation(len(scans))            # cloud i becomes cloud new[i]
    old = np.argsort(new)
    order = np.concatenate(([0], 1 + rng.permutation(len(edges) - 1)))
    E = new[edges[order]]
    H, out, _ = _joint(eng, 1, scans, edges, (0,), H0)
    Hp, outp, _ = _joint(eng, 1, [scans[i] for i in old], E, (int(new[0]),), H0[old])
    assert np.abs(Hp[new] - H).max() < 1e-9
    assert [o.n_kept for o in outp] == [out[e].n_kept for e in order]


def test_two_calls_give_the_same_bits(eng):
    scans, truth, H0, edges = strip(128, 20_000, 400)
    H, out, o = _joint(eng, 1, scans, edges, (0,), H0)
    H2, out2, o2 = _joint(eng, 1, scans, edges, (0,), H0)
    assert np.array_equal(H, H2)
    assert all(bytes(a) == bytes(b) for a, b in zip(out, out2))
    for (X, r, lg, T), (X2, r2, lg2, T2) in zip(o, o2):
        assert np.array_equal(X, X2) and np.array_equal(r, r2) and np.array_equal(T, T2)
        assert all(bytes(a) == bytes(b) for a, b in zip(lg, lg2))


def test_memory_kinds_give_the_same_bits(eng):
    scans, truth, H0, edges = ring()
    H, out, _ = _joint(eng, 1, scans, edges, (0,), H0)
    pinned = [torch.from_numpy(s).pin_memory() for s in scans]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    for kind in (pinned, dev):
        H2, out2, _ = _joint(eng, 1, kind, edges, (0,), H0)
        assert np.array_equal(H, H2)
        assert all(bytes(a) == bytes(b) for a, b in zip(out, out2))


def test_failures(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    eng.set_option("joint_solver", 1)
    try:
        # two clouds sampled from one plane: not positive definite, H_out not written
        rng = np.random.default_rng(3)
        P = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
        Q = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
        H_out = np.full((2, 4, 4), 7.0)
        rp = eng._register_params(1000, 10, p, 1.0, 0, -1.0)
        ptrs = (C.c_void_p * 2)(P.ctypes.data, Q.ctypes.data)
        counts = (C.c_int64 * 2)(5000, 5000)
        fix, mov = np.array([0], dtype=np.int32), np.array([1], dtype=np.int32)
        is_fixed = np.array([1, 0], dtype=np.int32)
        out = (_capi.PairResult * 1)()
        i32p = C.POINTER(C.c_int32)
        rc = eng._lib.sicp_register_joint(eng._h, 2, ptrs, counts, 1, fix.ctypes.data_as(i32p),
                                          mov.ctypes.data_as(i32p), is_fixed.ctypes.data_as(i32p), None, C.byref(rp),
                                          H_out.ctypes.data, out, None)
        assert rc == _capi.SICP_ERR_SINGULAR
        assert (H_out == 7.0).all()
        # no overlap: parked when a second path anchors the cloud, the call's failure when not
        W7 = scans[7] @ truth[7][:3, :3].T + truth[7][:3, 3]
        tail = np.ascontiguousarray(scans[7][W7[:, 0] >= 28.0])
        c4 = [scans[0], scans[2], scans[4], tail]
        H04 = np.stack([H0[0], H0[2], H0[4], H0[7]])
        fx4 = np.array([True, False, False, False])
        with pytest.raises(SicpError) as ei:
            eng.register_joint(c4, [(0, 1), (0, 3)], fx4, H04, 1000, 10, p, 1.0)
        assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
        H, out2 = eng.register_joint(c4, [(0, 1), (1, 2), (2, 3), (0, 3)], fx4, H04, 1000, 10, p, 1.0)
        assert [o.status for o in out2] == [0, 0, 0, _capi.SICP_ERR_NO_OVERLAP]
        assert np.abs(H[3] - truth[7]).max() < 1e-2
    finally:
        eng.set_option("joint_solver", 0)
    # the same parked problem through the dense solve
    Hd, outd = eng.register_joint(c4, [(0, 1), (1, 2), (2, 3), (0, 3)], fx4, H04, 1000, 10, p, 1.0)
    assert np.abs(H - Hd).max() < 1e-9 and [o.n_kept for o in out2] == [o.n_kept for o in outd]


def test_call_order(eng):
    scans, truth, H0, edges = ring()
    fresh = _capi.Engine(0)
    try:
        want = _joint(fresh, 0, scans, edges, (0,), H0)
        want_cov = fresh.joint_covariances(len(scans), len(edges))
    finally:
        fresh.close()
    H, out, outputs = _joint(eng, 1, scans, edges, (0,), H0)
    with pytest.raises(SicpError, match="covariances need joint_solver 0") as ei:
        eng.joint_covariances(len(scans), len(edges))
    assert ei.value.code == _capi.SICP_ERR_STATE
    assert len(eng.batch_outputs(out)) == len(edges)
    # a dense call after a sparse one on the same engine: the bits of a fresh engine
    got = _joint(eng, 0, scans, edges, (0,), H0)
    assert np.array_equal(got[0], want[0])
    assert all(bytes(a) == bytes(b) for a, b in zip(got[1], want[1]))
    for a, b in zip(got[2], want[2]):
        assert all(np.array_equal(x, y) for x, y in zip((a[0], a[1], a[3]), (b[0], b[1], b[3])))
    cov = eng.joint_covariances(len(scans), len(edges))
    assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(cov[:2], want_cov[:2])) and cov[2] == want_cov[2]
    # the option's values and "defaults"
    with pytest.raises(SicpError):
        eng.set_option("joint_solver", 2)
    eng.set_option("joint_solver", 1)
    eng.set_option("defaults", 0)
    again = _joint(eng, 0, scans, edges, (0,), H0)
    assert np.array_equal(again[0], want[0])


def test_simpleicp_joint_sparse_calls_leave_the_engine_dense():
    scans, truth, H0, edges = ring()
    dense = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    sparse = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0, solver="sparse",
                                full_output=True)
    assert np.abs(sparse.H - dense.H).max() < 1e-9 and sparse.iterations == dense.iterations
    assert len(sparse.results) == len(edges)
    again = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0, covariances=True)
    assert np.array_equal(again.H, dense.H) and again.cov is not None


def test_sixteen_strips_of_255_free_clouds_equal_each_strip_alone(eng):
    """F = 16 x 255 = 4080, two iterations: more supernodes per level than the grid has blocks, so
    every block factors several panels per level.  The first four strips against the dense solve."""
    parts, scans, truth, H0, edges = _strips(16, 256, 5_000, 800)
    kw = dict(max_iterations=2, min_change=0.0)
    H, out, outputs = _joint(eng, 1, scans, edges, tuple(range(0, 16 * 256, 256)), H0, **kw)
    assert all(o.status == 0 for o in out)
    for s, (sc, tr, h0, ed) in enumerate(parts[:4]):
        Hs, outs, _ = _joint(eng, 0, sc, ed, (0,), h0, **kw)
        assert np.abs(H[256 * s:256 * (s + 1)] - Hs).max() < 1e-9, s
        e = slice(s * len(ed), (s + 1) * len(ed))
        assert [o.n_kept for o in out[e]] == [o.n_kept for o in outs]

