"""sicp_register_joint_relative / simpleicp_joint(relative_pairs=, relative_poses=,
relative_weights=) on the GPU (DESIGN.md §6.13): the bits of sicp_register_joint_priors without an
observation read, an observation from a fixed cloud at the identity against a prior, lock-step with
the NumPy restatement (joint_relative_oracle.py) on the ring and on 127 free clouds under both
solves, a gap in the edge graph bridged by odometry, the covariances against the NumPy rule
(joint_relative_cov_rule.py), georeferenced coordinates, the C argument checks, determinism, the
misclosure and an end-to-end call."""
import ctypes as C

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

import joint_relative_cov_rule as JRC
import joint_relative_oracle as JRO
from test_gpu_joint import _device_normals, _params, strip
from test_gpu_joint_cov import _sig
from test_gpu_joint_priors import _c4, _everything, _noisy, _ring_priors
from test_joint_host import ring

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _odometry(truth, pairs, seed, rot_deg, pos_m, row_m):
    """Observations of T_a^-1 T_b for `pairs` from the truth with seeded noise of rot_deg and pos_m
    (standard deviations, in frame b), weighted for rows of row_m metres."""
    rng = np.random.default_rng(seed)
    Z = []
    for a, b in pairs:
        E = np.eye(4)
        E[:3, :3] = Rotation.from_rotvec(np.deg2rad(rng.normal(0, rot_deg, 3))).as_matrix()
        E[:3, 3] = rng.normal(0, pos_m, 3)
        Z.append(np.linalg.inv(truth[a]) @ truth[b] @ E)
    W = np.tile([row_m ** 2 / np.deg2rad(rot_deg) ** 2] * 3 + [row_m ** 2 / pos_m ** 2] * 3, (len(pairs), 1))
    return np.array(pairs, dtype=np.int64), np.array(Z), W


def _ring_rel(truth):
    """Odometry (i, i + 1) and (2, 6), (1, 5): clouds no edge joins, the last position only."""
    pairs, Z, W = _odometry(truth, [(i, i + 1) for i in range(7)] + [(2, 6), (1, 5)], 61, 0.03, 0.01, 0.005)
    W[-1, :3] = 0.0
    return pairs, Z, W


def _joint(eng, solver, scans, edges, fixed, H0, P=None, W=None, rel=(), mod=1.0, max_iterations=30):
    is_fixed = np.zeros(len(scans), dtype=bool)
    is_fixed[list(fixed)] = True
    eng.set_option("joint_solver", solver)
    try:
        return eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, _params(eng, max_iterations), mod, P, W, *rel)
    finally:
        eng.set_option("joint_solver", 0)


def _register_joint_priors(eng, scans, edges, fixed, H0, P, W, mod=1.0):
    """sicp_register_joint_priors itself, through ctypes."""
    fix = np.ascontiguousarray(np.asarray(edges)[:, 0], dtype=np.int32)
    mov = np.ascontiguousarray(np.asarray(edges)[:, 1], dtype=np.int32)
    keep, ptrs, counts = _capi._clouds_arg(scans, allow_none=True)
    is_fixed = np.zeros(len(scans), dtype=np.int32)
    is_fixed[list(fixed)] = 1
    p = _params(eng)
    rp = eng._register_params(1000, 10, p, mod, 0, -1.0)
    H = np.zeros((len(scans), 4, 4))
    i32p = C.POINTER(C.c_int32)
    out = eng._batched(eng._lib.sicp_register_joint_priors, p, counts, mov, len(counts), ptrs, counts, len(fix),
                       fix.ctypes.data_as(i32p), mov.ctypes.data_as(i32p), is_fixed.ctypes.data_as(i32p),
                       np.ascontiguousarray(H0).ctypes.data, _capi._ptr(P), _capi._ptr(W), C.byref(rp), H.ctypes.data)
    return H, out


@pytest.mark.parametrize("solver", [0, 1])
def test_without_observations_read_the_bits_of_sicp_register_joint_priors(eng, solver):
    scans, truth, H0, edges = ring()
    P, W = _ring_priors(truth)
    pairs, Z, Wr = _ring_rel(truth)
    dense = solver == 0
    is_fixed = np.zeros(8, dtype=bool)
    is_fixed[0] = True
    count = lambda: eng.timings()["kernel_launches"]  # noqa: E731  (the context's running count)
    eng.set_option("joint_solver", solver)
    try:
        n0 = count()
        H, out = _register_joint_priors(eng, scans, edges, (0,), H0, P, W)
        launches = count() - n0
        ref = _everything(eng, H, out, dense)
        runs = []
        for rel in ((), (pairs, np.full_like(Z, np.nan), np.zeros_like(Wr))):  # none, all-zero weights
            n0 = count()
            H, out = eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, _params(eng), 1.0, P, W, *rel)
            runs.append((count() - n0, _everything(eng, H, out, dense)))
    finally:
        eng.set_option("joint_solver", 0)
    for n, blobs in runs:
        assert n == launches
        assert blobs == ref
    # simpleicp_joint with all-zero weights against simpleicp_joint without observations
    kw = dict(fixed=(0,), H0=H0, max_overlap_distance=1.0, covariances=dense, solver="dense" if dense else "sparse")
    a = sb.simpleicp_joint(scans, edges, **kw)
    b = sb.simpleicp_joint(scans, edges, relative_pairs=pairs, relative_poses=np.full_like(Z, np.nan),
                           relative_weights=np.zeros_like(Wr), **kw)
    assert np.array_equal(a.H, b.H) and np.array_equal(a.table, b.table, equal_nan=True)
    assert a.relative_misclosure is None and b.relative_misclosure.shape == (len(pairs), 6)
    if dense:
        assert np.array_equal(a.cov, b.cov, equal_nan=True) and np.array_equal(a.edge_cov, b.edge_cov)
        assert a.s0 == b.s0


def test_observations_between_fixed_clouds_are_not_read(eng):
    """An observation whose two clouds are fixed is not read: NaN poses pass, the bits stay."""
    scans, truth, H0, edges = ring()
    H, out = _joint(eng, 0, scans, edges, (0, 4), H0)
    Hr, outr = _joint(eng, 0, scans, edges, (0, 4), H0, rel=([(0, 4)], np.full((1, 4, 4), np.nan), np.ones((1, 6))))
    assert _everything(eng, H, out, False) == _everything(eng, Hr, outr, False)


@pytest.mark.parametrize("solver", [0, 1])
def test_observation_from_a_fixed_cloud_at_the_identity_is_a_prior(eng, solver):
    """Cloud 0 fixed at H0[0] = I: an observation (0, 3, Z, w) is the prior P_3 = Z with the same
    weights.  R_a = I makes G_b = I exactly and both terms land after cloud 3's edges, so the poses
    (and the covariances) are the same bits."""
    scans, truth, H0, edges = ring()
    S = np.linalg.inv(H0[0])
    H0 = np.array([S @ h for h in H0])
    H0[0] = np.eye(4)
    T = np.array([S @ h for h in truth])
    pairs, Z, W = _odometry(T, [(0, 3)], 71, 0.03, 0.01, 0.005)
    P = np.full((8, 4, 4), np.nan)
    P[3] = Z[0]
    Wp = np.zeros((8, 6))
    Wp[3] = W[0]
    Hp, outp = _joint(eng, solver, scans, edges, (0,), H0, P, Wp)
    bp = _everything(eng, Hp, outp, solver == 0)
    Hr, outr = _joint(eng, solver, scans, edges, (0,), H0, rel=(pairs, Z, W))
    br = _everything(eng, Hr, outr, solver == 0)
    assert np.abs(Hp - Hr).max() <= 1e-12
    assert br == bp


def _lockstep(eng, solver, scans, H0, edges, fixed, rel, P=None, W=None, max_iterations=30, nrm=None):
    H, out = _joint(eng, solver, scans, edges, fixed, H0, P, W, rel=rel, max_iterations=max_iterations)
    logs = [o[2] for o in eng.batch_outputs(out)]
    if nrm is None:
        sel = J.simpleicp_joint(scans, edges, fixed=fixed, H0=H0, max_iterations=0, max_overlap_distance=1.0)
        nrm = {e: _device_normals(eng, scans[a], sel.idx_fix[e]) for e, (a, _) in enumerate(edges)}
    ref = JRO.simpleicp_joint(scans, edges, fixed=fixed, H0=H0, max_iterations=max_iterations,
                              max_overlap_distance=1.0, normals=nrm, prior_poses=P, prior_weights=W,
                              relative_pairs=rel[0], relative_poses=rel[1], relative_weights=rel[2])
    return H, out, logs, ref, nrm


def _assert_lockstep(H, out, logs, ref, tol=1e-9):
    assert all(o.status == 0 and o.iterations == len(ref.log) for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row], it
    assert np.abs(H - ref.H).max() < tol, np.abs(H - ref.H).max()


@pytest.mark.parametrize("solver", [0, 1])
def test_ring_lockstep_with_the_oracle(eng, solver):
    scans, truth, H0, edges = ring()
    rel = _ring_rel(truth)
    H, out, logs, ref, _ = _lockstep(eng, solver, scans, H0, edges, (0,), rel)
    _assert_lockstep(H, out, logs, ref)
    assert np.abs(H - truth).max() < 1e-2


def _strip127_rel(truth, edges):
    """Odometry (i, i + 1) on every cloud and (i, i + 13) every 9th cloud, pairs no edge joins
    (closures reach at most 10 clouds)."""
    pairs = [(i, i + 1) for i in range(127)] + [(i, i + 13) for i in range(0, 115, 9)]
    assert not {(a, b) for a, b in pairs[127:]} & {tuple(e) for e in edges.tolist()}
    return _odometry(truth, pairs, 81, 0.03, 0.02, 0.01)


def test_size_128_clouds_lockstep_with_the_oracle(eng):
    scans, truth, H0, edges = strip(128, 50_000, 400)
    rel = _strip127_rel(truth, edges)
    H, out, logs, ref, nrm = _lockstep(eng, 0, scans, H0, edges, (0,), rel, max_iterations=20)
    _assert_lockstep(H, out, logs, ref)
    Hs, outs = _joint(eng, 1, scans, edges, (0,), H0, rel=rel, max_iterations=20)
    _assert_lockstep(Hs, outs, [o[2] for o in eng.batch_outputs(outs)], ref)


@pytest.mark.parametrize("solver", [0, 1])
def test_a_gap_bridged_by_odometry(eng, solver):
    """test_gpu_joint_priors.test_no_overlap_anchoring's c4: cloud 3 is tied to the rest only by an
    edge without overlap, so the call fails with SICP_ERR_NO_OVERLAP.  One full-weight observation
    (1, 3) from the truth bridges the gap: SICP_OK, cloud 3 near its truth.  A position-only one
    does not link, and the call fails as before."""
    scans, truth, H0, edges = ring()
    c4, H04 = _c4(truth, scans, H0)
    with pytest.raises(SicpError) as ei:
        _joint(eng, solver, c4, [(0, 1), (0, 3)], (0,), H04)
    assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
    Z = (np.linalg.inv(truth[2]) @ truth[7])[None]
    W = np.full((1, 6), 1e4)
    with pytest.raises(SicpError) as ei:
        _joint(eng, solver, c4, [(0, 1), (0, 3)], (0,), H04, rel=([(1, 3)], Z, np.where(np.arange(6) < 3, 0.0, W)))
    assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
    H, out = _joint(eng, solver, c4, [(0, 1), (0, 3)], (0,), H04, rel=([(1, 3)], Z, W))
    assert [o.status for o in out] == [0, _capi.SICP_ERR_NO_OVERLAP]
    assert np.abs(H[1] - truth[2]).max() < 1e-2 and np.abs(H[3] - truth[7]).max() < 2e-2
    assert np.abs(np.linalg.inv(H[1]) @ H[3] - Z[0]).max() < 1e-6


@pytest.mark.parametrize("problem", ["ring", "strip127"])
def test_covariances_with_observations_against_the_rule(eng, problem):
    if problem == "ring":
        scans, truth, H0, edges = ring()
        rel, iters = _ring_rel(truth), 30
    else:
        scans, truth, H0, edges = strip(128, 50_000, 400)
        rel, iters = _strip127_rel(truth, edges), 20
        rel[2][5:20, :3] = 0.0  # position only on some
    H, out, logs, ref, nrm = _lockstep(eng, 0, scans, H0, edges, (0,), rel, max_iterations=iters)
    _assert_lockstep(H, out, logs, ref)
    cov, ecov, s0 = eng.joint_covariances(len(scans), len(edges))
    fi = JRC.final_iteration(scans, edges, ref, fixed=(0,), H0=H0, relative_pairs=rel[0], relative_poses=rel[1],
                             relative_weights=rel[2], max_overlap_distance=1.0)
    free = list(fi.slot)
    assert abs(s0 - fi.s0) <= 1e-12 * fi.s0, (s0, fi.s0)
    ku = np.linalg.cond(fi.N) * np.finfo(np.float64).eps / 2
    d_sig = np.abs(_sig(cov[free]) / _sig(fi.cov[free]) - 1).max()
    print(f"joint covariances with relative observations ({problem}): s0 {s0:.6e} rel {abs(s0 / fi.s0 - 1):.2e}, "
          f"kappa u {ku:.1e}, sigma rel {d_sig:.2e}")
    assert d_sig < max(10 * ku, 1e-12), (d_sig, ku)


def test_georeferenced_first_iteration_is_translation_invariant(eng):
    """The ring with its observations in UTM coordinates (start poses S H0; the observations are
    relative, so they stay): equal kept counts, statistics and rotations within 1e-7 after one
    iteration, as test_gpu_joint_priors' UTM test."""
    scans, truth, H0, edges = ring()
    rel = _ring_rel(truth)
    S = np.eye(4)
    S[:3, 3] = (4.5e5, 5.4e6, 300.0)
    H0_u = np.array([S @ h for h in H0])
    eng.set_option("sign_mode", 1)
    try:
        H, out = _joint(eng, 0, scans, edges, (0,), H0, rel=rel, max_iterations=1)
        logs = [o[2][0] for o in eng.batch_outputs(out)]
        H_u, out_u = _joint(eng, 0, scans, edges, (0,), H0_u, rel=rel, max_iterations=1)
        logs_u = [o[2][0] for o in eng.batch_outputs(out_u)]
    finally:
        eng.set_option("sign_mode", 0)
    for r, ru in zip(logs, logs_u):
        assert r.n_kept == ru.n_kept
        for f in ("median", "mad", "mean_res", "std_res"):
            assert abs(getattr(r, f) - getattr(ru, f)) < 1e-7, (f, getattr(r, f), getattr(ru, f))
        assert np.abs(np.array(r.x[:3]) - np.array(ru.x[:3])).max() < 1e-7
    assert np.abs(H[:, :3, :3] - H_u[:, :3, :3]).max() < 1e-7


def test_c_argument_checks(eng):
    scans, truth, H0, edges = ring()
    scans = scans + [None]  # cloud 8: no edge references it
    H0 = np.concatenate((H0, np.eye(4)[None]))
    is_fixed = np.zeros(9, dtype=np.int32)
    is_fixed[0] = 1
    pairs, Z, W = _ring_rel(truth)
    fix = np.ascontiguousarray(edges[:, 0], dtype=np.int32)
    mov = np.ascontiguousarray(edges[:, 1], dtype=np.int32)
    keep, ptrs, counts = _capi._clouds_arg(scans, allow_none=True)
    p = _params(eng)
    rp = eng._register_params(1000, 10, p, 1.0, 0, -1.0)
    i32p = C.POINTER(C.c_int32)

    def call(n_rel, ra, rb, Zk, Wk):
        H = np.zeros((9, 4, 4))
        return eng._batched(eng._lib.sicp_register_joint_relative, p, counts, mov, 9, ptrs, counts, len(fix),
                            fix.ctypes.data_as(i32p), mov.ctypes.data_as(i32p), is_fixed.ctypes.data_as(i32p),
                            H0.ctypes.data, None, None, n_rel, ra, rb, Zk, Wk, C.byref(rp), H.ctypes.data)

    def arrays(pairs, Z, W):
        a = np.ascontiguousarray(pairs[:, 0], dtype=np.int32)
        b = np.ascontiguousarray(pairs[:, 1], dtype=np.int32)
        Z, W = np.ascontiguousarray(Z), np.ascontiguousarray(W)
        return (a, b, Z, W), (a.ctypes.data_as(i32p), b.ctypes.data_as(i32p), Z.ctypes.data, W.ctypes.data)

    def refused(n_rel, args, msg):
        with pytest.raises(SicpError) as ei:
            call(n_rel, *args)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG and msg in str(ei.value), str(ei.value)

    keep_ok, ok = arrays(pairs, Z, W)
    n = len(pairs)
    refused(-1, ok, "n_rel must be in [0, 65535]")
    refused(65536, ok, "n_rel must be in [0, 65535]")
    for k in range(4):
        args = list(ok)
        args[k] = None
        refused(n, args, "must not be NULL")
    for bad, msg in (((0, 9), "cloud ids must be in [0, n_clouds)"), ((0, -1), "cloud ids must be in [0, n_clouds)"),
                     ((3, 3), "joins a cloud to itself"), ((2, 8), "must be referenced by an edge")):
        pp = pairs.copy()
        pp[4] = bad
        keep_b, args = arrays(pp, Z, W)
        refused(n, args, "relative observation 4")
        refused(n, args, msg)
    for v in (-1.0, np.nan, np.inf):
        W2 = W.copy()
        W2[3, 4] = v
        keep_b, args = arrays(pairs, Z, W2)
        refused(n, args, "negative or not finite")
    for idx, v, msg in (((2, 1, 3), np.nan, "rel_H[2] has non-finite"), ((2, 3, 0), 1e-3, "bottom row")):
        Z2 = Z.copy()
        Z2[idx] = v
        keep_b, args = arrays(pairs, Z2, W)
        refused(n, args, msg)
    Z2 = Z.copy()
    Z2[2, :3, :3] *= 1.0 + 1e-5
    keep_b, args = arrays(pairs, Z2, W)
    refused(n, args, "orthonormal")
    # not read: zero weights, NaN pose
    assert all(o.status == 0 for o in call(n, *ok))
    W3 = W.copy()
    W3[2] = 0.0
    Z3 = Z.copy()
    Z3[2] = np.nan
    keep_c, args = arrays(pairs, Z3, W3)
    out = call(n, *args)
    assert all(o.status == 0 for o in out)
    # n_rel = 0 with NULL arrays is sicp_register_joint_priors
    out0 = call(0, None, None, None, None)
    assert all(o.status == 0 for o in out0)


@pytest.mark.parametrize("solver", [0, 1])
def test_two_calls_give_the_same_bits(eng, solver):
    scans, truth, H0, edges = ring()
    rel = _ring_rel(truth)
    a = _everything(eng, *_joint(eng, solver, scans, edges, (0,), H0, rel=rel), solver == 0)
    b = _everything(eng, *_joint(eng, solver, scans, edges, (0,), H0, rel=rel), solver == 0)
    assert a == b


def test_simpleicp_joint_with_odometry_end_to_end():
    """The quick-start call with GNSS-like priors on clouds 0 and 4 only, fixed=(), and odometry
    along the ring: both solvers agree, the poses are near the truth, the covariances are finite
    and relative_misclosure is the NumPy statement at the returned poses."""
    scans, truth, H0, edges = ring()
    P = _noisy(truth, 51, 0.05, 0.02)
    W = np.zeros((8, 6))
    W[[0, 4]] = [0.005 ** 2 / np.deg2rad(0.05) ** 2] * 3 + [0.005 ** 2 / 0.02 ** 2] * 3
    pairs, Z, Wr = _ring_rel(truth)
    kw = dict(fixed=(), H0=H0, prior_poses=P, prior_weights=W, relative_pairs=pairs, relative_poses=Z,
              relative_weights=Wr, max_overlap_distance=1.0)
    d = sb.simpleicp_joint(scans, edges, covariances=True, **kw)
    s = sb.simpleicp_joint(scans, edges, solver="sparse", **kw)
    assert np.abs(d.H - s.H).max() < 1e-9
    # two priors of 2 cm per axis hold the ring: measured 2.6 cm on an H100
    assert np.abs(d.H - truth).max() < 5e-2
    assert np.isfinite(d.s0) and (np.einsum("cii->ci", d.cov) > 0).all()
    ref = np.array([JRO.observe(d.H[a], d.H[b], Zk) for (a, b), Zk in zip(pairs, Z)])
    assert d.relative_misclosure.shape == (len(pairs), 6)
    assert np.abs(d.relative_misclosure - ref).max() < 1e-9
