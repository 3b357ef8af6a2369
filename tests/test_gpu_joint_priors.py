"""sicp_register_joint_priors / simpleicp_joint(prior_poses=, prior_weights=) on the GPU (DESIGN.md
§6.12): the bits of sicp_register_joint without priors, lock-step with the NumPy restatement
(joint_prior_oracle.py) on the ring and on 127 free clouds under both solves, a huge weight
against a fixed cloud, long strips held by priors alone or with one fixed cloud, georeferenced
coordinates, the covariances against the NumPy rule (joint_prior_cov_rule.py), anchoring over the
edges with overlap, the C argument checks and determinism."""
import ctypes as C
import json

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

import joint_prior_cov_rule as JP
import joint_prior_oracle as JPO
from test_gpu_joint import _device_normals, _params, strip
from joint_cov_rule import lever
from test_gpu_joint_cov import _sig
from test_joint_host import ring

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _noisy(truth, seed, rot_deg, pos_m):
    """truth moved by seeded rotations of rot_deg and translations of pos_m (standard deviations)."""
    rng = np.random.default_rng(seed)
    R = Rotation.from_rotvec(np.deg2rad(rng.normal(0, rot_deg, (len(truth), 3)))).as_matrix()
    P = np.array(truth, dtype=np.float64)
    P[:, :3, :3] = R @ P[:, :3, :3]
    P[:, :3, 3] += rng.normal(0, pos_m, (len(truth), 3))
    return P


def _ring_priors(truth, anchor0=False):
    """Full priors on clouds 2 and 5 (and 0 with anchor0), position only on 3 and 7; truth plus
    0.05 degrees and 2 cm of seeded noise; weights for rows of 5 mm."""
    P = _noisy(truth, 21, 0.05, 0.02)
    W = np.zeros((len(truth), 6))
    full = [0.005 ** 2 / np.deg2rad(0.05) ** 2] * 3 + [0.005 ** 2 / 0.02 ** 2] * 3
    W[[2, 5]] = full
    W[[3, 7], 3:] = full[3:]
    if anchor0:
        W[0] = full
    return P, W


def _joint(eng, solver, scans, edges, fixed, H0, P=None, W=None, mod=1.0, max_iterations=30):
    is_fixed = np.zeros(len(scans), dtype=bool)
    is_fixed[list(fixed)] = True
    eng.set_option("joint_solver", solver)
    try:
        return eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, _params(eng, max_iterations), mod, P, W)
    finally:
        eng.set_option("joint_solver", 0)


def _register_joint_without_priors(eng, scans, edges, fixed, H0, mod=1.0):
    """sicp_register_joint itself, through ctypes as the binding called it before the priors."""
    fix = np.ascontiguousarray(np.asarray(edges)[:, 0], dtype=np.int32)
    mov = np.ascontiguousarray(np.asarray(edges)[:, 1], dtype=np.int32)
    keep, ptrs, counts = _capi._clouds_arg(scans, allow_none=True)
    is_fixed = np.zeros(len(scans), dtype=np.int32)
    is_fixed[list(fixed)] = 1
    p = _params(eng)
    rp = eng._register_params(1000, 10, p, mod, 0, -1.0)
    H = np.zeros((len(scans), 4, 4))
    i32p = C.POINTER(C.c_int32)
    out = eng._batched(eng._lib.sicp_register_joint, p, counts, mov, len(counts), ptrs, counts, len(fix),
                       fix.ctypes.data_as(i32p), mov.ctypes.data_as(i32p), is_fixed.ctypes.data_as(i32p),
                       np.ascontiguousarray(H0).ctypes.data, C.byref(rp), H.ctypes.data)
    return H, out


def _everything(eng, H, out, dense):
    """The bits of one call: poses, records, batch outputs and (dense) the covariances."""
    blobs = [H.tobytes()] + [bytes(o) for o in out]
    for X, r, log, T in eng.batch_outputs(out):
        blobs += [X.tobytes(), r.tobytes(), b"".join(bytes(x) for x in log), T.tobytes()]
    if dense:
        cov, ecov, s0 = eng.joint_covariances(len(H), len(out))
        blobs += [cov.tobytes(), ecov.tobytes(), np.float64(s0).tobytes()]
    return blobs


@pytest.mark.parametrize("solver", [0, 1])
def test_without_priors_the_bits_of_sicp_register_joint(eng, solver):
    scans, truth, H0, edges = ring()
    dense = solver == 0
    is_fixed = np.zeros(8, dtype=bool)
    is_fixed[0] = True
    P = np.full((8, 4, 4), np.nan)
    W = np.zeros((8, 6))
    W[0] = 1.0  # a fixed cloud's prior is not read
    eng.set_option("joint_solver", solver)
    try:
        ref = _everything(eng, *_register_joint_without_priors(eng, scans, edges, (0,), H0), dense)
        null = _everything(eng, *eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, _params(eng), 1.0), dense)
        zero = _everything(eng, *eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, _params(eng), 1.0, P, W),
                           dense)
    finally:
        eng.set_option("joint_solver", 0)
    assert null == ref and zero == ref
    # simpleicp_joint with all-zero weights against simpleicp_joint without priors
    kw = dict(fixed=(0,), H0=H0, max_overlap_distance=1.0, covariances=solver == 0,
              solver="dense" if solver == 0 else "sparse")
    a = sb.simpleicp_joint(scans, edges, **kw)
    b = sb.simpleicp_joint(scans, edges, prior_poses=np.full((8, 4, 4), np.nan), prior_weights=np.zeros((8, 6)), **kw)
    assert np.array_equal(a.H, b.H) and np.array_equal(a.table, b.table, equal_nan=True)
    assert (a.iterations, a.converged) == (b.iterations, b.converged)
    if solver == 0:
        assert np.array_equal(a.cov, b.cov, equal_nan=True) and np.array_equal(a.edge_cov, b.edge_cov)
        assert a.s0 == b.s0


def _lockstep(eng, solver, scans, H0, edges, fixed, P, W, max_iterations=30):
    H, out = _joint(eng, solver, scans, edges, fixed, H0, P, W, max_iterations=max_iterations)
    logs = [o[2] for o in eng.batch_outputs(out)]
    sel = J.simpleicp_joint(scans, edges, fixed=fixed, H0=H0, max_iterations=0, max_overlap_distance=1.0)
    nrm = {e: _device_normals(eng, scans[a], sel.idx_fix[e]) for e, (a, _) in enumerate(edges)}
    ref = JPO.simpleicp_joint(scans, edges, fixed=fixed, H0=H0, max_iterations=max_iterations,
                              max_overlap_distance=1.0, normals=nrm, prior_poses=P, prior_weights=W)
    return H, out, logs, ref, nrm


def _assert_lockstep(H, out, logs, ref, tol=1e-9):
    assert all(o.status == 0 and o.iterations == len(ref.log) for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row], it
    assert np.abs(H - ref.H).max() < tol, np.abs(H - ref.H).max()


@pytest.mark.parametrize("solver", [0, 1])
@pytest.mark.parametrize("fixed", [(0,), ()])
def test_ring_lockstep_with_the_oracle(eng, solver, fixed):
    scans, truth, H0, edges = ring()
    P, W = _ring_priors(truth, anchor0=not fixed)
    H, out, logs, ref, _ = _lockstep(eng, solver, scans, H0, edges, fixed, P, W)
    _assert_lockstep(H, out, logs, ref)
    assert ref.converged and np.abs(H - truth).max() < 1e-2


def test_size_128_clouds_lockstep_with_the_oracle(eng):
    """F = 127 with a prior on every free cloud (truth plus 0.03 degrees and 3 cm); both solves in
    lock-step with one oracle run."""
    scans, truth, H0, edges = strip(128, 50_000, 400)
    P = _noisy(truth, 31, 0.03, 0.03)
    W = np.tile([0.01 ** 2 / np.deg2rad(0.03) ** 2] * 3 + [0.01 ** 2 / 0.03 ** 2] * 3, (128, 1))
    H, out, logs, ref, nrm = _lockstep(eng, 0, scans, H0, edges, (0,), P, W, max_iterations=20)
    _assert_lockstep(H, out, logs, ref)
    Hs, outs = _joint(eng, 1, scans, edges, (0,), H0, P, W, max_iterations=20)
    _assert_lockstep(Hs, outs, [o[2] for o in eng.batch_outputs(outs)], ref)


@pytest.mark.parametrize("solver", [0, 1])
def test_huge_weight_equals_a_fixed_cloud(eng, solver):
    """As test_joint_prior_host.test_oracle_huge_weight_equals_a_fixed_cloud on the device: weights
    1e12 on cloud 3 with P_3 = H0[3] against cloud 3 fixed; the bound 1e3 |N| / w (|N| < 1e6) is
    derived there."""
    scans, truth, H0, edges = ring()
    Hf, outf = _joint(eng, solver, scans, edges, (0, 3), H0)
    logf = [o[2] for o in eng.batch_outputs(outf)]
    W = np.zeros((8, 6))
    W[3] = 1e12
    Hp, outp = _joint(eng, solver, scans, edges, (0,), H0, H0, W)
    logp = [o[2] for o in eng.batch_outputs(outp)]
    assert [(o.status, o.iterations) for o in outf] == [(o.status, o.iterations) for o in outp]
    for lf, lp in zip(logf, logp):
        assert [r.n_kept for r in lf[:outf[0].iterations]] == [r.n_kept for r in lp[:outf[0].iterations]]
    assert np.abs(Hf - Hp).max() < 1e3 * 1e6 / 1e12


def _rot_err(H, truth):
    return np.linalg.norm(Rotation.from_matrix(H[:, :3, :3] @ np.transpose(truth[:, :3, :3], (0, 2, 1))).as_rotvec(),
                          axis=1)


# The long strips: a prior on every cloud, truth plus 0.02 degrees and 3 cm of seeded noise, with the
# weights of rows of 1 cm, and the call starts from the priors, as one with GNSS/INS poses would.
# (The generator's own start poses are perturbed by 0.3 degrees about each cloud's frame origin,
# which lies up to 410 m below its data at the far end of 4096 clouds: those clouds start a median
# 2.5 m off, beyond the 1 m overlap filter.)  RMS errors of the final poses against the truth must be
# below those of the priors (5.1-5.3 cm, 0.034 degrees) and below 3.5 cm and 0.025 degrees: about 1.5
# times the largest measured on an H100, 2.2 cm and 0.0167 degrees (DESIGN.md §6.12).
LONG = {"1024": (1024, 3_000), "2048": (2048, 6_400), "4096": (4096, 12_800)}


@pytest.mark.parametrize("fixed", [(0,), ()])
@pytest.mark.parametrize("size", list(LONG))
def test_long_strip_held_by_priors(eng, size, fixed):
    n, n_edges = LONG[size]
    scans, truth, H0, edges = strip(n, 5_000, n_edges, seed=12)
    P = _noisy(truth, 41, 0.02, 0.03)
    W = np.tile([0.01 ** 2 / np.deg2rad(0.02) ** 2] * 3 + [0.01 ** 2 / 0.03 ** 2] * 3, (n, 1))
    import time

    t0 = time.perf_counter()
    H, out = _joint(eng, 1, scans, edges, fixed, P, P, W)
    ms = (time.perf_counter() - t0) * 1e3
    statuses = {int(k): int(v) for k, v in zip(*np.unique([o.status for o in out], return_counts=True))}
    free = np.ones(n, dtype=bool)
    free[list(fixed)] = False
    rms = lambda v: float(np.sqrt(np.mean(v[free] ** 2)))
    pos, rot = rms(np.linalg.norm(H[:, :3, 3] - truth[:, :3, 3], axis=1)), rms(_rot_err(H, truth))
    pos_p, rot_p = rms(np.linalg.norm(P[:, :3, 3] - truth[:, :3, 3], axis=1)), rms(_rot_err(P, truth))
    line = dict(size=n, fixed=list(fixed), edge_statuses=statuses, iterations=int(out[0].iterations),
                converged=bool(out[0].converged),
                call_ms=round(ms, 1), pos_rms_m=pos, rot_rms_deg=float(np.rad2deg(rot)), prior_pos_rms_m=pos_p,
                prior_rot_rms_deg=float(np.rad2deg(rot_p)), max_pos_m=float(np.abs(H[:, :3, 3] - truth[:, :3, 3]).max()))
    print("long strip", json.dumps(line))
    assert pos < pos_p and rot < rot_p
    assert pos < 0.035 and np.rad2deg(rot) < 0.025


def test_georeferenced_first_iteration_is_translation_invariant(eng):
    """test_gpu_joint's UTM test with the ring's priors: the world moved to UTM coordinates (start
    poses and priors S H; each cloud keeps its frame, so the priors observe the same origins).
    Equal kept counts, the same statistics and rotations to that test's tolerances after one
    iteration (the translations of the origin-based update differ by about |alpha|^2 D, as there)."""
    scans, truth, H0, edges = ring()
    P, W = _ring_priors(truth)
    utm = np.array([4.5e5, 5.4e6, 300.0])
    S = np.eye(4)
    S[:3, 3] = utm
    P_u = np.array([S @ h for h in P])  # the world moved, every cloud in its own frame as before
    H0_u = np.array([S @ h for h in H0])
    eng.set_option("sign_mode", 1)
    try:
        H, out = _joint(eng, 0, scans, edges, (0,), H0, P, W, max_iterations=1)
        logs = [o[2][0] for o in eng.batch_outputs(out)]
        H_u, out_u = _joint(eng, 0, scans, edges, (0,), H0_u, P_u, W, max_iterations=1)
        logs_u = [o[2][0] for o in eng.batch_outputs(out_u)]
    finally:
        eng.set_option("sign_mode", 0)
    for r, ru in zip(logs, logs_u):
        assert r.n_kept == ru.n_kept
        for f in ("median", "mad", "mean_res", "std_res"):
            assert abs(getattr(r, f) - getattr(ru, f)) < 1e-7, (f, getattr(r, f), getattr(ru, f))
        assert np.abs(np.array(r.x[:3]) - np.array(ru.x[:3])).max() < 1e-7
    assert np.abs(H[:, :3, :3] - H_u[:, :3, :3]).max() < 1e-7


@pytest.mark.parametrize("problem", ["ring", "strip127"])
def test_covariances_with_priors_against_the_rule(eng, problem):
    if problem == "ring":
        scans, truth, H0, edges = ring()
        P, W = _ring_priors(truth)
        iters = 30
    else:
        scans, truth, H0, edges = strip(128, 50_000, 400)
        P = _noisy(truth, 31, 0.03, 0.03)
        W = np.tile([0.01 ** 2 / np.deg2rad(0.03) ** 2] * 3 + [0.01 ** 2 / 0.03 ** 2] * 3, (128, 1))
        W[5:20, :3] = 0.0  # position only on some
        iters = 20
    H, out, logs, ref, nrm = _lockstep(eng, 0, scans, H0, edges, (0,), P, W, max_iterations=iters)
    _assert_lockstep(H, out, logs, ref)
    cov, ecov, s0 = eng.joint_covariances(len(scans), len(edges))
    fi = JP.final_iteration(scans, edges, ref, fixed=(0,), H0=H0, prior_poses=P, prior_weights=W,
                            max_overlap_distance=1.0)
    free = list(fi.slot)
    assert abs(s0 - fi.s0) <= 1e-12 * fi.s0, (s0, fi.s0)
    ku = np.linalg.cond(fi.N) * np.finfo(np.float64).eps / 2
    d_sig = np.abs(_sig(cov[free]) / _sig(fi.cov[free]) - 1).max()
    print(f"joint covariances with priors ({problem}): s0 {s0:.6e} rel {abs(s0 / fi.s0 - 1):.2e}, "
          f"kappa u {ku:.1e}, sigma rel {d_sig:.2e}")
    assert d_sig < max(10 * ku, 1e-12), (d_sig, ku)
    if problem != "ring":
        return
    # the priors never grow the unscaled block C_c / s0^2 = J_c (N^-1)_cc J_c^T: the device's against
    # the same final iteration's N without the prior blocks (s0 itself may rise)
    N0 = fi.N.copy()
    for pt in fi.priors:
        N0[6 * pt.slot:6 * pt.slot + 6, 6 * pt.slot:6 * pt.slot + 6] -= pt.N
    N0inv = np.linalg.inv(N0)
    for c, k in fi.slot.items():
        Jc = lever(np.eye(3), fi.H[c][:3, 3])
        d0 = np.diagonal(Jc @ N0inv[6 * k:6 * k + 6, 6 * k:6 * k + 6] @ Jc.T)
        d1 = np.diagonal(cov[c]) / s0 ** 2
        assert (d1 <= d0 * (1 + 10 * ku + 1e-12)).all(), (c, d1, d0)
        if c in (2, 5):  # the full priors shrink their own clouds' blocks (by about 1 % here)
            assert (d1 < d0 * (1 - 100 * ku)).all(), (c, d1, d0)


def _c4(truth, scans, H0):
    W7 = scans[7] @ truth[7][:3, :3].T + truth[7][:3, 3]
    tail = np.ascontiguousarray(scans[7][W7[:, 0] >= 28.0])
    return [scans[0], scans[2], scans[4], tail], np.stack([H0[0], H0[2], H0[4], H0[7]])


@pytest.mark.parametrize("solver", [0, 1])
def test_no_overlap_anchoring(eng, solver):
    """test_gpu_joint's cloud 3, tied to the rest only by an edge without overlap: the call fails
    with SICP_ERR_NO_OVERLAP without priors, as before; a full prior on cloud 3 anchors it, the edge
    alone fails, and the cloud goes to its prior's pose."""
    scans, truth, H0, edges = ring()
    c4, H04 = _c4(truth, scans, H0)
    with pytest.raises(SicpError) as ei:
        _joint(eng, solver, c4, [(0, 1), (0, 3)], (0,), H04)
    assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
    P = np.stack([H04[0]] + [np.eye(4)] * 2 + [truth[7]])
    W = np.zeros((4, 6))
    W[3] = 1.0
    with pytest.raises(SicpError) as ei:  # position and rotation, but not all six: no anchor
        W2 = W.copy()
        W2[3, 5] = 0.0
        _joint(eng, solver, c4, [(0, 1), (0, 3)], (0,), H04, P, W2)
    assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
    H, out = _joint(eng, solver, c4, [(0, 1), (0, 3)], (0,), H04, P, W)
    assert [o.status for o in out] == [0, _capi.SICP_ERR_NO_OVERLAP]
    assert np.abs(H[3] - truth[7]).max() < 1e-6
    # no edge with overlap at all, fixed=(): full priors hold both free clouds
    W[0] = 1.0
    H, out = _joint(eng, solver, c4, [(0, 3)], (), H04, P, W)
    assert out[0].status == _capi.SICP_ERR_NO_OVERLAP
    assert np.abs(H[0] - H04[0]).max() < 1e-12 and np.abs(H[3] - truth[7]).max() < 1e-6


def test_c_argument_checks(eng):
    scans, truth, H0, edges = ring()
    is_fixed = np.zeros(8, dtype=bool)
    is_fixed[0] = True
    p = _params(eng)
    P, W = _ring_priors(truth)

    def call(P, W, fixed=is_fixed):
        return eng.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0, P, W)

    def refused(P, W, msg, fixed=is_fixed):
        with pytest.raises(SicpError) as ei:
            call(P, W, fixed)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG and msg in str(ei.value), str(ei.value)

    refused(P, None, "both")
    refused(None, W, "both")
    for v in (-1.0, np.nan, np.inf):
        W2 = W.copy()
        W2[6, 1] = v
        refused(P, W2, "negative or not finite")
    P2 = P.copy()
    P2[2, 1, 3] = np.nan
    refused(P2, W, "prior_H[2] has non-finite")
    P2 = P.copy()
    P2[2, :3, :3] *= 1.0 + 1e-5
    refused(P2, W, "orthonormal")
    P2 = P.copy()
    P2[2, 3, 2] = 1.0
    refused(P2, W, "bottom row")
    W3 = W.copy()
    W3[[2, 5], :3] = 0.0  # position only everywhere: no anchor
    refused(P, W3, "without a fixed cloud", fixed=np.zeros(8, dtype=bool))
    Hf, outf = call(P, W, fixed=np.zeros(8, dtype=bool))  # the full priors of 2 and 5 anchor the ring
    assert all(o.status == 0 for o in outf)
    # not read: a fixed cloud's, an all-zero prior's
    P2 = P.copy()
    P2[[0, 1]] = np.nan
    W2 = W.copy()
    W2[0] = 5.0
    H, out = call(P2, W2)
    assert all(o.status == 0 for o in out)
    H2, out2 = call(P, W)
    assert np.array_equal(H, H2)


@pytest.mark.parametrize("solver", [0, 1])
def test_two_calls_give_the_same_bits(eng, solver):
    scans, truth, H0, edges = ring()
    P, W = _ring_priors(truth, anchor0=True)
    a = _everything(eng, *_joint(eng, solver, scans, edges, (), H0, P, W), solver == 0)
    b = _everything(eng, *_joint(eng, solver, scans, edges, (), H0, P, W), solver == 0)
    assert a == b


def test_simpleicp_joint_with_priors_end_to_end():
    """The quick-start call: fixed=() and GNSS-like priors on every cloud, both solvers and the
    covariances."""
    scans, truth, H0, edges = ring()
    P = _noisy(truth, 51, 0.05, 0.02)
    W = np.tile([0.005 ** 2 / np.deg2rad(0.05) ** 2] * 3 + [0.005 ** 2 / 0.02 ** 2] * 3, (8, 1))
    d = sb.simpleicp_joint(scans, edges, fixed=(), H0=H0, prior_poses=P, prior_weights=W, max_overlap_distance=1.0,
                           covariances=True)
    s = sb.simpleicp_joint(scans, edges, fixed=(), H0=H0, prior_poses=P, prior_weights=W, max_overlap_distance=1.0,
                           solver="sparse")
    assert np.abs(d.H - s.H).max() < 1e-9
    assert np.abs(d.H - truth).max() < 2e-2
    assert np.isfinite(d.s0) and (np.einsum("cii->ci", d.cov) > 0).all()
