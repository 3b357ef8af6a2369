"""sicp_register_joint / simpleicp_joint on the GPU: the reduction to the linearised pair path,
lock-step with the NumPy restatement (oracle/joint_oracle.py) on a ring of scans, the structure of
the problem (fixed clouds, unused clouds, shared roles, duplicated edges), a problem of 127 free
clouds, georeferenced coordinates, the failures, memory kinds, determinism and the side effects."""
import ctypes as C

import numpy as np
import pytest
import torch

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

from test_joint_host import _pair, ring

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _params(eng, max_iterations=30, min_planarity=0.3, min_change=1.0):
    lsq = eng.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
    return eng.run_params(min_planarity, min_change, max_iterations, lsq)


def _log(eng, out):
    return eng.batch_outputs(out)


@pytest.mark.parametrize("name,mod", [("dragon", -1.0), ("bunny", 1.0), ("multisensor", -1.0)])
def test_two_clouds_one_edge_equal_the_linearised_pair_path(eng, name, mod):
    X_fix, X_mov = _pair(name)
    x0 = np.array([0.01, -0.02, 0.015, 0.05, -0.03, 0.02])
    p = _params(eng)
    eng.set_option("variant", 1)
    try:
        pair = eng.register_pairs([X_fix, X_mov], [(0, 1)], 1000, 10, p, mod, observed=x0[None, :])
        po = _log(eng, pair)[0]
    finally:
        eng.set_option("variant", 0)
    H0 = np.stack([np.eye(4), J.rigid_from_x(x0)])
    H, out = eng.register_joint([X_fix, X_mov], [(0, 1)], [True, False], H0, 1000, 10, p, mod)
    jo = _log(eng, out)[0]
    a, b = pair[0], out[0]
    assert a.status == b.status == 0
    assert (a.iterations, a.converged) == (b.iterations, b.converged)
    assert np.abs(np.array(a.H) - np.array(b.H)).max() < 1e-9
    assert np.abs(np.array(a.x) - np.array(b.x)).max() < 1e-9
    assert np.abs(H[1] - np.array(b.H).reshape(4, 4)).max() < 1e-12
    assert np.array_equal(H[0], np.eye(4))
    rel = lambda u, v: abs(u - v) <= 1e-9 * max(abs(u), abs(v)) + 1e-15
    assert rel(a.mean_res, b.mean_res) and rel(a.std_res, b.std_res)
    for ra, rb in zip(po[2], jo[2]):
        assert ra.n_kept == rb.n_kept
        assert rel(ra.mean_res, rb.mean_res) and rel(ra.std_res, rb.std_res)
        assert rel(ra.median, rb.median) and rel(ra.mad, rb.mad)
    assert np.abs(po[1] - jo[1]).max() <= 1e-9 * np.abs(po[1]).max() + 1e-15


def _device_normals(eng, X, idx, k=10):
    eng.set_clouds(X, X[:10])
    eng.set_selected(idx)
    nx, ny, nz, pl = eng.estimate_normals(k)
    return np.column_stack((nx, ny, nz)), pl.copy()


def _lockstep(eng, scans, H0, edges, fixed, mod=1.0, max_iterations=30):
    p = _params(eng, max_iterations)
    is_fixed = np.zeros(len(scans), dtype=bool)
    is_fixed[list(fixed)] = True
    H, out = eng.register_joint(scans, edges, is_fixed, H0, 1000, 10, p, mod)
    logs = [o[2] for o in _log(eng, out)]
    # the oracle with the device's float32 normals of every edge's selection
    sel = J.simpleicp_joint(scans, edges, fixed=fixed, H0=H0, max_iterations=0, max_overlap_distance=mod)
    nrm = {e: _device_normals(eng, scans[a], sel.idx_fix[e]) for e, (a, _) in enumerate(edges)}
    ref = J.simpleicp_joint(scans, edges, fixed=fixed, H0=H0, max_iterations=max_iterations,
                            max_overlap_distance=mod, normals=nrm)
    return H, out, logs, ref


def test_ring_lockstep_with_the_oracle(eng):
    scans, truth, H0, edges = ring()
    H, out, logs, ref = _lockstep(eng, scans, H0, edges, (0,))
    assert all(o.iterations == len(ref.log) for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row]
    assert np.abs(H - ref.H).max() < 1e-9


def test_structure_fixed_clouds_unused_clouds_shared_roles_and_duplicates(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    # two fixed clouds (0 and 4), an unused cloud (None), cloud 2 fixed side of (2, 3) and movable
    # side of (1, 2), and edge (0, 1) twice
    clouds = list(scans[:6]) + [None]
    H0s = np.concatenate([H0[:6], np.eye(4)[None] * 2.0])
    E = np.array([(0, 1), (0, 1), (1, 2), (2, 3), (3, 4), (4, 5), (1, 3)])
    fixed = np.zeros(7, dtype=bool)
    fixed[[0, 4]] = True
    H, out = eng.register_joint(clouds, E, fixed, H0s, 1000, 10, p, 1.0)
    assert all(o.status == 0 for o in out)
    for c in (0, 4, 6):
        assert np.array_equal(H[c], H0s[c])
    nrm_ref = J.simpleicp_joint(clouds, E, fixed=(0, 4), H0=H0s, max_iterations=0, max_overlap_distance=1.0)
    nrm = {e: _device_normals(eng, clouds[a], nrm_ref.idx_fix[e]) for e, (a, _) in enumerate(E)}
    ref = J.simpleicp_joint(clouds, E, fixed=(0, 4), H0=H0s, max_iterations=30, max_overlap_distance=1.0,
                            normals=nrm)
    assert np.abs(H - ref.H).max() < 1e-9
    # determinism
    H2, out2 = eng.register_joint(clouds, E, fixed, H0s, 1000, 10, p, 1.0)
    assert np.array_equal(H, H2)
    assert all(bytes(a) == bytes(b) for a, b in zip(out, out2))


def test_memory_kinds_give_the_same_bits(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    fixed = np.zeros(len(scans), dtype=bool)
    fixed[0] = True
    H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0)
    pinned = [torch.from_numpy(s).pin_memory() for s in scans]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    for kind in (pinned, dev):
        H2, out2 = eng.register_joint(kind, edges, fixed, H0, 1000, 10, p, 1.0)
        assert np.array_equal(H, H2)
        assert all(bytes(a) == bytes(b) for a, b in zip(out, out2))


def test_failures_leave_h_out_and_clear_the_batch_outputs(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    far = scans[2] + 1000.0
    ok_H, ok = eng.register_joint(scans[:3], [(0, 1), (1, 2)], np.array([True, False, False]), H0[:3], 1000, 10, p,
                                  1.0)
    assert all(o.status == 0 for o in ok)
    # edge (1, 2) has no overlap and leaves the free cloud 2 without a path to a fixed cloud
    H_out = np.full((3, 4, 4), 7.0)
    rp = eng._register_params(1000, 10, p, 1.0, 0, -1.0)
    clouds = [scans[0], scans[1], far]
    ptrs = (C.c_void_p * 3)(*[c.ctypes.data for c in clouds])
    counts = (C.c_int64 * 3)(*[c.shape[0] for c in clouds])
    fix = np.array([0, 1], dtype=np.int32)
    mov = np.array([1, 2], dtype=np.int32)
    is_fixed = np.array([1, 0, 0], dtype=np.int32)
    out = (_capi.PairResult * 2)()
    i32p = C.POINTER(C.c_int32)
    rc = eng._lib.sicp_register_joint(eng._h, 3, ptrs, counts, 2, fix.ctypes.data_as(i32p), mov.ctypes.data_as(i32p),
                                      is_fixed.ctypes.data_as(i32p), None, C.byref(rp), H_out.ctypes.data, out, None)
    assert rc == _capi.SICP_ERR_NO_OVERLAP
    assert (H_out == 7.0).all()
    with pytest.raises(SicpError) as ei:
        eng.batch_outputs(ok)
    assert ei.value.code == _capi.SICP_ERR_STATE
    # an edge without overlap between two clouds that other edges anchor: only that edge fails.
    # Cloud 3 is the part of scan 7 at world x >= 28, 2 m beyond scan 0's end (x < 26): edge (0, 3)
    # has no overlap, while (2, 3) ties cloud 3 to scan 4 (x in [8, 34)) and so to cloud 0
    W7 = scans[7] @ truth[7][:3, :3].T + truth[7][:3, 3]
    tail = np.ascontiguousarray(scans[7][W7[:, 0] >= 28.0])
    c4 = [scans[0], scans[2], scans[4], tail]
    H04 = np.stack([H0[0], H0[2], H0[4], H0[7]])
    fx4 = np.array([True, False, False, False])
    with pytest.raises(SicpError) as ei:  # without (1, 2), (2, 3) cloud 3 hangs on (0, 3) alone
        eng.register_joint(c4, [(0, 1), (0, 3)], fx4, H04, 1000, 10, p, 1.0)
    assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
    H, out2 = eng.register_joint(c4, [(0, 1), (1, 2), (2, 3), (0, 3)], fx4, H04, 1000, 10, p, 1.0)
    assert [o.status for o in out2] == [0, 0, 0, _capi.SICP_ERR_NO_OVERLAP]
    assert np.abs(H[3] - truth[7]).max() < 1e-2
    # two clouds sampled from one plane: the joint matrix is singular
    rng = np.random.default_rng(3)
    P = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
    Q = np.column_stack([rng.uniform(0, 10, (5000, 2)), np.zeros(5000)])
    with pytest.raises(SicpError) as ei:
        eng.register_joint([P, Q], [(0, 1)], np.array([True, False]), None, 1000, 10, p, 1.0)
    assert ei.value.code == _capi.SICP_ERR_SINGULAR
    with pytest.raises(SicpError) as ei:
        eng.batch_outputs(out2)
    assert ei.value.code == _capi.SICP_ERR_STATE


def _one_pair_state(eng):
    res = np.empty(4096)
    n = C.c_int64(0)
    eng._check(eng._lib.sicp_get_residuals(eng._h, res.ctypes.data, res.size, C.byref(n)))
    return eng.get_transform(), res[:n.value].copy()


def test_side_effects_map_one_pair_state_and_batch_outputs(eng):
    scans, truth, H0, edges = ring()
    p = _params(eng)
    X_fix, X_mov = _pair("bunny")
    eng.register_fused(X_fix, X_mov, 500, 10, 1.0, p)
    before = _one_pair_state(eng)
    eng.set_map(scans[0])
    fixed = np.zeros(len(scans), dtype=bool)
    fixed[0] = True
    H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0)
    assert np.array_equal(eng.get_map(), scans[0])
    after = _one_pair_state(eng)
    assert np.array_equal(before[0], after[0]) and np.array_equal(before[1], after[1])
    eng.set_map(None)
    # the batch outputs: cloud b moved by the final T_a^-1 T_b, that transform, the final residuals
    H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0)
    for (a, b), o, (X_t, resid, log, T) in zip(edges, out, eng.batch_outputs(out)):
        R = np.array(o.H).reshape(4, 4)
        assert np.array_equal(T.reshape(4, 4), R)
        assert np.abs(R - np.linalg.inv(H[a]) @ H[b]).max() < 1e-12
        assert np.abs(X_t - (scans[b] @ R[:3, :3].T + R[:3, 3])).max() < 1e-12
        assert resid.size == o.n_kept == log[o.iterations - 1].n_kept
        assert abs(resid.mean() - o.mean_res) < 1e-12 and abs(np.std(resid, ddof=1) - o.std_res) < 1e-12
        assert log[o.iterations - 1].mean_res == o.mean_res and log[o.iterations - 1].std_res == o.std_res


def test_georeferenced_first_iteration_is_translation_invariant(eng):
    """Every cloud and the world translated to UTM coordinates, one iteration.  The selection, the
    rejection and the centred solve do not depend on the translation: equal kept counts, and the
    same order statistics, residual statistics and rotation increments to rounding.  (Only the
    translations of the origin-based update dH(x_c) differ, by about |alpha|^2 D: DESIGN.md §6.9.)
    The normals take the canonical sign: the eigen-solver's sign follows the covariance's last
    bits, which the translation changes, and a flipped normal moves the median of the distances."""
    scans, truth, H0, edges = ring()
    utm = np.array([4.5e5, 5.4e6, 300.0])
    S = np.eye(4)
    S[:3, 3] = utm
    p = _params(eng, max_iterations=1)
    fixed = np.zeros(len(scans), dtype=bool)
    fixed[0] = True
    H0_u = np.array([S @ h @ np.linalg.inv(S) for h in H0])
    eng.set_option("sign_mode", 1)
    try:
        H, out = eng.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0)
        logs = [o[2][0] for o in _log(eng, out)]
        H_u, out_u = eng.register_joint([s + utm for s in scans], edges, fixed, H0_u, 1000, 10, p, 1.0)
        logs_u = [o[2][0] for o in _log(eng, out_u)]
    finally:
        eng.set_option("sign_mode", 0)
    # distances carry the rounding of 5.4e6 m coordinates (ulp 9.3e-10 m) and of the float32 normals
    for r, ru in zip(logs, logs_u):
        assert r.n_kept == ru.n_kept
        for f in ("median", "mad", "mean_res", "std_res"):
            assert abs(getattr(r, f) - getattr(ru, f)) < 1e-7, (f, getattr(r, f), getattr(ru, f))
        assert np.abs(np.array(r.x[:3]) - np.array(ru.x[:3])).max() < 1e-7
    assert np.abs(H[:, :3, :3] - H_u[:, :3, :3]).max() < 1e-7


def strip(n_scans, n_points, n_edges, seed=11):
    """n_scans clouds of the C3 surface along a strip (x in [2 i, 2 i + 26), y in [0, 30)), each in
    its own frame (centred on its patch, turned by up to 1 degree, moved by up to 0.3 m), start
    poses perturbed in that frame by 0.3 degrees and 5 cm, and the edges (i, i + 1), (i, i + 2) and
    random closures (i, j), 3 <= j - i <= 10, n_edges in all."""
    rng = np.random.default_rng(seed)
    scans, truth, H0 = [], [], []
    for i in range(n_scans):
        x = rng.uniform(2.0 * i, 2.0 * i + 26.0, n_points)
        y = rng.uniform(0.0, 30.0, n_points)
        z = 0.05 * x + 0.03 * y + 2 * np.sin(2 * np.pi * x / 25) * np.cos(2 * np.pi * y / 40)
        P = np.column_stack((x, y, z + rng.normal(0, 0.01, n_points)))
        T = J.rigid_from_x(np.concatenate((np.deg2rad(rng.uniform(-1, 1, 3)), rng.uniform(-0.3, 0.3, 3))))
        T[:3, 3] += (2.0 * i + 13.0, 15.0, 0.0)
        Ti = np.linalg.inv(T)
        scans.append(np.ascontiguousarray(P @ Ti[:3, :3].T + Ti[:3, 3]))
        truth.append(T)
        dH = J.rigid_from_x(np.concatenate((np.deg2rad(rng.normal(0, 0.3, 3)), rng.normal(0, 0.05, 3))))
        H0.append(T if i == 0 else T @ dH)
    edges = [(i, i + 1) for i in range(n_scans - 1)] + [(i, i + 2) for i in range(n_scans - 2)]
    seen = set(edges)
    while len(edges) < n_edges:
        i = int(rng.integers(0, n_scans - 3))
        j = i + int(rng.integers(3, 11))
        if j < n_scans and (i, j) not in seen:
            seen.add((i, j))
            edges.append((i, j))
    return scans, np.array(truth), np.array(H0), np.array(edges)


def test_size_128_clouds_lockstep_with_the_oracle(eng):
    """128 clouds of 50 000 points, 400 edges, F = 127: the joint matrix has 762 unknowns, 24 tile
    rows, so the panel and trailing tiles of the Cholesky are spread over many blocks."""
    scans, truth, H0, edges = strip(128, 50_000, 400)
    H, out, logs, ref = _lockstep(eng, scans, H0, edges, (0,), max_iterations=20)
    assert all(o.status == 0 and o.iterations == len(ref.log) for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row], it
    assert np.abs(H - ref.H).max() < 1e-9


def test_simpleicp_joint_end_to_end():
    scans, truth, H0, edges = ring()
    res = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0, full_output=True)
    assert res.H.shape == (8, 4, 4) and res.table.shape == (len(edges), 20)
    assert np.abs(res.H - truth).max() < 1e-2
    assert res.iterations >= 2 and len(res.results) == len(edges)
    for (a, b), row in zip(edges, res.table):
        assert np.abs(row[:16].reshape(4, 4) - np.linalg.inv(res.H[a]) @ res.H[b]).max() < 1e-9
