"""Host-side tests of the joint (multi-scan) registration: the NumPy restatement
(oracle/joint_oracle.py) against the pair variant it reduces to and against ground truth, the
argument checks of simpleicp_joint, and the C ABI declaration of sicp_register_joint."""
import re
from pathlib import Path

import numpy as np
import pytest

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from oracle import linearized_oracle as L
from oracle import simpleicp_oracle as O
from simpleicp_b200 import _capi

REPO = Path(__file__).resolve().parents[1]
GOLDEN = REPO / "tests" / "golden"


def _pair(name):
    z = np.load(GOLDEN / f"data_{name}.npz")
    s = float(z["scale"])
    return z["fix"] / s, z["mov"] / s


@pytest.mark.parametrize("name,kw", [("dragon", {}), ("bunny", {"max_overlap_distance": 1.0})])
def test_two_clouds_one_edge_reduce_to_the_linearised_pair(name, kw):
    X_fix, X_mov = _pair(name)
    ref = L.simpleicp_linearized(X_fix, X_mov, compose="pre", keep_arrays=True, max_iterations=30, **kw)
    res = J.simpleicp_joint([X_fix, X_mov], [(0, 1)], fixed=(0,), max_iterations=30,
                            normals={0: (ref.normals, ref.planarity)}, **kw)
    assert len(res.log) == len(ref.iterations) and res.converged == ref.converged
    for it, r in zip(res.log, ref.iterations):
        e = it[0]
        assert np.array_equal(e.keep, r.keep)
        assert e.n_kept == r.n_kept
        assert abs(e.mean - r.mean) <= 1e-12 + 1e-9 * abs(r.mean)
        assert abs(e.std - r.std) <= 1e-12 + 1e-9 * abs(r.std)
    assert np.abs(res.H[1] - ref.T).max() < 1e-12
    assert np.array_equal(res.H[0], np.eye(4))


def ring(n=8, seed=90_000, shift=(0.0, 0.0, 0.0), noise=0.005):
    """n scans of one 40 m surface, scan i over x in [2 i, 2 i + 26) seen from its true pose
    (world <- scan) with `noise` m of Gaussian noise per coordinate, the true poses, noisy start poses (cloud 0 at its true pose) and the edges
    (i, i + 1), (i, i + 2) and the loop closure (n - 1, 0).  `shift` translates the world."""
    rng = np.random.default_rng(seed)
    S = O.surface(60_000, seed, extent=40.0)
    scans, truth, H0 = [], [], []
    for i in range(n):
        part = S[(S[:, 0] >= 2.0 * i) & (S[:, 0] < 2.0 * i + 26.0)]
        x = np.concatenate((np.deg2rad(rng.uniform(-1, 1, 3)), rng.uniform(-0.3, 0.3, 3)))
        T = J.rigid_from_x(x)
        T[:3, 3] += np.asarray(shift)
        seen = O.transform_by_H(part + np.asarray(shift), np.linalg.inv(T)) + rng.normal(0, noise, part.shape)
        scans.append(np.ascontiguousarray(seen))
        truth.append(T)
        dx = np.concatenate((np.deg2rad(rng.normal(0, 0.3, 3)), rng.normal(0, 0.05, 3)))
        H0.append(T if i == 0 else J.rigid_from_x(dx) @ T)
    edges = [(i, i + 1) for i in range(n - 1)] + [(i, i + 2) for i in range(n - 2)] + [(n - 1, 0)]
    return scans, np.array(truth), np.array(H0), np.array(edges)


def pose_error(H, truth):
    return max(np.abs(H[i] - truth[i]).max() for i in range(len(truth)))


def test_ring_joint_beats_chained_pairs_and_closes_the_loop():
    scans, truth, H0, edges = ring()
    res = J.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    # chaining the pairwise linearised results along (i, i + 1)
    chain = [truth[0]]
    for i in range(len(scans) - 1):
        R0 = np.linalg.inv(H0[i]) @ H0[i + 1]
        X = O.transform_by_H(scans[i + 1], R0)
        r = L.simpleicp_linearized(scans[i], X, compose="pre", max_iterations=30, max_overlap_distance=1.0)
        chain.append(chain[-1] @ r.T @ R0)
    chain = np.array(chain)
    assert pose_error(res.H, truth) < pose_error(chain, truth)
    loop = lambda H: np.abs(np.linalg.inv(H[-1]) @ H[0] - np.linalg.inv(truth[-1]) @ truth[0]).max()
    assert loop(res.H) < loop(chain)
    assert pose_error(res.H, truth) < 1e-2


def test_oracle_sparse_solve_equals_its_dense_solve_on_the_ring():
    """solver="sparse" (scipy.sparse.linalg.spsolve of the same blocks) against the dense path:
    the same iterations and kept counts, the poses within 1e-12 (measured 3.0e-15)."""
    scans, truth, H0, edges = ring()
    kw = dict(fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    dense = J.simpleicp_joint(scans, edges, **kw)
    sparse = J.simpleicp_joint(scans, edges, solver="sparse", **kw)
    assert [[e.n_kept for e in r] for r in dense.log] == [[e.n_kept for e in r] for r in sparse.log]
    assert sparse.converged == dense.converged
    assert np.abs(sparse.H - dense.H).max() < 1e-12


def test_oracle_sparse_solve_equals_its_dense_solve_on_the_128_cloud_strip():
    """The strip of tests/test_gpu_joint.py, 128 clouds of 5 000 points, 400 edges, three
    iterations.  The oracle's unknowns are about the world origin, so its matrix is ill-conditioned
    on a 270 m strip and the two solves of the first iteration part by 8.4e-9 in the poses; the
    iterations pull both to the same poses, 3.3e-11 apart after three (bound 1e-10).  Every kept
    count exact."""
    from test_gpu_joint import strip

    scans, truth, H0, edges = strip(128, 5_000, 400)
    kw = dict(fixed=(0,), H0=H0, max_iterations=3, max_overlap_distance=1.0)
    dense = J.simpleicp_joint(scans, edges, **kw)
    sparse = J.simpleicp_joint(scans, edges, solver="sparse", **kw)
    assert [[e.n_kept for e in r] for r in dense.log] == [[e.n_kept for e in r] for r in sparse.log]
    assert np.abs(sparse.H - dense.H).max() < 1e-10


def test_first_iteration_sums_are_the_first_iterations_rows():
    """first_iteration_sums against the rows simpleicp_joint solves: the kept counts of its first
    iteration, and the first increments from a dense solve assembled from the sums."""
    scans, truth, H0, edges = ring()
    ref = J.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_iterations=1, max_overlap_distance=1.0)
    s = J.first_iteration_sums(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    assert list(s.n_kept) == [e.n_kept for e in ref.log[0]] and s.free == list(range(1, 8))
    F = len(s.free)
    M, g = np.zeros((6 * F, 6 * F)), np.zeros(6 * F)
    for (a, b), N, h, Ta in zip(edges, s.N, s.g, s.T_a):
        Ad = J.ad_world_to_frame(Ta)
        for c, sgn in ((a, -1.0), (b, 1.0)):
            if c > 0:
                i = 6 * (c - 1)
                g[i:i + 6] += sgn * Ad.T @ h
                for d, sgn2 in ((a, -1.0), (b, 1.0)):
                    if d > 0:
                        j = 6 * (d - 1)
                        M[i:i + 6, j:j + 6] += sgn * sgn2 * Ad.T @ N @ Ad
    x = np.linalg.solve(M, g)
    for c in range(1, 8):
        assert np.abs(J.rigid_from_x(x[6 * (c - 1):6 * c]) @ H0[c] - ref.H[c]).max() < 1e-12


def test_an_edge_without_overlap_has_no_rows_and_takes_no_part():
    """Edge (1, 2) to a fixed cloud 1 km away has an empty selection under max_overlap_distance:
    kept count 0 in every iteration and in first_iteration_sums, and the poses are those of the
    same problem without that edge, bit for bit."""
    scans, truth, H0, edges = ring()
    clouds = [scans[0], scans[1], scans[2] + 1000.0]
    kw = dict(fixed=(0, 2), H0=H0[:3], max_iterations=30, max_overlap_distance=1.0)
    res = J.simpleicp_joint(clouds, [(0, 1), (1, 2)], **kw)
    alone = J.simpleicp_joint(clouds, [(0, 1)], **kw)
    assert all(r[1].n_kept == 0 and r[1].xi is None for r in res.log)
    assert len(res.log) == len(alone.log) and np.array_equal(res.H, alone.H)
    s = J.first_iteration_sums(clouds, [(0, 1), (1, 2)], fixed=(0, 2), H0=H0[:3], max_overlap_distance=1.0)
    assert s.n_kept[1] == 0 and not s.N[1].any() and not s.g[1].any()


def _clouds(n=3, m=200):
    rng = np.random.default_rng(1)
    return [rng.normal(size=(m, 3)) for _ in range(n)]


@pytest.mark.parametrize("edges,kw,exc,msg", [
    (np.zeros((2, 3), dtype=int), {}, ValueError, "shape"),
    ([(0.0, 1.0)], {}, ValueError, "integer"),
    ([(0, 3)], {}, ValueError, "index"),
    ([(1, 1)], {}, ValueError, "self edge"),
    ([(0, 1)], {"fixed": ()}, ValueError, "fixed"),
    ([(1, 2)], {}, ValueError, "no path to a fixed cloud"),
    ([(0, 1)], {"fixed": (0, 1)}, ValueError, "free clouds"),
    ([(0, 1)], {"H0": np.tile(np.eye(4), (2, 1, 1))}, ValueError, "H0 must have shape"),
    ([(0, 1)], {"H0": np.tile(np.eye(4), (3, 1, 1)) * np.array([1, 1, np.nan])[:, None, None]}, ValueError, "finite"),
    ([(0, 1)], {"rbp_observed_values": (0,) * 6}, TypeError, "unsupported"),
    ([(0, 1)], {"mov_neighbors": 10}, TypeError, "unsupported"),
    ([(0, 1)], {"rbp_observation_weights": (0,) * 6}, TypeError, "unsupported"),
    ([(0, 1)], {"correspondences": 5000}, ValueError, "4096"),
])
def test_simpleicp_joint_argument_checks(edges, kw, exc, msg):
    with pytest.raises(exc, match=msg):
        sb.simpleicp_joint(_clouds(), edges, **kw)


def test_more_than_256_free_clouds_are_refused():
    clouds = [np.zeros((20, 3))] * 258
    edges = [(0, i) for i in range(1, 258)]
    with pytest.raises(ValueError, match="free clouds"):
        sb.simpleicp_joint(clouds, edges)


def test_abi_declares_the_joint_entry_point():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    decl = re.search(r"int32_t sicp_register_joint\(([^;]*)\);", header)
    assert decl and "sicp_register_joint" in _capi.SYMBOLS
    # one parameter per ctypes argument type
    assert re.sub(r"/\*.*?\*/", "", decl.group(1)).count(",") + 1 == 13
