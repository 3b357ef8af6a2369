"""sicp_overlap_graph / sb.overlap_graph on the GPU: exact counts on designed dyadic geometry (at
the origin and at UTM coordinates), equality with the one-pair overlap filter on the ring and the
strip for every ordered pair, general poses, the cull boundary under rotated boxes, memory kinds,
the cap, determinism and side effects, 4096 clouds, and the path poses -> overlap graph -> edges ->
simpleicp_joint."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200._capi import SicpError

from test_gpu_joint import strip
from test_joint_host import _pair, ring

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _graph(eng, clouds, H, r, s, cap=None):
    total, pairs, counts = eng.overlap_graph(clouds, H, max_distance=r, stride=s, cap=10 ** 6 if cap is None else cap)
    assert cap is not None or len(pairs) == total
    return total, pairs, counts


def _one_pair_keep(eng, Xa, Xb, T, r, s):
    """The overlap filter flags of the pair (fixed Xa, movable Xb) under T for X_a[::s]."""
    eng.set_clouds(Xa, Xb)
    eng.set_selected(np.arange(0, len(Xa), s))
    try:
        return eng.select_in_range(T, r)
    except SicpError as e:
        assert e.code == _capi.SICP_ERR_NO_OVERLAP
        return np.zeros(eng.K, dtype=bool)


# ---- 1. exact on designed geometry --------------------------------------------------------------

def _perm_pose(rng, t):
    P = np.eye(3)[rng.permutation(3)] * rng.choice([-1.0, 1.0], 3)[:, None]
    H = np.eye(4)
    H[:3, :3] = P
    H[:3, 3] = t
    return H


def _exact_counts(clouds, H, r, s):
    """Brute force with the device's operation order: every product of the signed permutations is
    exact, q = (+-p) + t rounds once, d2 = (dx dx + dy dy) + dz dz."""
    n = len(clouds)
    out = {}
    for a in range(n):
        for b in range(n):
            if a == b or len(clouds[a]) == 0 or len(clouds[b]) == 0:
                out[a, b] = 0
                continue
            T = np.eye(4) if H is None else np.linalg.inv(H[a]) @ H[b]  # exact for these poses
            Ti = np.linalg.inv(T)
            Q = clouds[a][::s] @ Ti[:3, :3].T + Ti[:3, 3]
            D = Q[:, None, :] - clouds[b][None, :, :]
            d2 = (D[..., 0] * D[..., 0] + D[..., 1] * D[..., 1]) + D[..., 2] * D[..., 2]
            out[a, b] = int(np.count_nonzero(d2.min(axis=1) < r * r))
    return out


@pytest.mark.parametrize("offset", [(0.0, 0.0, 0.0), (4.5e5, 5.4e6, 300.0)])
@pytest.mark.parametrize("posed", [False, True])
def test_exact_counts_on_dyadic_geometry(eng, offset, posed):
    rng = np.random.default_rng(17)
    off = np.array(offset)
    r = 1.0
    # four patches of a 0.25 m lattice, 2.5 m apart along x (neighbours overlap), in the world frame
    g = np.stack(np.meshgrid(np.arange(12), np.arange(10), np.arange(2), indexing="ij"), -1).reshape(-1, 3) * 0.25
    world = [g + (2.5 * i, 0.0, 0.0) + off for i in range(4)]
    # cloud 4: probes off patch 1's corner of largest x and smallest y, z along -y, where no lattice
    # point is nearer: at exactly r, one ulp inside and one ulp outside
    c = world[1][np.argmax(world[1][:, 0] - world[1][:, 1] - world[1][:, 2])]
    y = c[1] - r
    world.append(np.array([[c[0], y, c[2]], [c[0], np.nextafter(y, np.inf), c[2]],
                           [c[0], np.nextafter(y, -np.inf), c[2]]]))
    world.append(np.zeros((0, 3)))  # an empty cloud
    if posed:
        H = np.array([_perm_pose(rng, off + rng.integers(-8, 8, 3) * 0.5) for _ in world])
        clouds = [(X - h[:3, 3]) @ h[:3, :3] for X, h in zip(world, H)]  # exact: signed permutations
        assert all(np.array_equal(Xl @ h[:3, :3].T + h[:3, 3], X) for Xl, h, X in zip(clouds, H, world))
    else:
        H, clouds = None, world
    refs = {}
    for s in (1, 3):
        ref = refs[s] = _exact_counts(clouds, H, r, s)
        total, pairs, counts = _graph(eng, clouds, H, r, s)
        want = [(a, b, ref[a, b], ref[b, a]) for a in range(len(clouds)) for b in range(a + 1, len(clouds))
                if ref[a, b] + ref[b, a] > 0]
        got = [tuple(int(v) for v in p) + tuple(int(v) for v in k) for p, k in zip(pairs, counts)]
        assert got == want, (s, got, want)
    # the probe cloud: one ulp inside is within, exactly r and one ulp outside are not (posed at the
    # origin, the move into the local frames rounds the ulp of a coordinate near 1 away)
    if not posed or off.any():
        assert refs[1][4, 1] == 1 and refs[1][1, 4] == 1


# ---- 2. equal to the one-pair filter on natural data --------------------------------------------

def _world(scans, H):
    return [np.ascontiguousarray(X @ h[:3, :3].T + h[:3, 3]) for X, h in zip(scans, H)]


@pytest.mark.parametrize("data", ["ring", "strip"])
def test_counts_equal_the_one_pair_filter(eng, data):
    if data == "ring":
        scans, truth, _, _ = ring()
    else:
        scans, truth, _, _ = strip(40, 4000, 80)
    clouds = _world(scans, truth)
    r = 1.0
    strides = (1, 7, max(len(X) for X in clouds) + 1)
    graphs = {s: _graph(eng, clouds, None, r, s) for s in strides}
    for a in range(len(clouds)):
        for b in range(len(clouds)):
            if a == b:
                continue
            eng.set_clouds(clouds[a], clouds[b])
            for s in strides:
                _, pairs, counts = graphs[s]
                eng.set_selected(np.arange(0, len(clouds[a]), s))
                try:
                    want = int(eng.select_in_range(np.eye(4), r).sum())
                except SicpError as e:
                    assert e.code == _capi.SICP_ERR_NO_OVERLAP
                    want = 0
                lo, hi = min(a, b), max(a, b)
                row = np.flatnonzero((pairs[:, 0] == lo) & (pairs[:, 1] == hi))
                got = int(counts[row[0], 0 if a < b else 1]) if len(row) else 0
                assert got == want, (a, b, s, got, want)
    assert len(graphs[1][1]) > len(clouds)


# ---- 3. general poses ---------------------------------------------------------------------------

def test_general_poses_differ_only_at_the_bound(eng):
    scans, truth, H0, _ = strip(24, 4000, 48)
    r, s = 1.0, 3
    _, pairs, counts = _graph(eng, scans, H0, r, s)
    got = {(int(a), int(b)): (int(x), int(y)) for (a, b), (x, y) in zip(pairs, counts)}
    n_nonzero = 0
    for a in range(len(scans)):
        for b in range(len(scans)):
            if a == b:
                continue
            T = np.linalg.inv(H0[a]) @ H0[b]
            keep = _one_pair_keep(eng, scans[a], scans[b], T, r, s)
            lo, hi = min(a, b), max(a, b)
            c = got.get((lo, hi), (0, 0))[0 if a < b else 1]
            n_nonzero += keep.sum() > 0
            if c != keep.sum():
                Ti = np.linalg.inv(T)
                d, _ = cKDTree(scans[b]).query(scans[a][::s] @ Ti[:3, :3].T + Ti[:3, 3])
                near = np.abs(d * d - r * r) <= 1e-9 * r * r
                assert abs(c - int(keep.sum())) <= int(near.sum()), (a, b, c, int(keep.sum()))
    assert n_nonzero > 2 * len(scans)


# ---- 4. the cull boundary under rotated boxes ---------------------------------------------------

def _rz(deg, t):
    a = np.deg2rad(deg)
    H = np.eye(4)
    H[:3, :3] = [[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]
    H[:3, 3] = t
    return H


@pytest.mark.parametrize("factor", [1 - 1e-12, 1 + 1e-12])
def test_cull_boundary_with_rotated_boxes(eng, factor):
    rng = np.random.default_rng(4)
    r = 0.5
    Xb = np.vstack((rng.uniform(0, 10, size=(3000, 3)) * (1, 1, 0.1), [[10.0, 10.0, 1.0]]))  # a box corner
    Hb = _rz(45.0, (100.0, 50.0, 3.0))
    corner = Hb[:3, :3] @ np.array([10.0, 10.0, 1.0]) + Hb[:3, 3]
    # cloud a: points beyond that corner along the diagonal, the closest at r * factor in the world
    # the corner's outward diagonal: every point of b's box is at least t from corner + t u
    u = Hb[:3, :3] @ (np.array([1.0, 1.0, 1.0]) / np.sqrt(3.0))
    Ha = _rz(30.0, corner + 5.0 * u)
    W = corner + np.outer(r * factor + rng.uniform(0, 3, 500), u)
    W[0] = corner + r * factor * u
    Xa = (W - Ha[:3, 3]) @ Ha[:3, :3]
    H = np.array([Ha, Hb])
    total, pairs, counts = _graph(eng, [Xa, Xb], H, r, 1)
    want_ab = int(_one_pair_keep(eng, Xa, Xb, np.linalg.inv(Ha) @ Hb, r, 1).sum())
    want_ba = int(_one_pair_keep(eng, Xb, Xa, np.linalg.inv(Hb) @ Ha, r, 1).sum())
    if want_ab + want_ba == 0:
        assert total == 0
    else:
        assert total == 1 and counts[0].tolist() == [want_ab, want_ba]
    assert (total == 1) == (factor < 1)  # the closest pair decides: inside r by 1e-12 or outside


# ---- 5. memory kinds ----------------------------------------------------------------------------

def test_memory_kinds_give_the_same_bits(eng):
    scans, truth, H0, _ = ring()
    ref = _graph(eng, scans, H0, 1.0, 2)
    pinned = [torch.from_numpy(X).pin_memory().numpy() for X in scans]
    device = [torch.from_numpy(X).cuda() for X in scans]
    for clouds in (pinned, device):
        got = _graph(eng, clouds, H0, 1.0, 2)
        assert got[0] == ref[0] and np.array_equal(got[1], ref[1]) and np.array_equal(got[2], ref[2])


# ---- 6. cap, determinism and side effects -------------------------------------------------------

def test_cap_determinism_and_side_effects(eng):
    scans, truth, H0, edges = ring()
    full = _graph(eng, scans, H0, 1.0, 1)
    assert full[0] > 3
    again = _graph(eng, scans, H0, 1.0, 1)
    assert again[0] == full[0] and np.array_equal(again[1], full[1]) and np.array_equal(again[2], full[2])
    for cap in (0, 1, 3):
        total, pairs, counts = eng.overlap_graph(scans, H0, max_distance=1.0, stride=1, cap=cap)
        assert total == full[0] and np.array_equal(pairs, full[1][:cap]) and np.array_equal(counts, full[2][:cap])
    total = C.c_int64(-1)
    n = (C.c_int64 * len(scans))(*[len(X) for X in scans])
    ptrs = (C.c_void_p * len(scans))(*[X.ctypes.data for X in scans])
    eng._check(eng._lib.sicp_overlap_graph(eng._h, len(scans), ptrs, n, H0.ctypes.data, 1.0, 1, None, None, None, None,
                                           5, C.byref(total)))
    assert total.value == full[0]

    # the state of every other path is untouched
    e = _capi.Engine(0)
    try:
        lsq = e.lsq_params((0.0,) * 6, (0.0,) * 6, [0.0] * 6, 1)
        p = e.run_params(0.3, 1.0, 30, lsq)
        e.set_option("keep_knn", 1)
        X_fix, X_mov = _pair("bunny")
        e.register_fused(X_fix, X_mov, 500, 10, 1.0, p)
        e.K = 500

        def one_pair():
            res = np.empty(4096)
            k = C.c_int64(0)
            e._check(e._lib.sicp_get_residuals(e._h, res.ctypes.data, res.size, C.byref(k)))
            return e.get_transform(), res[:k.value].copy(), e.get_knn(10)

        e.set_map(scans[0])
        fixed = np.zeros(len(scans), dtype=bool)
        fixed[0] = True
        H, out = e.register_joint(scans, edges, fixed, H0, 1000, 10, p, 1.0)
        before = (one_pair(), e.batch_outputs(out), e.joint_covariances(len(scans), len(edges)), e.get_map())
        got = e.overlap_graph(scans, H0, max_distance=1.0, stride=1, cap=100)
        assert got[0] == full[0] and np.array_equal(got[1], full[1]) and np.array_equal(got[2], full[2])
        after = (one_pair(), e.batch_outputs(out), e.joint_covariances(len(scans), len(edges)), e.get_map())
    finally:
        e.close()
    (T0, R0, (i0, d0)), (T1, R1, (i1, d1)) = before[0], after[0]
    assert np.array_equal(T0, T1) and np.array_equal(R0, R1) and np.array_equal(i0, i1) and np.array_equal(d0, d1)
    for o0, o1 in zip(before[1], after[1]):
        assert np.array_equal(o0[0], o1[0]) and np.array_equal(o0[1], o1[1]) and np.array_equal(o0[3], o1[3])
    for c0, c1 in zip(before[2][:2], after[2][:2]):
        assert np.array_equal(c0, c1, equal_nan=True)
    assert np.array_equal(before[3], after[3])


def test_library_refusals(eng):
    X = np.zeros((10, 3))
    good = np.tile(np.eye(4), (2, 1, 1))

    def call(n_clouds=2, ptrs=(X, X), counts=(10, 10), H=None, r=1.0, s=1, cap=0, n_pairs=True):
        p = (C.c_void_p * max(len(ptrs), 1))(*[None if a is None else a.ctypes.data for a in ptrs])
        n = (C.c_int64 * max(len(counts), 1))(*counts)
        tot = C.c_int64(0)
        return eng._lib.sicp_overlap_graph(eng._h, n_clouds, p, n, None if H is None else H.ctypes.data, r, s, None,
                                           None, None, None, cap, C.byref(tot) if n_pairs else None)

    bad_row, skew, nan = good.copy(), good.copy(), good.copy()
    bad_row[1, 3, 2] = 1.0
    skew[0, 1, 2] = 1e-5
    nan[1, 0, 3] = np.nan
    for kw in ({"n_clouds": 0}, {"counts": (10, -1)}, {"ptrs": (X, None)}, {"H": nan}, {"H": bad_row}, {"H": skew},
               {"r": 0.0}, {"r": np.inf}, {"s": 0}, {"cap": -1}, {"counts": (1 << 31, 1 << 31)}, {"n_pairs": False}):
        assert call(**kw) == _capi.SICP_ERR_BAD_ARG, kw
    Y = np.array([[0.0, 0.0, np.nan]] * 10)
    assert call(ptrs=(X, Y)) == _capi.SICP_ERR_BAD_ARG  # the grid builder refuses it
    assert call(ptrs=(X, None), counts=(10, 0)) == _capi.SICP_OK  # an empty cloud needs no pointer


# ---- 7. at scale --------------------------------------------------------------------------------

def test_4096_strip_clouds(eng):
    n = 4096
    scans, truth, _, _ = strip(n, 20_000, n)
    r, s = 0.5, 4
    total, pairs, counts = _graph(eng, scans, truth, r, s)
    gap = pairs[:, 1] - pairs[:, 0]
    seen = set(map(tuple, pairs.tolist()))
    assert all((i, j) in seen for i in range(n) for j in range(i + 1, min(i + 13, n)))
    assert gap.max() < 14
    rng = np.random.default_rng(0)
    for k in rng.choice(len(pairs), 200, replace=False):
        a, b = (int(v) for v in pairs[k])
        for (x, y), c in (((a, b), counts[k, 0]), ((b, a), counts[k, 1])):
            T = np.linalg.inv(truth[x]) @ truth[y]
            keep = _one_pair_keep(eng, scans[x], scans[y], T, r, s)
            if c != keep.sum():  # general poses: only points at the bound may differ (test 3)
                Ti = np.linalg.inv(T)
                d, _ = cKDTree(scans[y]).query(scans[x][::s] @ Ti[:3, :3].T + Ti[:3, 3])
                assert abs(int(c) - int(keep.sum())) <= int((np.abs(d * d - r * r) <= 1e-9 * r * r).sum())


# ---- 8. end to end ------------------------------------------------------------------------------

def test_poses_overlap_graph_edges_joint():
    scans, truth, H0, _ = ring()
    g = sb.overlap_graph(scans, H0, max_distance=1.0, stride=10)
    assert g.pairs.shape[1] == 2 and np.array_equal(g.sampled, [(len(X) + 9) // 10 for X in scans])
    edges = g.pairs[g.fraction.min(axis=1) > 0.2]
    assert len(edges) >= len(scans)
    res = sb.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    assert np.abs(res.H - truth).max() < 1e-2
