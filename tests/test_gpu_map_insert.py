"""Growing the resident map (sicp_map_insert, sicp_get_map, Map.insert, Map.points) against the
NumPy statement of the rule in test_map_insert_host.py: the points, their order and their bits
(np.array_equal), the per-cloud counts, the transforms, every memory kind, the errors, and
registrations on the grown map equal to those on a fresh Map of the same points."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import simpleicp_oracle as O
from test_gpu_batch_outputs import _result_bytes
from test_gpu_map import _map_and_scans
from test_gpu_memory_kinds import KINDS, Buf, _cloud
from test_gpu_nn_exact import ORIGINS
from test_map_insert_host import insert_oracle

import simpleicp_b200 as sb
from simpleicp_b200 import _capi

pytestmark = pytest.mark.gpu

# the map of most tests: 20 000 points over 20 m x 20 m, so the map grid's cells are about 0.25 m
EXTENT = 20.0


def _base_map(origin, seed=5):
    return O.surface(20_000, seed, extent=EXTENT) - EXTENT / 2 + np.asarray(origin)


def _designed(M, v, origin, seed=6):
    """New clouds: points exactly on voxel faces k v and one ulp either side, negative
    coordinates, duplicates of map points, a crowd in one empty voxel, points in the voxels next
    to occupied ones, points far outside the map's box, NaN and inf points, an empty cloud."""
    rng = np.random.default_rng(seed)
    o = np.asarray(origin)
    k = np.floor(o / v) + rng.integers(-int(EXTENT / v) // 2, int(EXTENT / v) // 2 + 1, (300, 3))
    k[:, 2] = np.floor(o[2] / v) + rng.integers(-2, 4, 300)
    faces = k * v
    near = M[rng.integers(0, len(M), 300)]
    beside = near + v * rng.integers(-1, 2, (300, 3))
    crowd = np.floor(o / v) * v + np.array([0.0, 0.0, 40.0 * v]) + rng.uniform(0.1, 0.9, (40, 3)) * v
    far = o + rng.uniform(-1, 1, (50, 3)) * 10 * EXTENT + np.array([1e3, -1e3, 50.0])
    bad = near[:8].copy()
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3] = np.nan, np.inf, -np.inf, np.nan
    bad[4, 0] = -np.inf
    return [faces, np.nextafter(faces, -np.inf), np.zeros((0, 3)), np.nextafter(faces, np.inf), near[:100],
            beside, crowd, far, bad, rng.uniform(-EXTENT / 2, EXTENT / 2, (5000, 3)) * [1, 1, 0.2] + o]


def _insert_and_check(m, M_before, clouds, v, H=None, moved=None):
    added = m.insert(clouds, H, voxel_size=v)
    want, counts = insert_oracle(M_before, clouds if moved is None else moved, v)
    got = m.points()
    assert got.dtype == np.float64 and np.array_equal(got, want), "the grown map differs from the rule"
    assert np.array_equal(added, counts) and m.n_points == len(want)
    return got


@pytest.mark.parametrize("where", sorted(ORIGINS))
@pytest.mark.parametrize("v", [0.05, 0.3, 2.5])  # below, about and far above the map's cell size
def test_designed_geometry(gpu, where, v):
    M = _base_map(ORIGINS[where])
    clouds = _designed(M, v, ORIGINS[where])
    with sb.Map(M) as m:
        got = _insert_and_check(m, M, clouds, v)
    assert len(got) > len(M)


def test_with_H_equals_the_transformed_clouds(gpu):
    M = _base_map(ORIGINS["utm"])
    rng = np.random.default_rng(7)
    clouds = [M[rng.integers(0, len(M), n)] + rng.normal(0, 0.3, (n, 3)) for n in (3000, 1, 0, 2001)]
    H = np.empty((len(clouds), 4, 4))
    moved = []
    with _capi.Engine() as e:
        for i, X in enumerate(clouds):
            H[i] = O.rbp_to_H(np.concatenate((rng.uniform(-0.05, 0.05, 3), rng.uniform(-2, 2, 3))))
            if len(X) == 0:
                moved.append(X)
                continue
            e.set_clouds(M, X)
            moved.append(np.array(e.transform(H[i])))
    with sb.Map(M) as a, sb.Map(M) as b:
        got = _insert_and_check(a, M, clouds, 0.2, H=H, moved=moved)
        b.insert(moved, voxel_size=0.2)
        assert np.array_equal(got, b.points())


def _scan_kw(rows, **kw):
    return dict(rbp_observed_values=rows, on_error="nan", full_output=True, **kw)


def test_an_insert_that_adds_nothing_changes_nothing(gpu):
    X, scans, rows = _map_and_scans(n_map=60_000, extent=60.0, seed=72_000)
    kw = _scan_kw(rows, max_overlap_distance=1.0)
    with sb.Map(X) as m:
        t0, r0 = m.register(scans, **kw)
        nan = np.full((100, 3), np.nan)
        added = m.insert([X[::7], X[3::11], nan, np.zeros((0, 3))], voxel_size=0.5)
        assert added.tolist() == [0, 0, 0, 0] and m.n_points == len(X)
        assert np.array_equal(m.points(), X)
        t1, r1 = m.register(scans, **kw)
    assert np.array_equal(t0, t1, equal_nan=True)
    for a, b in zip(r0, r1):
        assert (a is None and b is None) or _result_bytes(a) == _result_bytes(b)


def test_three_inserts_equal_the_rule_three_times(gpu):
    M = _base_map(ORIGINS["origin"])
    rng = np.random.default_rng(8)
    with sb.Map(M) as m:
        cur = M
        for step, v in enumerate((0.3, 0.3, 0.7)):
            clouds = [rng.uniform(-EXTENT, EXTENT, (4000, 3)) * [1, 1, 0.3] for _ in range(3)]
            cur = _insert_and_check(m, cur, clouds, v)
        assert len(cur) > len(M) + 3000


def test_every_memory_kind_gives_the_same_map(gpu):
    M = _base_map(ORIGINS["utm"])
    rng = np.random.default_rng(9)
    # the first cloud is 4.8 MB: pageable, it goes through the threaded staging
    clouds = [M[rng.integers(0, len(M), 200_000)] + rng.normal(0, 0.5, (200_000, 3)),
              rng.uniform(-EXTENT, EXTENT, (3001, 3)) + ORIGINS["utm"]]
    H = np.stack([O.rbp_to_H(np.array([0.01, -0.02, 0.03, 0.5, -0.25, 0.125])), np.eye(4)])
    want = None
    for kind in KINDS:
        objs = [_cloud(kind, X)[0] for X in clouds]
        with sb.Map(M) as m:
            added = m.insert(objs, H, voxel_size=0.25)
            got = m.points()
            out = Buf(kind, got.shape, np.float64)
            n = C.c_int64(0)
            m._engine._check(m._engine._lib.sicp_get_map(m._engine._h, out.addr, len(got), C.byref(n)))
            assert n.value == len(got) and np.array_equal(out.get(), got), kind
        if want is None:
            want = (got, added)
        assert np.array_equal(got, want[0]) and np.array_equal(added, want[1]), kind
    torch.cuda.synchronize()


@pytest.mark.parametrize("overlap", [dict(max_overlap_distance=1.0), dict()])
def test_registrations_on_the_grown_map_equal_a_fresh_map(gpu, overlap):
    X, scans, rows = _map_and_scans(n_map=100_000, extent=80.0, seed=73_000)
    X2, scans2, rows2 = _map_and_scans(n_map=100_000, extent=80.0, seed=74_000)
    kw = dict(max_overlap_distance=1.0)
    with sb.Map(X) as m:
        table, results = m.register(scans, **_scan_kw(rows, **kw))
        ok = [i for i, r in enumerate(results) if r is not None]
        assert len(ok) >= 5
        H = table[ok, :16].reshape(-1, 4, 4)
        added = m.insert([scans[i] for i in ok], H, voxel_size=0.4)
        want, counts = insert_oracle(X, [results[i].X_mov_transformed for i in ok], 0.4)
        grown = m.points()
        assert np.array_equal(grown, want) and np.array_equal(added, counts) and counts.sum() > 0
        t_grown, r_grown = m.register(scans2, **_scan_kw(rows2, **overlap))
    with sb.Map(want) as fresh:
        t_fresh, r_fresh = fresh.register(scans2, **_scan_kw(rows2, **overlap))
    assert np.array_equal(t_grown, t_fresh, equal_nan=True)
    assert sum(r is not None for r in r_grown) >= 5
    for a, b in zip(r_grown, r_fresh):
        assert (a is None and b is None) or _result_bytes(a) == _result_bytes(b)


def _raw_insert(e, clouds, n, H=None, v=1.0):
    k = len(n)
    ptrs = (C.c_void_p * k)(*[None if X is None else X.ctypes.data for X in clouds])
    counts = (C.c_int64 * k)(*n)
    return e._lib.sicp_map_insert(e._h, k, ptrs, counts, None if H is None else H.ctypes.data, float(v), None)


def test_errors(gpu):
    M = _base_map(ORIGINS["origin"])
    X = M[:100] + 5.0
    with _capi.Engine() as e:
        with pytest.raises(_capi.SicpError) as ei:
            e.map_insert([X], voxel_size=1.0)
        assert ei.value.code == _capi.SICP_ERR_STATE
        with pytest.raises(_capi.SicpError) as ei:
            e.get_map()
        assert ei.value.code == _capi.SICP_ERR_STATE
        e.set_map(M)
        _, scans, rows = _map_and_scans(n_map=20_000, extent=EXTENT, seed=75_000)
        scans = [S - EXTENT / 2 for S in scans]
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        before = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
        bad_H = np.tile(np.eye(4), (1, 1, 1))
        bad_H[0, 1, 1] = np.nan
        # n_map + the clouds' points reaches 2^32: refused on the count, nothing is read
        assert _raw_insert(e, [X], [2 ** 32 - len(M)]) == _capi.SICP_ERR_BAD_ARG
        assert _raw_insert(e, [X, None], [100, 2 ** 62]) == _capi.SICP_ERR_BAD_ARG
        assert _raw_insert(e, [X, None], [100, 5]) == _capi.SICP_ERR_BAD_ARG      # NULL with points
        assert _raw_insert(e, [X], [-1]) == _capi.SICP_ERR_BAD_ARG
        assert _raw_insert(e, [X], [100], H=bad_H) == _capi.SICP_ERR_BAD_ARG
        assert e._lib.sicp_map_insert(e._h, 0, None, None, None, 1.0, None) == _capi.SICP_ERR_BAD_ARG
        for v in (0.0, -1.0, np.nan, np.inf):
            assert _raw_insert(e, [X], [100], v=v) == _capi.SICP_ERR_BAD_ARG
        assert np.array_equal(e.get_map(), M) and e.n_map == len(M)
        after = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
        assert bytes(after) == bytes(before)
        # an insert clears the batch outputs, as set_map does
        e.batch_outputs(after)
        want, counts = insert_oracle(M, [X, np.zeros((0, 3))], 1.0)
        assert np.array_equal(e.map_insert([X, np.zeros((0, 3))], voxel_size=1.0), counts) and counts[0] > 0
        assert np.array_equal(e.get_map(), want)
        with pytest.raises(_capi.SicpError) as ei:
            e.batch_outputs(after)
        assert ei.value.code == _capi.SICP_ERR_STATE
