"""Shrinking the resident map (sicp_map_crop, sicp_map_thin, Map.crop, Map.thin) against the NumPy
statements of both rules in test_map_crop_host.py: the points, their order and their bits
(np.array_equal), the counts, registrations and distances on the shrunk map equal to those on a
fresh Map of the same points, calls that remove nothing or everything, a bounded mapping loop
replayed on the host, and the errors."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_batch_outputs import _result_bytes
from test_gpu_map import _map_and_scans
from test_gpu_map_insert import EXTENT, _base_map, _designed
from test_gpu_nn_exact import ORIGINS
from test_map_crop_host import U, boundary_lattice, crop_oracle, thin_oracle
from test_map_insert_host import insert_oracle, voxel_keys

import simpleicp_b200 as sb
from simpleicp_b200 import _capi

pytestmark = pytest.mark.gpu


def _crop_and_check(m, M_before, centers, r):
    removed = m.crop(centers, radius=r)
    want = crop_oracle(M_before, np.asarray(centers).reshape(-1, 3), r)
    got = m.points()
    assert got.dtype == np.float64 and np.array_equal(got, want), "the cropped map differs from the rule"
    assert removed == len(M_before) - len(want) and m.n_points == len(want)
    return got


@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_crop_designed_geometry(gpu, where):
    o = np.asarray(ORIGINS[where], dtype=np.float64)
    P, Cn, r = boundary_lattice(o)
    rng = np.random.default_rng(21)
    with sb.Map(P) as m:
        # the boundary lattice: points exactly at r and one ulp either side, two overlapping balls
        # and one that holds only the far block
        got = _crop_and_check(m, P, Cn, r)
        assert 0 < len(got) < len(P)
    # 700 centres (three shared-memory chunks), most of them outside the map's box, and one centre
    # given as a (3,) row
    M = _base_map(o)
    far = o + rng.uniform(-1, 1, (650, 3)) * 1e3 + np.array([5e3, 0.0, 0.0])
    inside = M[rng.integers(0, len(M), 50)] + rng.integers(-4, 5, (50, 3)) * U
    centres = np.concatenate([far[:300], inside, far[300:]])
    with sb.Map(M) as m:
        cur = _crop_and_check(m, M, centres, 1.25)
        assert 0 < len(cur) < len(M)
        cur = _crop_and_check(m, cur, inside[7], 2.0)
        assert 0 < len(cur)


@pytest.mark.parametrize("where", sorted(ORIGINS))
@pytest.mark.parametrize("v", [0.05, 0.3, 2.5])  # below, about and far above the map's cell size
def test_thin_designed_geometry(gpu, where, v):
    M0 = _base_map(ORIGINS[where])
    clouds = _designed(M0, v, ORIGINS[where])
    parts = [M0] + [X[np.isfinite(X).all(axis=1)] for X in clouds]
    M = np.concatenate(parts)  # faces, one ulp either side, duplicates, crowds, far points
    want = thin_oracle(M, v)
    assert len(want) < len(M)
    with sb.Map(M) as m:
        removed = m.thin(voxel_size=v)
        got = m.points()
        assert np.array_equal(got, want) and removed == len(M) - len(want) and m.n_points == len(want)
        assert m.thin(voxel_size=v) == 0 and np.array_equal(m.points(), want)
        # later inserts at the same voxel size keep the map at one point per voxel
        rng = np.random.default_rng(22)
        new = clouds + [rng.uniform(-3, 3, (3000, 3)) * EXTENT + np.asarray(ORIGINS[where])]
        added = m.insert(new, voxel_size=v)
        grown = m.points()
        assert np.array_equal(grown, insert_oracle(want, new, v)[0]) and added.sum() > 0
        assert len(np.unique(voxel_keys(grown, v), axis=0)) == len(grown)


def _scan_kw(rows, **kw):
    return dict(rbp_observed_values=rows, on_error="nan", full_output=True, **kw)


def _same_registrations(a, b):
    ta, ra = a
    tb, rb = b
    assert np.array_equal(ta, tb, equal_nan=True)
    for x, y in zip(ra, rb):
        assert (x is None and y is None) or _result_bytes(x) == _result_bytes(y)


def _distance_bytes(ds):
    return [(d.index.tobytes(), d.distance.tobytes(), d.plane_distance.tobytes(), d.planarity.tobytes(), d.n_within)
            for d in ds]


@pytest.mark.parametrize("op", ["crop", "thin"])
def test_shrunk_map_registers_and_measures_as_a_fresh_map(gpu, op):
    X, scans, rows = _map_and_scans(n_map=100_000, extent=80.0, seed=76_000)
    with sb.Map(X) as m:
        t, res = m.register(scans, **_scan_kw(rows, max_overlap_distance=1.0))
        ok = [i for i, r in enumerate(res) if r is not None]
        assert len(ok) >= 5
        H = t[ok, :16].reshape(-1, 4, 4)
        if op == "crop":
            # the scans' positions are near the map's corner at the origin: the far corner goes
            removed = m.crop(H[:, :3, 3], radius=70.0)
            want = crop_oracle(X, H[:, :3, 3], 70.0)
        else:
            removed = m.thin(voxel_size=0.6)
            want = thin_oracle(X, 0.6)
        assert removed > 0 and np.array_equal(m.points(), want)
        got = [m.register(scans, **_scan_kw(rows, **kw)) for kw in (dict(max_overlap_distance=1.0), dict())]
        d_got = m.distances([scans[i] for i in ok], H, max_distance=0.5, neighbors=10)
    with sb.Map(want) as fresh:
        for g, kw in zip(got, (dict(max_overlap_distance=1.0), dict())):
            _same_registrations(g, fresh.register(scans, **_scan_kw(rows, **kw)))
        d_want = fresh.distances([scans[i] for i in ok], H, max_distance=0.5, neighbors=10)
    assert sum(r is not None for r in got[0][1]) >= 3
    assert _distance_bytes(d_got) == _distance_bytes(d_want)


def test_calls_that_remove_nothing_or_everything_change_nothing(gpu):
    X, scans, rows = _map_and_scans(n_map=60_000, extent=60.0, seed=77_000)
    kw = _scan_kw(rows, max_overlap_distance=1.0)
    with sb.Map(X) as m:
        before = m.register(scans, **kw)
        assert m.crop(X.mean(axis=0), radius=1e4) == 0
        assert m.crop(np.concatenate([X[:1] + 1e5, X.mean(axis=0)[None]]), radius=1e3) == 0
        assert m.thin(voxel_size=1e-7) == 0
        assert m.n_points == len(X) and np.array_equal(m.points(), X)
        _same_registrations(before, m.register(scans, **kw))
        # a crop that would keep nothing: SICP_ERR_NO_OVERLAP, and the map is as it was
        with pytest.raises(_capi.SicpError) as ei:
            m.crop(X.max(axis=0) + 100.0, radius=50.0)
        assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP
        assert m.n_points == len(X) and m._engine.n_map == len(X) and np.array_equal(m.points(), X)
        _same_registrations(before, m.register(scans, **kw))


def test_bounded_mapping_loop_equals_the_host_replay(gpu):
    X, scans_a, rows_a = _map_and_scans(n_map=100_000, extent=80.0, seed=78_000)
    _, scans_b, rows_b = _map_and_scans(n_map=100_000, extent=80.0, seed=79_000)
    # the scans' positions H[:, :3, 3] lie near the map's corner at the origin, the map spans
    # [0, 80]^2: every crop removes more of the far corner
    steps = [(scans_a, rows_a, 0.4, 105.0), (scans_b, rows_b, 0.4, 95.0), (scans_a, rows_a, 0.3, 85.0)]
    host = X
    with sb.Map(X) as m:
        for step, (scans, rows, v, radius) in enumerate(steps):
            t, res = m.register(scans, **_scan_kw(rows, max_overlap_distance=1.0))
            with sb.Map(host) as fresh:
                _same_registrations((t, res), fresh.register(scans, **_scan_kw(rows, max_overlap_distance=1.0)))
            ok = [i for i, r in enumerate(res) if r is not None]
            assert len(ok) >= 3, step
            H = t[ok, :16].reshape(-1, 4, 4)
            added = m.insert([scans[i] for i in ok], H, voxel_size=v)
            host, counts = insert_oracle(host, [res[i].X_mov_transformed for i in ok], v)
            assert np.array_equal(added, counts)
            n_before = len(host)
            removed = m.crop(H[:, :3, 3], radius=radius)
            host = crop_oracle(host, H[:, :3, 3], radius)
            assert removed == n_before - len(host) and removed > 0, step
            assert m.n_points == len(host) and np.array_equal(m.points(), host), step


def _raw_crop(e, centers, r, n=None):
    c = None if centers is None else np.ascontiguousarray(centers, dtype=np.float64).reshape(-1, 3)
    k = (0 if c is None else len(c)) if n is None else n
    out = C.c_int64(-1)
    rc = e._lib.sicp_map_crop(e._h, k, None if c is None else c.ctypes.data, float(r), C.byref(out))
    return rc, out.value


def test_errors(gpu):
    M = _base_map(ORIGINS["origin"])
    with _capi.Engine() as e:
        assert _raw_crop(e, M[:2], 1.0)[0] == _capi.SICP_ERR_STATE
        assert e._lib.sicp_map_thin(e._h, 1.0, None) == _capi.SICP_ERR_STATE
        e.set_map(M)
        _, scans, _ = _map_and_scans(n_map=20_000, extent=20.0, seed=75_000)
        scans = [S - 10.0 for S in scans]
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        before = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
        nan_c, inf_c = M[:3].copy(), M[:3].copy()
        nan_c[1, 2], inf_c[2, 0] = np.nan, -np.inf
        assert _raw_crop(e, M[:3], 1.0, n=0)[0] == _capi.SICP_ERR_BAD_ARG
        assert _raw_crop(e, M[:3], 1.0, n=-2)[0] == _capi.SICP_ERR_BAD_ARG
        assert _raw_crop(e, None, 1.0, n=1)[0] == _capi.SICP_ERR_BAD_ARG
        assert _raw_crop(e, nan_c, 1.0)[0] == _capi.SICP_ERR_BAD_ARG
        assert _raw_crop(e, inf_c, 1.0)[0] == _capi.SICP_ERR_BAD_ARG
        for bad in (0.0, -1.0, np.nan, np.inf, -np.inf):
            assert _raw_crop(e, M[:3], bad)[0] == _capi.SICP_ERR_BAD_ARG
            assert e._lib.sicp_map_thin(e._h, bad, None) == _capi.SICP_ERR_BAD_ARG
        assert _raw_crop(e, M[:3] + 1e6, 1.0)[0] == _capi.SICP_ERR_NO_OVERLAP
        assert np.array_equal(e.get_map(), M) and e.n_map == len(M)
        after = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
        assert bytes(after) == bytes(before)
        # a crop and a thin clear the batch outputs, as an insert does; NULL n_removed is fine
        for call in (lambda: _raw_crop(e, M.mean(axis=0), 8.0), lambda: e._lib.sicp_map_thin(e._h, 0.5, None)):
            res = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
            e.batch_outputs(res)
            rc = call()
            assert (rc[0] if isinstance(rc, tuple) else rc) == _capi.SICP_OK
            with pytest.raises(_capi.SicpError) as ei:
                e.batch_outputs(res)
            assert ei.value.code == _capi.SICP_ERR_STATE
        rc, removed = _raw_crop(e, M.mean(axis=0), 1e6)
        assert rc == _capi.SICP_OK and removed == 0
        want = thin_oracle(crop_oracle(M, M.mean(axis=0), 8.0), 0.5)
        assert np.array_equal(e.get_map(), want)
