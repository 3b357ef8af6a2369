"""Cloud-to-map distances (sicp_map_distances, Map.distances) against exact references: a NumPy
brute force on designed dyadic geometry (bit for bit), cKDTree and sicp_select_in_range on the
dragon and bunny pairs, sicp_estimate_normals for the normals, sicp_transform for H, every memory
kind, the state the call must leave alone, and the errors."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from conftest import load_golden, load_pair
from test_gpu_map import _map_and_scans
from test_gpu_memory_kinds import KINDS, Buf, _cloud

import simpleicp_b200 as sb
from simpleicp_b200 import _capi

pytestmark = pytest.mark.gpu

O_UTM = np.array([612345.25, 5432109.875, 310.5])  # easting / northing / height: the 1/8 lattice is exact there


def brute(M, P, r):
    """(idx, d2, n_within) by the definition: d2 = (dx dx + dy dy) + dz dz to every map point, the
    lowest index among the smallest, within iff d2 < fl(r r)."""
    r2 = r * r
    idx = np.full(len(P), -1, dtype=np.int64)
    d2 = np.full(len(P), np.inf)
    fin = np.isfinite(P).all(axis=1)
    d2[~fin] = np.nan
    for j in np.flatnonzero(fin):
        d = P[j] - M
        dd = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        i = int(np.argmin(dd))  # the first of the smallest
        if dd[i] < r2:
            idx[j], d2[j] = i, dd[i]
    return idx, d2, int((idx >= 0).sum())


def lattice_map(origin, seed=0):
    """A dense block of the 1/4 lattice (midpoints of 2, 4 and 8 equidistant points inside it), a
    sparse scatter of lattice points with a hole, isolated points, and duplicates."""
    rng = np.random.default_rng(seed)
    g = np.arange(12) / 4.0
    block = np.stack(np.meshgrid(g, g, np.arange(4) / 4.0, indexing="ij"), -1).reshape(-1, 3)
    sparse = rng.integers(0, 80, (1500, 3)) / 4.0 * [1, 1, 0.25] + [5.0, 0.0, 0.0]
    hole = np.all(np.abs(sparse[:, :2] - [15.0, 10.0]) < 5.0, axis=1)  # a few map cells wide
    sparse = sparse[~hole]
    isolated = np.array([[30.0, 25.0, 3.0], [-3.0, 22.0, 1.0], [28.0, -3.0, 0.0]])
    M = np.concatenate([block, sparse, isolated])
    M = np.concatenate([M, M[rng.integers(0, len(M), 200)]])  # duplicates: the lower index wins
    M = M[rng.permutation(len(M))]
    return M + origin


def lattice_queries(M, origin, seed=1):
    rng = np.random.default_rng(seed)
    o = np.asarray(origin)
    base = o + np.concatenate([rng.integers(0, 11, (40, 2)), rng.integers(0, 3, (40, 1))], axis=1) / 4.0  # in the block
    on = M[rng.integers(0, len(M), 60)]
    e = 1 / 8.0
    mid2, mid4, mid8 = base + [e, 0, 0], base + [e, e, 0], base + [e, e, e]
    iso = o + np.array([[30.0, 25.0, 3.0], [-3.0, 22.0, 1.0], [28.0, -3.0, 0.0]])
    at_bound = np.concatenate([iso + [0.5, 0, 0], iso - [0, 0.5, 0], iso + [0, 0, 0.5]])  # d2 = 0.25 exactly
    in_hole = o + np.array([[15.0, 10.0, 2.0], [14.0, 9.5, 0.5], [16.25, 11.0, 1.0]])  # nearest several cells out
    # beyond the map's box: near its corner, and far from everything
    far = o + np.array([[-2.0, -1.0, 0.0], [1e3, 0, 0], [0, -1e3, 0], [300.0, 200.0, 1e3], [-9.0, -9.0, 0.0]])
    bad = base[:4].copy()
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3] = np.nan, np.inf, -np.inf, np.nan
    return [on, mid2, np.zeros((0, 3)), mid4, mid8, at_bound, in_hole, far, bad]


@pytest.mark.parametrize("where", ["origin", "utm"])
def test_designed_geometry_is_exact(gpu, where):
    origin = np.zeros(3) if where == "origin" else O_UTM
    M = lattice_map(origin)
    clouds = lattice_queries(M, origin)
    # 0.5: the at-bound points are excluded (d2 == r2); one ulp above 0.5, fl(r r) lies above 0.25
    # and they are in; 6.0 reaches across the hole and past the box's corner
    with sb.Map(M) as m:
        for r in (0.5, np.nextafter(0.5, 1.0), 6.0):
            idx, d2, pd, pl, n_within = m._engine.map_distances(clouds, max_distance=r)
            assert pd is None and pl is None
            for i, P in enumerate(clouds):
                wi, wd, wn = brute(M, P, r)
                assert np.array_equal(idx[i], wi), (r, i)
                assert np.array_equal(d2[i], wd, equal_nan=True), (r, i)
                assert n_within[i] == wn, (r, i)
            res = m.distances(clouds, max_distance=r)
            for i, P in enumerate(clouds):
                assert np.array_equal(res[i].index, idx[i]) and res[i].n_within == n_within[i]
                assert np.array_equal(res[i].distance, np.sqrt(d2[i]), equal_nan=True)
        hole = m._engine.map_distances([clouds[6]], max_distance=6.0)
        assert (hole[0][0] >= 0).all() and (hole[1][0] > 4.0 ** 2).any()
        at = clouds[5]
        assert m._engine.map_distances([at], max_distance=0.5)[4][0] == 0
        assert m._engine.map_distances([at], max_distance=np.nextafter(0.5, 1.0))[4][0] == len(at)


@pytest.mark.parametrize("rep", [100, 330])
def test_designed_geometry_on_the_8_and_4_lane_forms(gpu, rep):
    """The designed clouds repeated: 20 100 points in one call take the 8-lane search, 66 330 the
    4-lane one (16 lanes up to 16 384), with their ties and the lower-index rule."""
    M = lattice_map(O_UTM)
    base = lattice_queries(M, O_UTM)
    clouds = [np.tile(P, (rep, 1)) for P in base]
    total = sum(len(X) for X in clouds)
    assert (16384 < total <= 65536) if rep == 100 else total > 65536
    with sb.Map(M) as m:
        for r in (0.5, np.nextafter(0.5, 1.0), 6.0):
            idx, d2, _, _, n_within = m._engine.map_distances(clouds, max_distance=r)
            for i, P in enumerate(base):
                wi, wd, wn = brute(M, P, r)
                assert np.array_equal(idx[i], np.tile(wi, rep)), (r, i)
                assert np.array_equal(d2[i], np.tile(wd, rep), equal_nan=True), (r, i)
                assert n_within[i] == rep * wn, (r, i)


def _natural(name):
    M, X = load_pair(name)
    H = load_golden(name)["H"]
    with _capi.Engine() as e:
        e.set_clouds(M, X)
        P = np.array(e.transform(H))
    return M, X, H, P


@pytest.mark.parametrize("name", ["dragon", "bunny"])
def test_natural_data_against_ckdtree_and_select_in_range(gpu, name):
    M, X, H, P = _natural(name)
    tree = cKDTree(M)
    dd, ii = tree.query(P, k=2)
    r = float(1.2 * np.median(dd[:, 0]))  # about half of the points within
    with sb.Map(M) as m:
        idx, d2, _, _, n_within = m._engine.map_distances([P], max_distance=r)
    idx, d2 = idx[0], d2[0]
    within = idx >= 0
    assert 0.2 * len(P) < n_within[0] == within.sum() < len(P)
    # the distances: cKDTree's to rounding (the search's d2 may contract to fused multiply-adds)
    assert np.allclose(d2[within], dd[within, 0] ** 2, rtol=1e-12, atol=1e-24)
    assert np.all(np.isinf(d2[~within])) and np.all(dd[~within, 0] ** 2 >= r * r * (1 - 1e-12))
    clear = within & (dd[:, 1] ** 2 > dd[:, 0] ** 2 * (1 + 1e-12))
    assert np.array_equal(idx[clear], ii[clear, 0]) and clear.sum() > 0.9 * within.sum()
    # the within flags are sicp_select_in_range's with the moved cloud as the fixed one
    with _capi.Engine() as e:
        e.set_clouds(P, M)
        e.set_selected(None)
        keep = e.select_in_range(np.eye(4), r)
    assert np.array_equal(keep, within)


def _plane(P, Mm, nx, ny, nz):
    d = P - Mm
    return (d[:, 0] * nx.astype(np.float64) + d[:, 1] * ny.astype(np.float64)) + d[:, 2] * nz.astype(np.float64)


@pytest.mark.parametrize("k", [10, 30])
@pytest.mark.parametrize("sign", [_capi.SIGN_DGEEV, _capi.SIGN_CANONICAL])
def test_normals_equal_estimate_normals(gpu, k, sign):
    M, X, H, P = _natural("dragon")
    clouds = [X, X[::3] + 0.01, X[::5] + 0.2]  # the last mostly beyond the bound
    Hs = np.stack([H, H, H])
    r = 0.05
    with sb.Map(M) as m:
        m._engine.set_option("sign_mode", sign)
        res = m.distances(clouds, Hs, max_distance=r, neighbors=k)
    with _capi.Engine() as e:
        e.set_option("sign_mode", sign)
        for i, X_i in enumerate(clouds):
            e.set_clouds(M, X_i)
            P_i = np.array(e.transform(Hs[i]))
            idx = res[i].index
            w = idx >= 0
            assert 0 < w.sum()
            uniq = np.unique(idx[w])
            e.set_selected(uniq)
            nx, ny, nz, pl = e.estimate_normals(k)
            at = np.searchsorted(uniq, idx[w])
            got_pl, got_pd = res[i].planarity, res[i].plane_distance
            assert got_pl.dtype == np.float32 and got_pd.dtype == np.float64
            assert got_pl[w].tobytes() == pl[at].tobytes()
            assert got_pd[w].tobytes() == _plane(P_i[w], M[idx[w]], nx[at], ny[at], nz[at]).tobytes()
            assert np.isnan(got_pl[~w]).all() and np.isnan(got_pd[~w]).all()


def _bits(res):
    return [(r.index.tobytes(), r.distance.tobytes(), None if r.plane_distance is None else r.plane_distance.tobytes(),
             None if r.planarity is None else r.planarity.tobytes(), r.n_within) for r in res]


def test_H_gives_the_bits_of_the_transformed_clouds(gpu):
    M, X, H, _ = _natural("dragon")
    rng = np.random.default_rng(3)
    clouds = [X, np.zeros((0, 3)), X[1::4]]
    Hs = np.stack([H, np.eye(4), H])
    Hs[2, :3, 3] += rng.normal(0, 0.01, 3)
    with _capi.Engine() as e:
        moved = []
        for X_i, H_i in zip(clouds, Hs):
            if len(X_i) == 0:
                moved.append(X_i)
                continue
            e.set_clouds(M, X_i)
            moved.append(np.array(e.transform(H_i)))
    with sb.Map(M) as m:
        a = m.distances(clouds, Hs, max_distance=0.05, neighbors=10)
        b = m.distances(moved, max_distance=0.05, neighbors=10)
    assert _bits(a) == _bits(b) and a[0].n_within > 0 and a[1].n_within == 0 and np.isnan(a[1].fitness)


def _raw(e, clouds, n, H=None, r=1.0, k=0, idx=None, d2=None, pd=None, pl=None, n_within=None):
    m = len(n)
    arr = lambda a: None if a is None else (C.c_void_p * m)(*a)  # noqa: E731
    return e._lib.sicp_map_distances(e._h, m, (C.c_void_p * m)(*clouds), (C.c_int64 * m)(*n),
                                     None if H is None else H.ctypes.data, float(r), int(k), arr(idx), arr(d2),
                                     arr(pd), arr(pl), None if n_within is None else n_within.ctypes.data)


def test_every_memory_kind_gives_the_same_bits(gpu):
    M = load_pair("dragon")[0]
    rng = np.random.default_rng(9)
    # the first cloud is 4.8 MB: pageable, it goes through the threaded staging
    clouds = [M[rng.integers(0, len(M), 200_000)] + rng.normal(0, 0.02, (200_000, 3)),
              rng.uniform(-12, 12, (3001, 3))]
    n = [len(X) for X in clouds]
    H = np.stack([np.eye(4), np.eye(4)])
    H[1, :3, 3] = [0.5, -0.25, 0.125]
    want = None
    with sb.Map(M) as m:
        e = m._engine
        for kind in KINDS:
            objs = [_cloud(kind, X)[0] for X in clouds]
            addr = [o.ctypes.data if isinstance(o, np.ndarray) else o.data_ptr() for o in objs]
            outs = [[Buf(kind, k, dt) for k in n] for dt in (np.int64, np.float64, np.float64, np.float32)]
            nw = np.zeros(2, dtype=np.int64)
            assert _raw(e, addr, n, H, 0.05, 10, *[[b.addr for b in o] for o in outs], nw) == _capi.SICP_OK, kind
            got = [[b.get() for b in o] for o in outs] + [nw]
            if want is None:
                want = got
                assert nw[0] > 0.5 * n[0]
            for a, b in zip(got, want):
                for x, y in zip(a, b):
                    assert x.tobytes() == y.tobytes(), kind
        # NULL arrays and NULL entries skip only what they should
        out_d2 = [Buf("P", k, np.float64) for k in n]
        out_pl = [Buf("D", k, np.float32) for k in n]
        nw = np.zeros(2, dtype=np.int64)
        assert _raw(e, [X.ctypes.data for X in clouds], n, H, 0.05, 10, None, [b.addr for b in out_d2], None,
                    [out_pl[0].addr, None], nw) == _capi.SICP_OK
        assert out_d2[0].get().tobytes() == want[1][0].tobytes() and out_d2[1].get().tobytes() == want[1][1].tobytes()
        assert out_pl[0].get().tobytes() == want[3][0].tobytes() and np.isnan(out_pl[1].get()).all()
        assert np.array_equal(nw, want[4])
    torch.cuda.synchronize()


def _outputs_bytes(outs):
    return [None if o is None else (o[0].tobytes(), o[1].tobytes(), bytes(memoryview(b"".join(bytes(r) for r in o[2]))),
                                    o[3].tobytes()) for o in outs]


def test_nothing_else_changes(gpu):
    X, scans, rows = _map_and_scans(n_map=60_000, extent=60.0, seed=72_000)
    with sb.Map(X) as m:
        e = m._engine
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        res = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
        assert sum(r.status == _capi.SICP_OK for r in res) >= 3
        e.set_option("keep_knn", 1)
        e.set_clouds(X[:5000], X[:100])
        e.set_selected(None)
        e.estimate_normals(10)
        knn0 = e.get_knn(10)
        out0 = _outputs_bytes(e.batch_outputs(res))
        t0 = e.timings()
        H = np.stack([np.eye(4)] * len(scans))
        d = m.distances(scans, H, max_distance=0.5, neighbors=10)
        assert sum(r.n_within for r in d) > 0
        assert np.array_equal(m.points(), X)
        assert _outputs_bytes(e.batch_outputs(res)) == out0
        knn1 = e.get_knn(10)
        assert knn0[0].tobytes() == knn1[0].tobytes() and knn0[1].tobytes() == knn1[1].tobytes()
        t1 = e.timings()
        assert {k: v for k, v in t0.items() if k != "kernel_launches"} == {k: v for k, v in t1.items() if k != "kernel_launches"}
        # after an insert: the distances of a fresh map of the grown points
        m.insert(scans[:3], H[:3], voxel_size=0.4)
        grown = m.points()
        a = m.distances(scans, H, max_distance=0.5, neighbors=10)
    with sb.Map(grown) as fresh:
        b = fresh.distances(scans, H, max_distance=0.5, neighbors=10)
    assert _bits(a) == _bits(b)


def test_errors(gpu):
    M = lattice_map(np.zeros(3))
    X = np.ascontiguousarray(M[:100] + 0.1)
    p = [X.ctypes.data]
    with _capi.Engine() as e:
        assert _raw(e, p, [100]) == _capi.SICP_ERR_STATE
        e.set_map(M)
        bad_H = np.eye(4)[None].copy()
        bad_H[0, 0, 3] = np.inf
        out = np.zeros(100)
        for code, kw in [
            (_capi.SICP_ERR_BAD_ARG, dict(n=[-1])),
            (_capi.SICP_ERR_BAD_ARG, dict(clouds=[X.ctypes.data, None], n=[100, 5])),   # NULL with points
            (_capi.SICP_ERR_BAD_ARG, dict(clouds=p * 2, n=[100, 2 ** 32 - 100])),   # sum n = 2^32: not read
            (_capi.SICP_ERR_BAD_ARG, dict(clouds=[X.ctypes.data, None], n=[100, 2 ** 62])),
            (_capi.SICP_ERR_BAD_ARG, dict(H=bad_H)),
            (_capi.SICP_ERR_BAD_ARG, dict(r=0.0)), (_capi.SICP_ERR_BAD_ARG, dict(r=-1.0)),
            (_capi.SICP_ERR_BAD_ARG, dict(r=np.nan)), (_capi.SICP_ERR_BAD_ARG, dict(r=np.inf)),
            (_capi.SICP_ERR_BAD_ARG, dict(k=1)), (_capi.SICP_ERR_BAD_ARG, dict(k=65)), (_capi.SICP_ERR_BAD_ARG, dict(k=-3)),
            (_capi.SICP_ERR_BAD_ARG, dict(pd=[out.ctypes.data])), (_capi.SICP_ERR_BAD_ARG, dict(pl=[out.ctypes.data])),
        ]:
            args = dict(clouds=p, n=[100])
            args.update(kw)
            assert _raw(e, args.pop("clouds"), args.pop("n"), **args) == code, kw
        assert e._lib.sicp_map_distances(e._h, 0, None, None, None, 1.0, 0, None, None, None, None, None) \
            == _capi.SICP_ERR_BAD_ARG
        assert np.isnan(out).sum() == 0 and not out.any()
        assert np.array_equal(e.get_map(), M)
        e.set_map(M[:20])
        assert _raw(e, p, [100], k=21) == _capi.SICP_ERR_BAD_ARG
        assert np.array_equal(e.get_map(), M[:20])
        nw = np.zeros(2, dtype=np.int64)
        assert _raw(e, [X.ctypes.data, None], [100, 0], r=5.0, k=20, n_within=nw) == _capi.SICP_OK
        assert nw[0] > 0 and nw[1] == 0
