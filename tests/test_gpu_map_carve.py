"""Carving the resident map (sicp_map_carve, Map.carve) against the NumPy statement of the rule in
test_map_carve_host.py: the pass counts, the carved map (points, order and bits), the counts,
every memory kind, registrations and distances on the carved map equal to those on a fresh Map of
the same points, a mapping loop with a transient object replayed on the host, a map of millions
of points with about a million rays, and the errors."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from test_gpu_map import _map_and_scans
from test_gpu_map_crop import _distance_bytes, _same_registrations, _scan_kw
from test_gpu_map_insert import _base_map
from test_gpu_nn_exact import ORIGINS
from test_map_carve_host import carve_oracle, carve_passes, designed_carve, rays_of
from test_map_insert_host import insert_oracle

import simpleicp_b200 as sb
from oracle import simpleicp_oracle as O
from simpleicp_b200 import _capi

pytestmark = pytest.mark.gpu


def _carve_and_check(m, M_before, clouds, origins, r, margin, min_passes=1, H=None, moved=None, **kw):
    removed, passes = m.carve(clouds, H, origins=None if H is not None and origins is None else origins, radius=r,
                              margin=margin, min_passes=min_passes, return_passes=True, **kw)
    if origins is None:
        origins = H[:, :3, 3]
    want, want_passes = carve_oracle(M_before, clouds if moved is None else moved, origins, r, margin, min_passes)
    assert passes.dtype == np.uint32 and np.array_equal(passes, want_passes), "passes differ from the rule"
    got = m.points()
    assert np.array_equal(got, want), "the carved map differs from the rule"
    assert removed == len(M_before) - len(want) and m.n_points == len(want)
    return got, passes


@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_designed_geometry(gpu, where):
    M, clouds, origins, r, margin = designed_carve(ORIGINS[where])
    for rr in (r, np.nextafter(r, np.inf), np.nextafter(r, -np.inf)):
        for k in (1, 2, 3):
            with sb.Map(M) as m:
                got, passes = _carve_and_check(m, M, clouds, origins, rr, margin, k)
                assert 0 < len(got) < len(M) and passes.max() >= 3


def _rays_in(M, rng, n, length, origin_box):
    """n rays: origins drawn in origin_box around M's centre, ends at random map points moved on
    by up to `length`."""
    c = M.mean(axis=0)
    o = c + rng.uniform(-1, 1, (n, 3)) * origin_box
    tgt = M[rng.integers(0, len(M), n)]
    v = tgt - o
    return o, o + v * (1.0 + rng.uniform(0, length, (n, 1)) / np.linalg.norm(v, axis=1, keepdims=True))


@pytest.mark.parametrize("where", sorted(ORIGINS))
@pytest.mark.parametrize("r", [0.02, 0.3, 4.0])  # below, about and far above the map's cell size
def test_tube_sizes_and_ray_placement(gpu, where, r):
    M = _base_map(ORIGINS[where])  # 20 000 points over 20 m x 20 m
    rng = np.random.default_rng(41)
    c = M.mean(axis=0)
    M = np.concatenate([M, c + [[-60.0, -60.0, 0.0], [-61.0, -60.0, 0.5]]])  # no ray comes near these two
    clouds, origins = [], []
    # origins inside the map's box, rays ending at or past map points
    for _ in range(3):
        o, p = _rays_in(M, rng, 300, 3.0, np.array([8.0, 8.0, 1.0]))
        for i in range(0, 300, 100):  # one origin per cloud: take the first ray's
            origins.append(o[i])
            clouds.append(o[i] + (p[i:i + 100] - o[i:i + 100]))
    # origins far outside the box, rays longer than the map, rays missing the box
    far = c + np.array([60.0, -45.0, 30.0])
    clouds.append(M[rng.integers(0, len(M), 200)] + rng.normal(0, 0.05, (200, 3)))
    origins.append(far)
    clouds.append(c + np.array([-80.0, 50.0, -40.0]) + rng.normal(0, 1.0, (100, 3)))  # through and past
    origins.append(far)
    clouds.append(far + rng.uniform(0, 10, (100, 3)) + np.array([0.0, 0.0, 50.0]))  # misses the box
    origins.append(far)
    # zero-length rays, NaN / inf endpoints, an empty cloud
    bad = np.tile(c, (6, 1))
    bad[1, 0], bad[2, 1], bad[3, 2], bad[4] = np.nan, np.inf, -np.inf, np.nan
    clouds += [bad, np.zeros((0, 3))]
    origins += [c, c]
    origins = np.array(origins)
    for margin in (0.0, 0.5):
        with sb.Map(M) as m:
            got, passes = _carve_and_check(m, M, clouds, origins, r, margin)
            assert passes.max() >= 1 and len(got) < len(M)
            # the rays of the clouds that are none, alone: nothing passed, nothing removed
            assert m.carve(clouds[-2:], origins=origins[-2:], radius=r, margin=margin) == 0


def test_H_with_default_origins_and_explicit_origins(gpu):
    M = _base_map(ORIGINS["utm"])
    rng = np.random.default_rng(42)
    c = M.mean(axis=0)
    # scans in their sensor frame: H's translation is the sensor position in the map's frame
    pos = c + np.array([[2.0, -3.0, 4.0], [-5.0, 1.0, 3.0], [0.5, 6.0, 2.0]])
    H = np.empty((3, 4, 4))
    clouds, moved = [], []
    with _capi.Engine() as e:
        for i in range(3):
            H[i] = O.rbp_to_H(np.concatenate((rng.uniform(-0.3, 0.3, 3), pos[i] - 0.0)))
            tgt = M[rng.integers(0, len(M), 2000)]
            local = O.transform_by_H(tgt, np.linalg.inv(H[i])) * 1.02  # rays ending a little past the map
            clouds.append(local)
            e.set_clouds(M, local)
            moved.append(np.array(e.transform(H[i])))
    with sb.Map(M) as a, sb.Map(M) as b:
        got, passes = _carve_and_check(a, M, clouds, None, 0.1, 0.3, H=H, moved=moved)
        assert passes.sum() > 0
        # the same carve from the moved clouds with the translations as explicit origins
        removed, p2 = b.carve(moved, origins=H[:, :3, 3], radius=0.1, margin=0.3, return_passes=True)
        assert np.array_equal(p2, passes) and np.array_equal(b.points(), got)
        # explicit origins win over H's translations
        a2 = sb.Map(M)
        o2 = H[:, :3, 3] + 1.0
        _carve_and_check(a2, M, clouds, o2, 0.1, 0.3, H=H, moved=moved)
        a2.close()


def _bundles(X, rng, n_sensors=10, per=400):
    """Bundles of rays: from sensors 5 m above the surface to patches of 2 m x 2 m, and ghost map
    points in the air around the bundles' middles, which many rays of a bundle pass."""
    lo, hi = X.min(axis=0), X.max(axis=0)
    origins = np.column_stack([rng.uniform(lo[0] + 5, hi[0] - 5, n_sensors), rng.uniform(lo[1] + 5, hi[1] - 5, n_sensors),
                               np.full(n_sensors, hi[2] + 5.0)])
    clouds, ghosts = [], []
    for o in origins:
        t = o + np.array([rng.uniform(-15, 15), rng.uniform(-15, 15), lo[2] - o[2] - 1.0])
        P = t + rng.uniform(-1, 1, (per, 3)) * [1.0, 1.0, 0.0]
        clouds.append(P)
        ghosts.append(o + 0.5 * (P[:20] - o) + rng.normal(0, 0.2, (20, 3)))
    return clouds, origins, np.concatenate(ghosts)


def test_min_passes_and_calls_that_remove_nothing_or_everything(gpu):
    X0, scans, rows = _map_and_scans(n_map=60_000, extent=60.0, seed=77_000)
    kw = _scan_kw(rows, max_overlap_distance=1.0)
    rng = np.random.default_rng(43)
    clouds, origins, ghosts = _bundles(X0, rng)
    X = np.concatenate([X0, ghosts])
    with sb.Map(X) as m:
        before = m.register(scans, **kw)
        _, passes = carve_oracle(X, clouds, origins, 0.3, 0.5)
        assert passes.max() >= 3
        # above every count: nothing removed, the map untouched, passes still returned
        removed, got = m.carve(clouds, origins=origins, radius=0.3, margin=0.5, min_passes=int(passes.max()) + 1,
                               return_passes=True)
        assert removed == 0 and np.array_equal(got, passes)
        assert m.n_points == len(X) and np.array_equal(m.points(), X)
        _same_registrations(before, m.register(scans, **kw))
        # a carve that would remove every point: SICP_ERR_NO_OVERLAP, the map unchanged, passes written
        every = [X + np.array([0.0, 0.0, -1.0])]  # one ray per map point from high above, past it
        top = np.array([[X[:, 0].mean(), X[:, 1].mean(), 1e4]])
        out = np.full(len(X), 0, dtype=np.uint32)
        with pytest.raises(_capi.SicpError) as ei:
            m._engine.map_carve(every, origins=top, radius=0.01, margin=0.5, passes=out)
        assert ei.value.code == _capi.SICP_ERR_NO_OVERLAP and out.min() >= 1
        sel = np.concatenate([np.arange(len(X0), len(X)), rng.integers(0, len(X0), 200)])  # ghosts and a sample
        assert np.array_equal(out[sel], carve_passes(X[sel], *rays_of(every, top), 0.01, 0.5))
        assert m.n_points == len(X) and m._engine.n_map == len(X) and np.array_equal(m.points(), X)
        _same_registrations(before, m.register(scans, **kw))
        # min_passes 1 and 2
        cur = X
        for k in (2, 1):
            cur, _ = _carve_and_check(m, cur, clouds, origins, 0.3, 0.5, k)


def test_memory_kinds(gpu):
    M = _base_map(ORIGINS["origin"])
    rng = np.random.default_rng(44)
    o, p = _rays_in(M, rng, 3000, 1.0, np.array([6.0, 6.0, 1.0]))
    origins = o[::1000]
    clouds = [origins[j] + (p[1000 * j:1000 * j + 1000] - o[1000 * j:1000 * j + 1000]) for j in range(3)]
    want, want_passes = carve_oracle(M, clouds, origins, 0.2, 0.2)
    assert len(want) < len(M)
    kinds = [lambda X: X, lambda X: torch.from_numpy(X).pin_memory(), lambda X: torch.from_numpy(X).cuda()]
    for kind in kinds:
        with sb.Map(M) as m:
            removed, passes = m.carve([kind(X) for X in clouds], origins=origins, radius=0.2, margin=0.2,
                                      return_passes=True)
            assert np.array_equal(passes, want_passes) and np.array_equal(m.points(), want)
    # passes into host and device memory through the binding
    for out in (np.zeros(len(M), dtype=np.uint32), torch.zeros(len(M), dtype=torch.int32, device="cuda")):
        with sb.Map(M) as m:
            m._engine.map_carve(clouds, origins=origins, radius=0.2, margin=0.2, passes=out)
            got = out if isinstance(out, np.ndarray) else out.cpu().numpy().view(np.uint32)
            assert np.array_equal(got, want_passes) and np.array_equal(m.points(), want)


def test_carved_map_registers_and_measures_as_a_fresh_map(gpu):
    X0, scans, rows = _map_and_scans(n_map=100_000, extent=80.0, seed=76_000)
    clouds, origins, ghosts = _bundles(X0, np.random.default_rng(45))
    X = np.concatenate([X0, ghosts])
    with sb.Map(X) as m:
        t, res = m.register(scans, **_scan_kw(rows, max_overlap_distance=1.0))
        ok = [i for i, r in enumerate(res) if r is not None]
        H = t[ok, :16].reshape(-1, 4, 4)
        want, _ = carve_oracle(X, clouds, origins, 0.25, 0.3)
        assert m.carve(clouds, origins=origins, radius=0.25, margin=0.3) == len(X) - len(want) > 0
        assert np.array_equal(m.points(), want)
        got = [m.register(scans, **_scan_kw(rows, **kw)) for kw in (dict(max_overlap_distance=1.0), dict())]
        d_got = m.distances([scans[i] for i in ok], H, max_distance=0.5, neighbors=10)
    with sb.Map(want) as fresh:
        for g, kw in zip(got, (dict(max_overlap_distance=1.0), dict())):
            _same_registrations(g, fresh.register(scans, **_scan_kw(rows, **kw)))
        d_want = fresh.distances([scans[i] for i in ok], H, max_distance=0.5, neighbors=10)
    assert sum(r is not None for r in got[0][1]) >= 3
    assert _distance_bytes(d_got) == _distance_bytes(d_want)


# ---- a mapping loop with a transient object --------------------------------------------------
ROOM = np.array([[0.0, 0.0, 0.0], [12.0, 10.0, 3.0]])
BOX = np.array([[5.0, 4.0, 0.5], [6.5, 5.5, 1.5]])  # an object in the air (a person's torso, a trolley's load)


def _box_hit(o, v, lo, hi, inside):
    """Ray parameter of the first face of box [lo, hi] along o + t v: the entry for a box seen from
    outside, the exit for the room seen from inside; inf where it is missed."""
    with np.errstate(divide="ignore", invalid="ignore"):
        t0, t1 = (lo - o) / v, (hi - o) / v
    tn, tf = np.minimum(t0, t1).max(axis=1), np.maximum(t0, t1).min(axis=1)
    if inside:
        return tf
    return np.where((tn <= tf) & (tn > 0), tn, np.inf)


def scan_room(pos, with_box, n=20_000, seed=0, toward=None):
    """A ray caster: n rays from pos hit the room's walls, floor and ceiling or (with_box) the box;
    returns the hit points.  The rays go in random directions, or toward random points of the box
    `toward`."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3)) if toward is None else rng.uniform(toward[0], toward[1], (n, 3)) - pos
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    o = np.broadcast_to(pos, (n, 3))
    t = _box_hit(o, v, ROOM[0], ROOM[1], inside=True)
    if with_box:
        t = np.minimum(t, _box_hit(o, v, BOX[0], BOX[1], inside=False))
    return o + t[:, None] * v


def _on_box(P):
    return ((P >= BOX[0] - 1e-9) & (P <= BOX[1] + 1e-9)).all(axis=1)


def test_mapping_loop_with_a_transient_object(gpu):
    first = [np.array([2.0, 2.0, 1.5]), np.array([9.0, 2.5, 1.5])]
    later = [np.array([2.5, 8.0, 1.6]), np.array([9.5, 7.5, 1.4]), np.array([3.0, 5.0, 2.0])]
    v, r, margin = 0.1, 0.05, 0.3
    S0 = [scan_room(p, True, seed=10 + i) for i, p in enumerate(first)]
    # the later scans look at where the box was (rays through its volume, grown by 0.3 m)
    S1 = [scan_room(p, False, n=10_000, seed=20 + i, toward=(BOX[0] - 0.3, BOX[1] + 0.3)) for i, p in enumerate(later)]
    base = S0[0][::4]
    host, _ = insert_oracle(base, S0, v)
    assert _on_box(host).sum() > 100
    with sb.Map(base) as m:
        m.insert(S0, voxel_size=v)
        assert np.array_equal(m.points(), host)
        removed, passes = m.carve(S1, origins=np.array(later), radius=r, margin=margin, min_passes=2,
                                  return_passes=True)
        want, want_passes = carve_oracle(host, S1, np.array(later), r, margin, 2)
        assert np.array_equal(passes, want_passes) and np.array_equal(m.points(), want)
        assert removed == len(host) - len(want)
        assert not _on_box(want).any(), "every box point is removed"
        host, _ = insert_oracle(want, S1, v)
        m.insert(S1, voxel_size=v)
        assert np.array_equal(m.points(), host) and m.n_points == len(host)


# ---- at the sizes the engine is built for ------------------------------------------------------
def test_millions_of_points_and_a_million_rays(gpu):
    M = O.surface(3_000_000, 9, extent=500.0)
    rng = np.random.default_rng(46)
    sensors = np.column_stack([rng.uniform(50, 450, 24), rng.uniform(50, 450, 24), np.zeros(24)])
    clouds = []
    for s in sensors:  # about 60 000 map points within 40 m of each sensor
        near = M[np.linalg.norm(M[:, :2] - s[:2], axis=1) < 40.0]
        s[2] = near[:, 2].mean() + 2.0 if len(near) else 2.0
        # endpoints at map points seen from the sensor, some of them cut short by a few cm
        near = near[rng.permutation(len(near))[:65_000]]
        cut = rng.uniform(0, 1, (len(near), 1)) < 0.2
        clouds.append(np.where(cut, s + (near - s) * 0.97, near))
    origins = sensors
    n_rays = sum(len(X) for X in clouds)
    assert n_rays > 1_000_000
    r, margin, k = 0.05, 0.3, 2
    with sb.Map(M) as m:
        removed, passes = m.carve(clouds, origins=origins, radius=r, margin=margin, min_passes=k, return_passes=True)
        assert np.array_equal(m.points(), M[passes < k]) and removed == (passes >= k).sum() > 0
    # a few hundred map points, near tube boundaries and at random, by brute force over all rays:
    # for some rays, the map points near its tube's wall (e2 within 30 % of r^2) and near its end
    # cap (e2 < r^2, s within 5 cm of L - margin), where a walk that misses a cell would show
    # (the rays graze the terrain, so those points lie within a few metres of the ray's end)
    Orays, Prays = rays_of(clouds, origins)
    tree = cKDTree(M[:, :2])
    edge = []
    for j in rng.choice(len(Prays), 2500, replace=False):
        o, d = Orays[j], Prays[j] - Orays[j]
        L = np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
        near = np.array(tree.query_ball_point(Prays[j, :2], 3.0), dtype=np.int64)
        u = M[near] - o
        s_ = ((u[:, 0] * d[0] + u[:, 1] * d[1]) + u[:, 2] * d[2]) / L
        e2 = ((u[:, 0] * u[:, 0] + u[:, 1] * u[:, 1]) + u[:, 2] * u[:, 2]) - s_ * s_
        wall = np.flatnonzero((s_ > 0) & (s_ < L - margin) & (np.abs(e2 - r * r) < 0.3 * r * r))
        cap = np.flatnonzero((e2 < r * r) & (np.abs(s_ - (L - margin)) < 0.05))
        edge += [near[wall[:3]], near[cap[:3]]]
    edge = np.unique(np.concatenate(edge))
    assert len(edge) >= 200
    sel = np.concatenate([edge[rng.permutation(len(edge))[:300]], rng.integers(0, len(M), 150)])
    want = carve_passes(M[sel], Orays, Prays, r, margin)
    assert np.array_equal(passes[sel], want) and want.max() > 0


def _raw(e, clouds, H=None, origins=None, r=0.1, margin=0.0, k=1, passes=None):
    n = len(clouds)
    keep = [np.ascontiguousarray(X, dtype=np.float64) for X in clouds]
    ptrs = (C.c_void_p * n)(*[X.ctypes.data for X in keep])
    counts = (C.c_int64 * n)(*[len(X) for X in keep])
    out = C.c_int64(-1)
    return e._lib.sicp_map_carve(e._h, n, ptrs, counts, None if H is None else H.ctypes.data,
                                 None if origins is None else origins.ctypes.data, float(r), float(margin), int(k),
                                 None if passes is None else passes.ctypes.data, C.byref(out)), out.value


def test_errors(gpu):
    M = _base_map(ORIGINS["origin"])
    c = M.mean(axis=0)
    clouds = [M[:100] - 0.5 * (M[:100] - c)]
    org = np.array([c + [0.0, 0.0, 5.0]])
    with _capi.Engine() as e:
        assert _raw(e, clouds, origins=org)[0] == _capi.SICP_ERR_STATE
        e.set_map(M)
        H = np.eye(4)[None].copy()
        nan_o, nan_H = org.copy(), H.copy()
        nan_o[0, 1], nan_H[0, 2, 3] = np.nan, np.inf
        for kw in (dict(), dict(origins=nan_o), dict(H=nan_H, origins=org), dict(origins=org, r=0.0),
                   dict(origins=org, r=np.inf), dict(origins=org, margin=-1.0), dict(origins=org, margin=np.nan),
                   dict(origins=org, k=0), dict(origins=org, k=-3)):
            assert _raw(e, clouds, **kw)[0] == _capi.SICP_ERR_BAD_ARG, kw
        assert e._lib.sicp_map_carve(e._h, 0, None, None, None, org.ctypes.data, 0.1, 0.0, 1, None, None) \
            == _capi.SICP_ERR_BAD_ARG
        assert np.array_equal(e.get_map(), M) and e.n_map == len(M)
        # a carve clears the batch outputs; NULL passes and n_removed are fine; H alone gives the origins
        _, scans, _ = _map_and_scans(n_map=20_000, extent=20.0, seed=75_000)
        scans = [S - 10.0 for S in scans]
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        res = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
        e.batch_outputs(res)
        H[0, :3, 3] = org[0]
        for call in (lambda: e._lib.sicp_map_carve(
                         e._h, 1, (C.c_void_p * 1)(np.ascontiguousarray(clouds[0]).ctypes.data), (C.c_int64 * 1)(100),
                         None, org.ctypes.data, 0.3, 0.0, 1, None, None),
                     lambda: _raw(e, clouds, H=H)[0]):
            res = e.register_to_map(scans, 500, 10, params, max_overlap_distance=1.0)
            e.batch_outputs(res)
            assert call() == _capi.SICP_OK
            with pytest.raises(_capi.SicpError) as ei:
                e.batch_outputs(res)
            assert ei.value.code == _capi.SICP_ERR_STATE
