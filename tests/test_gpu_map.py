"""Many scans against one resident map (sicp_set_map / sicp_register_to_map, sb.Map): against
sicp_register scan by scan, bit for bit against sicp_register_batch with the map repeated, and
the culled overlap filter at its boundary."""
import numpy as np
import pytest

from oracle import simpleicp_oracle as O
from test_gpu_batch_overlap import _lsq, _same_as_register, _same_bits
from test_gpu_nn_exact import ORIGINS, U, exact_knn, perm_H

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200.linearized import VARIANT_LINEARIZED
from simpleicp_b200.simpleicp import _observed_in_radians

pytestmark = pytest.mark.gpu


def _tile(X, x0, y0, w):
    m = (X[:, 0] >= x0) & (X[:, 0] < x0 + w) & (X[:, 1] >= y0) & (X[:, 1] < y0 + w)
    return np.ascontiguousarray(X[m])


def _map_and_scans(n_map=300_000, extent=120.0, seed=70_000):
    """A surface map and ragged tiles of a second realisation, each moved by a small rigid
    transform and given a noisy prior (degrees): tiles inside the map, tiles hanging over its
    edges, and one tile entirely off it (last)."""
    X = O.surface(n_map, seed, extent=extent)
    second = O.surface(n_map, seed + 1, extent=extent)
    rng = np.random.default_rng(seed)
    tiles = [(10, 10, 25), (60, 40, 30), (100, 95, 30), (-15, 50, 30), (40, 80, 20), (70, -10, 22)]
    raw = [_tile(second, *(np.array(t) * extent / 120.0)) for t in tiles]
    raw.append(O.surface(20_000, seed + 2, extent=20.0) + np.array([10 * extent, 10 * extent, 0.0]))  # off the map
    scans, rows = [], []
    for S in raw:
        true = np.concatenate((rng.uniform(-1, 1, 2), rng.uniform(-4, 4, 1), rng.uniform(-0.4, 0.4, 3)))
        scans.append(O.transform_by_H(S, np.linalg.inv(O.rbp_to_H(_observed_in_radians(true)))))
        rows.append(true + np.concatenate((rng.normal(0, 0.05, 3), rng.normal(0, 0.03, 3))))
    return X, scans, np.array(rows)


_DATA = {}


def _data():
    if "big" not in _DATA:
        _DATA["big"] = _map_and_scans()
    return _DATA["big"]


def _rad(rows):
    return np.array([_observed_in_radians(r) for r in rows])


@pytest.mark.parametrize("variant", [0, VARIANT_LINEARIZED])
def test_equal_to_register_per_scan(gpu, variant):
    X, scans, rows = _data()
    with _capi.Engine() as e:
        e.set_option("variant", variant)
        e.set_map(X)
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        for mod in (0.5, 1.0):
            res = e.register_to_map(scans, 1000, 10, params, max_overlap_distance=mod, observed=_rad(rows))
            assert res[-1].status == _capi.SICP_ERR_NO_OVERLAP and res.n_selected[-1] == 0
            for i, S in enumerate(scans[:-1]):
                r = sb.register(X, S, engine=e, want_normals=False, max_overlap_distance=mod,
                                rbp_observed_values=rows[i])
                _same_as_register(res[i], int(res.n_selected[i]), r, f"variant {variant} mod {mod} scan {i}")


@pytest.mark.parametrize("variant", [0, VARIANT_LINEARIZED])
def test_without_filter_selects_from_the_whole_map(gpu, variant):
    X, scans, rows = _map_and_scans(n_map=30_000, extent=40.0, seed=71_000)
    scans, rows = scans[:2] + [scans[4]], rows[[0, 1, 4]]
    with _capi.Engine() as e:
        e.set_option("variant", variant)
        e.set_map(X)
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        res = e.register_to_map(scans, 1000, 10, params, observed=_rad(rows))
        for i, S in enumerate(scans):
            r = sb.register(X, S, engine=e, want_normals=False, rbp_observed_values=rows[i])
            _same_as_register(res[i], int(res.n_selected[i]), r, f"variant {variant} scan {i}")


@pytest.mark.parametrize("opts", [dict(max_overlap_distance=1.0),
                                  dict(max_overlap_distance=1.0, mov_neighbors=10, max_angle_rad=np.deg2rad(20.0)),
                                  dict(mov_neighbors=10, max_angle_rad=np.deg2rad(20.0)),
                                  dict()])
def test_bits_equal_the_batch_with_the_map_repeated(gpu, opts):
    X, scans, rows = _data()
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        e.set_map(X)
        a = e.register_to_map(scans, 1000, 10, params, observed=_rad(rows), **opts)
        b = e.register_batch([(X, S) for S in scans], 1000, 10, params, observed=_rad(rows), **opts)
    assert np.array_equal(a.n_selected, b.n_selected), (a.n_selected, b.n_selected)
    for i in range(len(scans)):
        assert _same_bits(a[i], b[i]), f"{opts} scan {i}"


def _grown_box_count(X, S, row, r, slack):
    """Map points inside the box of S's bounding box (its high faces moved out by `slack`, more
    than a grid cell) mapped by the prior and grown by r + 1 mm: a superset of the cull box."""
    lo, hi = S.min(axis=0), S.max(axis=0) + slack
    C = np.array([[(hi if k & (1 << a) else lo)[a] for a in range(3)] for k in range(8)])
    TC = O.transform_by_H(C, O.rbp_to_H(_observed_in_radians(row)))
    blo, bhi = TC.min(axis=0) - r - 1e-3, TC.max(axis=0) + r + 1e-3
    return int(np.all((X >= blo) & (X <= bhi), axis=1).sum())


def test_the_cull_searches_few_map_points(gpu):
    X, scans, rows = _data()
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        e.set_map(X)
        for mod in (0.5, 1.0):
            res = e.register_to_map(scans, 1000, 10, params, max_overlap_distance=mod, observed=_rad(rows))
            n = e.timings()["overlap_candidates"]
            bound = sum(_grown_box_count(X, S, row, mod, 2.0) for S, row in zip(scans, rows))
            assert 0 < n <= bound, (n, bound)
            assert n < len(scans) * len(X) / 8, n
            assert n >= res.n_selected.sum()
        e.register_to_map(scans, 1000, 10, params, observed=_rad(rows))
        assert e.timings()["overlap_candidates"] == 0


# ------------------------------------------------------------------------- filter boundary
R_LAT = 300  # max_overlap_distance = R_LAT U: its square is exact
SIDE = 19 * 1024


def _lattice():
    """A scan: 20 x 20 lattice points, 1024 units apart, flat; its box minimum is a point."""
    return np.stack(np.meshgrid(*[np.arange(0, SIDE + 1, 1024)] * 2, [0], indexing="ij"), -1).reshape(-1, 3)


def _boundary_queries(rng, mk):
    """Offsets at exactly r, at the largest d^2 below r^2 and around r^2, half of them outwards
    from the corners and edges of the scan (next to the faces of its box), half from inner points
    with random signs; lattice units in the scan's frame."""
    r = R_LAT
    offs = []
    for target in range(r * r - 40, r * r + 41):
        a = rng.integers(0, r + 1)
        b2 = target - a * a
        if b2 < 0:
            continue
        b = int(np.sqrt(b2))
        cc = int(np.sqrt(b2 - b * b))
        if cc * cc == b2 - b * b:
            offs.append([a, b, cc])
    offs += [[r, 0, 0], [0, r, 0], [0, 0, r], [0, 0, r - 1], [r - 1, 1, 0], [r, 1, 0], [1, 0, r]]
    inside = max(a * a + b * b + c * c for a in range(r) for b in range(40) for c in range(40)
                 if a * a + b * b + c * c < r * r)
    offs += [[a, b, c] for a in range(r - 2, r) for b in range(40) for c in range(40)
             if a * a + b * b + c * c == inside] * 2
    offs = np.array(offs)
    edges = np.array([[x, y, 0] for x in (0, 9 * 1024, SIDE) for y in (0, 9 * 1024, SIDE) if (x, y) != (9 * 1024,) * 2])
    qk = []
    for j, o in enumerate(offs):
        if j % 2 == 0:
            base = edges[rng.integers(0, len(edges))]
            sign = [(-1 if v == 0 else (1 if v == SIDE else rng.choice([-1, 1]))) for v in base[:2]] + [rng.choice([-1, 1])]
        else:
            base = mk[rng.integers(0, len(mk))]
            sign = rng.choice([-1, 1], 3)
        qk.append(base + o * np.array(sign))
    qk = np.array(qk)
    _, d2 = exact_knn(mk, qk, 1)
    assert (d2[:, 0] == r * r).any() and (d2[:, 0] == inside).any() and (d2[:, 0] > r * r).any()
    return qk, d2[:, 0]


def _rz(deg):
    return O.rbp_to_H(np.array([0.0, 0.0, np.deg2rad(deg), 0.0, 0.0, 0.0]))[:3, :3]


def _boundary_map(origin):
    """Scans at `origin` whose priors are dyadic translations, signed axis permutations (yaws of
    multiples of 90 degrees) and yaws in (-90, 0) degrees, placed far apart in one map.  Around
    each of the first two kinds lie the boundary queries; next to the corner of each of the last
    kind (the box minimum, which that yaw maps to the low x face of the transformed box) lies a
    sweep of points along x, one ulp apart, across the distance r.  Returns the map, the scans,
    their priors (radians) and, per scan, the integer reference counts (strictly below r^2, at
    exactly r^2) or None."""
    rng = np.random.default_rng(12)
    mk = _lattice()
    o = np.asarray(origin, dtype=np.float64)
    Xm = o + mk * U
    kinds = [("t", 0), ("t", 0), ("p", 90), ("p", 180), ("p", -90), ("y", -30), ("y", -50), ("y", -10), ("y", -75)]
    pts, scans, rows, refs = [], [], [], []
    for i, (kind, deg) in enumerate(kinds):
        s = np.array([40_000 * i + 5, -3 + 7 * i, 2 - i])
        if kind == "t":
            H = perm_H(np.eye(3), s, origin)
            x = np.array([0, 0, 0, *H[:3, 3]])
        else:
            R = _rz(deg)
            x = np.array([0.0, 0.0, np.deg2rad(deg), *(o + s * U - R @ o)])
            H = O.rbp_to_H(x)
        if kind in "tp":
            qk, d2 = _boundary_queries(rng, mk)
            P = np.rint(H[:3, :3]) if kind == "p" else np.eye(3)
            pts.append(o + (qk @ P.T + s) * U)
            refs.append((int((d2 < R_LAT ** 2).sum()), int((d2 == R_LAT ** 2).sum())))
        else:
            corner = O.transform_by_H(Xm[:1], H)[0]
            edge = corner[0] - R_LAT * U
            xs = [edge]
            for _ in range(60):
                xs.append(np.nextafter(xs[-1], np.inf))
                xs.insert(0, np.nextafter(xs[0], -np.inf))
            pts.append(np.column_stack((xs, np.full(len(xs), corner[1]), np.full(len(xs), corner[2]))))
            refs.append(None)
        scans.append(Xm.copy())
        rows.append(x)
    return np.concatenate(pts), scans, np.array(rows), refs


@pytest.mark.parametrize("where", list(ORIGINS))
def test_filter_boundary_is_exact(gpu, where):
    X, scans, rows, refs = _boundary_map(ORIGINS[where])
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 5, _lsq(e))
        e.set_map(X)
        a = e.register_to_map(scans, 4096, 10, params, max_overlap_distance=R_LAT * U, observed=rows)
        b = e.register_batch([(X, S) for S in scans], 4096, 10, params, max_overlap_distance=R_LAT * U,
                             observed=rows)
    assert np.array_equal(a.n_selected, b.n_selected), (a.n_selected, b.n_selected)
    for i, ref in enumerate(refs):
        if ref is None:
            assert 0 < a.n_selected[i] < 121, f"scan {i}: the sweep does not straddle the boundary"
        elif rows[i][2] == 0:
            assert a.n_selected[i] == ref[0], (i, a.n_selected[i], ref)
        else:
            # the Euler rotation of a multiple of 90 degrees is a permutation up to 1e-16: only
            # neighbours at exactly r may land on either side
            assert ref[0] <= a.n_selected[i] <= ref[0] + ref[1], (i, a.n_selected[i], ref)


# ------------------------------------------------------------------------- residency, API
def test_map_stays_resident(gpu):
    X, scans, rows = _data()
    pair = _map_and_scans(n_map=20_000, extent=30.0, seed=72_000)
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        with pytest.raises(_capi.SicpError) as ex:
            e.register_to_map(scans, 1000, 10, params, max_overlap_distance=1.0)
        assert ex.value.code == _capi.SICP_ERR_STATE
        e.set_map(X)
        a = e.register_to_map(scans, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        sb.register(pair[0], pair[1][0], engine=e, want_normals=False, max_overlap_distance=1.0)
        e.register_batch([(pair[0], S) for S in pair[1][:3]], 1000, 10, params, max_overlap_distance=1.0)
        b = e.register_to_map(scans, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        for i in range(len(scans)):
            assert _same_bits(a[i], b[i]), f"scan {i}"
        assert np.array_equal(a.n_selected, b.n_selected)
        # a new map replaces the old one
        e.set_map(pair[0])
        c = e.register_to_map(pair[1][:3], 1000, 10, params, max_overlap_distance=1.0)
        d = e.register_batch([(pair[0], S) for S in pair[1][:3]], 1000, 10, params, max_overlap_distance=1.0)
        for i in range(3):
            assert _same_bits(c[i], d[i]), f"scan {i}"
        e.set_map(None)
        with pytest.raises(_capi.SicpError) as ex:
            e.register_to_map(scans, 1000, 10, params)
        assert ex.value.code == _capi.SICP_ERR_STATE


def test_public_map_equals_simpleicp_batch(gpu):
    X, scans, rows = _data()
    kw = dict(max_overlap_distance=1.0, rbp_observed_values=rows)
    with sb.Map(X) as m:
        with pytest.raises(sb.BatchError) as ex:
            m.register(scans, batch_size=4, **kw)
        table = m.register(scans, batch_size=4, on_error="nan", **kw)
    ref = sb.simpleicp_batch([(X, S) for S in scans], on_error="nan", **kw)
    assert np.array_equal(table, ref, equal_nan=True)
    assert np.array_equal(ex.value.table, table, equal_nan=True)
    assert ex.value.failed.tolist() == [len(scans) - 1]
    assert table[-1, 16] == -_capi.SICP_ERR_NO_OVERLAP
    ok = slice(0, len(scans) - 1)
    with sb.Map(X) as m:
        assert np.array_equal(m.register(scans[ok], rbp_observed_values=rows[ok], max_overlap_distance=1.0,
                                         mov_neighbors=10, max_angle_between_normals=20.0),
                              sb.simpleicp_batch([(X, S) for S in scans[ok]], rbp_observed_values=rows[ok],
                                                 max_overlap_distance=1.0, mov_neighbors=10,
                                                 max_angle_between_normals=20.0))
