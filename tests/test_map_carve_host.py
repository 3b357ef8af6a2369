"""Map.carve without a device: the NumPy statement of the carve rule (checked against a plain
per-ray, per-point loop), the argument checks that fail before the engine is reached, and the ABI
declarations.

The rule: every finite moved point p of cloud i is a ray from the origin o_i.  For a map point m,
with every operation one IEEE double operation rounded on its own (no fused multiply-add):
  d = p - o, u = m - o, L2 = (dx dx + dy dy) + dz dz, L = sqrt(L2),
  s = ((ux dx + uy dy) + uz dz) / L, e2 = ((ux ux + uy uy) + uz uz) - s s,
  the ray passes m iff L2 > 0, L2 finite, s > 0, s < L - margin and e2 < fl(r r).
passes[m] counts the rays of the call that pass m; m is removed iff passes[m] >= min_passes, and
the kept points keep their order."""
import math
import re

import numpy as np
import pytest

from conftest import REPO
from test_map_crop_host import O_UTM, U
from test_map_insert_host import _NoEngine

from simpleicp_b200 import _capi, batch


def carve_passes(M, O, P, r, margin, chunk=1 << 22):
    """passes (uint32, one per row of M) of the rays (O[k], P[k]), in chunks of rays of about
    `chunk` (ray, point) pairs; NumPy evaluates every operation on float64 arrays on its own."""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    O = np.asarray(O, dtype=np.float64).reshape(-1, 3)
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        d = P - O
        L2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        ray = np.isfinite(P).all(axis=1) & (L2 > 0) & np.isfinite(L2)
        O, d, L = O[ray], d[ray], np.sqrt(L2[ray])
        Lm = L - float(margin)
        r2 = float(r) * float(r)
        passes = np.zeros(len(M), dtype=np.int64)
        k = max(1, chunk // max(len(M), 1))
        for a in range(0, len(O), k):
            u = [M[None, :, i] - O[a:a + k, i, None] for i in range(3)]
            dd = [d[a:a + k, i, None] for i in range(3)]
            s = ((u[0] * dd[0] + u[1] * dd[1]) + u[2] * dd[2]) / L[a:a + k, None]
            e2 = ((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]) - s * s
            passes += ((s > 0) & (s < Lm[a:a + k, None]) & (e2 < r2)).sum(axis=0)
    return passes.astype(np.uint32)


def rays_of(clouds, origins):
    """(O, P): one row per point of the concatenated clouds, O its cloud's origin."""
    P = np.concatenate([np.asarray(X, dtype=np.float64).reshape(-1, 3) for X in clouds])
    O = np.repeat(np.asarray(origins, dtype=np.float64).reshape(-1, 3), [len(X) for X in clouds], axis=0)
    return O, P


def carve_oracle(M, clouds, origins, r, margin, min_passes=1):
    """(new map, passes) of carving map M with the (already moved) clouds from origins."""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    passes = carve_passes(M, *rays_of(clouds, origins), r, margin)
    return M[passes < min_passes], passes


def _carve_loop(M, O, P, r, margin):
    r2 = float(r) * float(r)
    out = []
    rays = []
    for o, p in zip(np.asarray(O, dtype=np.float64).tolist(), np.asarray(P, dtype=np.float64).tolist()):
        if not all(math.isfinite(x) for x in p):
            continue
        d = [p[i] - o[i] for i in range(3)]
        L2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
        if L2 > 0 and math.isfinite(L2):
            rays.append((o, d, math.sqrt(L2)))
    for m in np.asarray(M, dtype=np.float64).tolist():
        n = 0
        for o, d, L in rays:
            u = [m[i] - o[i] for i in range(3)]
            s = ((u[0] * d[0] + u[1] * d[1]) + u[2] * d[2]) / L
            e2 = ((u[0] * u[0] + u[1] * u[1]) + u[2] * u[2]) - s * s
            if s > 0 and s < L - margin and e2 < r2:
                n += 1
        out.append(n)
    return np.array(out, dtype=np.uint32)


def designed_carve(origin):
    """Dyadic geometry where the rule's boundaries are hit exactly: a lattice of map points along
    the x axis from the origin o at s = 0, 0.5, ..., 6 (= L - margin), ... with lateral offsets at
    e2 = 0, 9 U^2, r^2 = 25 U^2 (three ways) and 36 U^2, and copies one ulp off on x and on y;
    rays along +x (twice), along -x from the far end, diagonal, and rays that are none (zero
    length, NaN, inf, an empty cloud).  Returns (M, clouds, origins, r, margin)."""
    o = np.asarray(origin, dtype=np.float64)
    xs = np.arange(-2, 19) * 0.5
    lat = np.array([[0, 0], [3, 4], [4, 3], [5, 0], [0, -5], [3, 0], [6, 0], [-4, -3]]) * U
    B = o + np.array([[x, a, b] for x in xs for a, b in lat])
    parts = [B]
    for ax in (0, 1):
        for to in (-np.inf, np.inf):
            C = B.copy()
            C[:, ax] = np.nextafter(C[:, ax], to)
            parts.append(C)
    M = np.concatenate(parts)
    end = o + [8.0, 0.0, 0.0]
    bad = np.array([[np.nan, 0.0, 0.0], [0.0, np.inf, 0.0], [0.0, 0.0, -np.inf]]) + o
    clouds = [np.stack([end, end]),                            # two rays along +x: L = 8
              np.array([o + [-1.0, 0.0, 0.0]]),               # from the far end back past o
              np.array([o + [6.0, 6.0, 0.0], o + [5.0, 3.0, 4.0]]),  # diagonal rays
              np.concatenate([o[None], bad]),                 # zero length, NaN, inf: no rays
              np.zeros((0, 3))]
    origins = np.stack([o, end, o, o, o])
    return M, clouds, origins, 5 * U, 2.0


@pytest.mark.parametrize("origin", [np.zeros(3), O_UTM], ids=["origin", "utm"])
def test_rule_equals_a_plain_loop_on_the_designed_geometry(origin):
    M, clouds, origins, r, margin = designed_carve(origin)
    O, P = rays_of(clouds, origins)
    want = _carve_loop(M, O, P, r, margin)
    assert np.array_equal(carve_passes(M, O, P, r, margin), want)
    assert np.array_equal(carve_passes(M, O, P, r, margin, chunk=7), want)  # chunking does not matter
    # the boundaries are really hit, by the two rays along +x (L - margin = 6) and the one back
    # from x = 8 (s = 8 - x, L - margin = 7): e2 == r^2, s == L - margin and s == 0 are not
    # passed, one ulp inside is (s one ulp of m's x inside, e2 one ulp of r inside)
    o = np.asarray(origin)
    axis = carve_passes(M, *rays_of(clouds[:2], origins[:2]), r, margin)
    n = len(M) // 5
    B = M[:n]
    part = [axis[i * n:(i + 1) * n] for i in range(5)]  # B, x down, x up, y down, y up
    on_axis = (B[:, 1] == o[1]) & (B[:, 2] == o[2])
    on_tube = (B[:, 1] - o[1] == 5 * U) & (B[:, 2] == o[2])  # e2 = r^2 exactly
    inner = (B[:, 0] - o[0] > 1.0) & (B[:, 0] - o[0] < 6.0)
    at_end, at_start = on_axis & (B[:, 0] - o[0] == 6.0), on_axis & (B[:, 0] == o[0])
    assert at_end.sum() == 1 and at_start.sum() == 1 and (on_axis & inner).sum() == 9
    assert (part[0][on_axis & inner] == 3).all()
    assert (part[0][on_tube & inner] == 0).all() and (part[4][on_tube & inner] == 0).all()
    # e2 == r^2 is passed with r one ulp up (a lateral ulp of m vanishes in e2's cancellation)
    up = carve_passes(M[:n], *rays_of(clouds[:2], origins[:2]), np.nextafter(r, np.inf), margin)
    assert (up[on_tube & inner] == 3).all()
    assert part[0][at_end] == 1 and part[1][at_end] == 3 and part[2][at_end] == 1
    assert part[0][at_start] == 0 and part[1][at_start] == 0 and part[2][at_start] == 2
    # rays that are none: a cloud of only them changes nothing
    assert not carve_passes(M, *rays_of(clouds[3:], origins[3:]), r, margin).any()


@pytest.mark.parametrize("origin", [np.zeros(3), O_UTM], ids=["origin", "utm"])
@pytest.mark.parametrize("r", [0.05, 0.7, 6.0])
def test_rule_with_random_rays(origin, r):
    rng = np.random.default_rng(31)
    O = origin + rng.uniform(-12, 12, (60, 3))
    P = np.concatenate([origin + rng.uniform(-10, 10, (50, 3)), O[50:]])  # the last rays have length 0
    # random points, and points near the rays at about the tube's radius
    near = O[:50] + rng.uniform(-0.2, 1.2, (50, 1)) * (P[:50] - O[:50]) + rng.normal(0, r, (50, 3))
    M = np.concatenate([origin + rng.uniform(-10, 10, (400, 3)), near])
    for margin in (0.0, 0.5, 30.0):
        want = _carve_loop(M, O, P, r, margin)
        assert np.array_equal(carve_passes(M, O, P, r, margin, chunk=1000), want)
    assert want.sum() == 0  # margin 30: no ray is long enough
    assert _carve_loop(M, O, P, r, 0.0).sum() > 0


def test_oracle_removes_the_points_with_enough_passes():
    M, clouds, origins, r, margin = designed_carve(np.zeros(3))
    passes = carve_passes(M, *rays_of(clouds, origins), r, margin)
    for k in (1, 2, 3, 4):
        got, p = carve_oracle(M, clouds, origins, r, margin, k)
        assert np.array_equal(p, passes) and np.array_equal(got, M[passes < k])
    assert 0 < (passes >= 2).sum() < (passes >= 1).sum() < len(M)


def _map():
    m = batch.Map.__new__(batch.Map)
    m.device, m.n_points, m._engine = 0, 1000, _NoEngine()
    return m


CLOUDS = [np.zeros((5, 3)), np.ones((2, 3))]
OR = np.zeros((2, 3))


@pytest.mark.parametrize("r", [0.0, -1.0, np.nan, np.inf, -np.inf])
def test_bad_radius_raises(r):
    with pytest.raises(ValueError, match="radius"):
        _map().carve(CLOUDS, origins=OR, radius=r, margin=0.0)


@pytest.mark.parametrize("margin", [-1e-300, -1.0, np.nan, np.inf, -np.inf])
def test_bad_margin_raises(margin):
    with pytest.raises(ValueError, match="margin"):
        _map().carve(CLOUDS, origins=OR, radius=1.0, margin=margin)


@pytest.mark.parametrize("k", [0, -1, 1.5, True, 1 << 31])
def test_bad_min_passes_raises(k):
    with pytest.raises(ValueError, match="min_passes"):
        _map().carve(CLOUDS, origins=OR, radius=1.0, margin=0.0, min_passes=k)


@pytest.mark.parametrize("origins", [np.zeros((1, 3)), np.zeros((2, 2)), np.zeros(6), np.zeros((3, 3))])
def test_bad_origins_shape_raises(origins):
    with pytest.raises(ValueError, match="shape"):
        _map().carve(CLOUDS, origins=origins, radius=1.0, margin=0.0)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_origins_or_H_raise(bad):
    o = OR.copy()
    o[1, 2] = bad
    with pytest.raises(ValueError, match="finite"):
        _map().carve(CLOUDS, origins=o, radius=1.0, margin=0.0)
    H = np.tile(np.eye(4), (2, 1, 1))
    H[0, 1, 3] = bad
    with pytest.raises(ValueError, match="finite"):
        _map().carve(CLOUDS, H, radius=1.0, margin=0.0)


def test_no_origins_and_no_H_raises():
    with pytest.raises(ValueError, match="origins"):
        _map().carve(CLOUDS, radius=1.0, margin=0.0)


@pytest.mark.parametrize("H", [np.zeros((2, 4, 3)), np.zeros((1, 4, 4)), np.zeros((2, 16))])
def test_bad_H_shape_raises(H):
    with pytest.raises(ValueError, match="shape"):
        _map().carve(CLOUDS, H, radius=1.0, margin=0.0)


@pytest.mark.parametrize("cloud", [np.zeros((5, 2)), np.zeros(6), [1.0, 2.0, 3.0]])
def test_bad_cloud_raises(cloud):
    with pytest.raises(ValueError, match=r"\(n, 3\)"):
        _map().carve([np.zeros((4, 3)), cloud], origins=OR, radius=1.0, margin=0.0)


def test_no_cloud_raises():
    with pytest.raises(ValueError, match="at least one"):
        _map().carve([], origins=np.zeros((0, 3)), radius=1.0, margin=0.0)


def test_abi_declares_the_carve_entry_point():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    assert re.search(r"int32_t sicp_map_carve\(", header) and "sicp_map_carve" in _capi.SYMBOLS
