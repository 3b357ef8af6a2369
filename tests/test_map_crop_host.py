"""Map.crop and Map.thin without a device: the NumPy statements of both rules (checked against
plain loops, and the thin rule against the insert rule), the argument checks that fail before the
engine is reached, and the ABI declarations.

Crop: map point p is kept iff d2 = (dx dx + dy dy) + dz dz < fl(radius^2) for at least one centre
c, with d = p - c and every operation rounded in double (no fused multiply-add).
Thin: key(p) = floor(p / v) per axis (IEEE division, compared as doubles), the insert's key; map
point j is kept iff no map point j' < j has its key.
Both keep the kept points in their old order."""
import math
import re

import numpy as np
import pytest

from conftest import REPO
from test_map_insert_host import _NoEngine, insert_oracle, voxel_keys

from simpleicp_b200 import _capi, batch

O_UTM = np.array([612_345.0, 5_432_109.0, 250.0])
U = 2.0 ** -4  # lattice unit: dyadic, so lattice differences and their squares are exact


def crop_keep(P, C, r):
    """The crop rule's keep flags: NumPy evaluates every operation on its own, as the kernel does."""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    C = np.asarray(C, dtype=np.float64).reshape(-1, 3)
    d = P[:, None, :] - C[None, :, :]
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    r = float(r)
    return (d2 < r * r).any(axis=1)


def crop_oracle(P, C, r):
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    return P[crop_keep(P, C, r)]


def thin_oracle(M, v):
    """The first point of every voxel key, in map order."""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    _, first = np.unique(voxel_keys(M, v), axis=0, return_index=True)
    return M[np.sort(first)]


def _crop_loop(P, C, r):
    r2 = float(r) * float(r)
    keep = []
    for p in np.asarray(P, dtype=np.float64).reshape(-1, 3).tolist():
        hit = False
        for c in np.asarray(C, dtype=np.float64).reshape(-1, 3).tolist():
            dx, dy, dz = p[0] - c[0], p[1] - c[1], p[2] - c[2]
            if (dx * dx + dy * dy) + dz * dz < r2:
                hit = True
                break
        keep.append(hit)
    return np.array(keep, dtype=bool)


def _thin_loop(M, v):
    seen, out = set(), []
    for p in np.asarray(M, dtype=np.float64).reshape(-1, 3).tolist():
        k = tuple(float(math.floor(x / v)) + 0.0 for x in p)
        if k not in seen:
            seen.add(k)
            out.append(p)
    return np.array(out, dtype=np.float64).reshape(-1, 3)


def boundary_lattice(origin, m=5, span=7):
    """Centres on a dyadic lattice and the radius m U: the lattice points around each centre
    (several at d2 == r^2 exactly: m = 5 has (3, 4, 0) U and (5, 0, 0) U among them), each also
    moved one ulp down and up on every axis.  Returns (points, centres, radius)."""
    o = np.asarray(origin, dtype=np.float64)
    k = np.stack(np.meshgrid(*[np.arange(-span, span + 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    C = o + np.array([[0, 0, 0], [3, -2, 1], [40, 0, 0]]) * U  # two overlapping balls and a far one
    P = np.concatenate([o + k * U, C[2] + k[::5] * U])
    P = np.concatenate([P, np.nextafter(P, -np.inf), np.nextafter(P, np.inf)])
    return P, C, m * U


@pytest.mark.parametrize("origin", [np.zeros(3), O_UTM], ids=["origin", "utm"])
def test_crop_rule_equals_a_plain_loop_on_the_boundary_lattice(origin):
    P, C, r = boundary_lattice(origin)
    want = _crop_loop(P, C, r)
    assert np.array_equal(crop_keep(P, C, r), want)
    # the lattice really has points exactly on the sphere, kept one ulp inside and not on it
    d = P[:, None, :] - C[None, 0, :]
    d2 = ((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])[:, 0]
    on = d2 == r * r
    assert on.sum() >= 30 and 0 < want.sum() < len(P)
    # one centre alone at the origin: every point exactly at r is dropped
    assert not crop_keep(P[on], C[:1], r).any()


@pytest.mark.parametrize("origin", [np.zeros(3), O_UTM], ids=["origin", "utm"])
def test_crop_rule_with_random_points_and_far_centres(origin):
    rng = np.random.default_rng(11)
    P = origin + rng.uniform(-50, 50, (3000, 3))
    C = np.concatenate([origin + rng.uniform(-40, 40, (7, 3)), origin + [[1e4, 0, 0], [0, -1e4, 5]]])
    for r in (0.5, 7.0, 30.0, 1e5):
        assert np.array_equal(crop_keep(P, C, r), _crop_loop(P, C, r))
    assert crop_keep(P, C, 1e5).all() and not crop_keep(P, C[-2:], 1.0).any()


@pytest.mark.parametrize("v", [1.0, 0.3, 2.0 ** -7, 1e3])
def test_thin_rule_equals_the_insert_rule_and_a_loop(v):
    rng = np.random.default_rng(12)
    M = np.concatenate([rng.integers(-6, 6, (400, 3)) * v + rng.uniform(0, v, (400, 3)),
                        rng.integers(-8, 8, (60, 3)) * v])  # points exactly on voxel faces
    M = np.concatenate([M, np.nextafter(M[-60:], -np.inf), M[rng.integers(0, len(M), 50)]])  # one ulp below, duplicates
    got = thin_oracle(M, v)
    assert np.array_equal(got, insert_oracle(M[:1], [M[1:]], v)[0])
    assert np.array_equal(got, _thin_loop(M, v))
    assert len(got) < len(M) and np.array_equal(thin_oracle(got, v), got)


def test_thin_rule_zero_keys_and_utm():
    # -0.0 and +0.0 share key 0; UTM-scale coordinates with voxels of one ulp's multiple
    M = np.array([[0.0, 0.0, 0.0], [-0.0, 0.0, 0.0], [-5e-324, 0.0, 0.0], [0.5, 0.5, 0.5]])
    assert np.array_equal(thin_oracle(M, 1.0), M[[0, 2]])
    rng = np.random.default_rng(13)
    P = O_UTM + rng.integers(-200, 200, (5000, 3)) * U
    for v in (U, 4 * U, 0.3):
        assert np.array_equal(thin_oracle(P, v), _thin_loop(P, v))


def _map():
    m = batch.Map.__new__(batch.Map)
    m.device, m.n_points, m._engine = 0, 1000, _NoEngine()
    return m


@pytest.mark.parametrize("centers", [np.zeros(2), np.zeros((0, 3)), np.zeros((2, 2)), np.zeros((2, 3, 1)),
                                     np.zeros(6), [[1.0, 2.0]]])
def test_bad_centers_shape_raises(centers):
    with pytest.raises(ValueError, match="shape"):
        _map().crop(centers, radius=1.0)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_centers_raise(bad):
    c = np.zeros((3, 3))
    c[2, 1] = bad
    with pytest.raises(ValueError, match="finite"):
        _map().crop(c, radius=1.0)


@pytest.mark.parametrize("r", [0.0, -1.0, np.nan, np.inf, -np.inf])
def test_bad_radius_raises(r):
    with pytest.raises(ValueError, match="radius"):
        _map().crop(np.zeros(3), radius=r)


@pytest.mark.parametrize("v", [0.0, -1.0, np.nan, np.inf, -np.inf])
def test_bad_thin_voxel_size_raises(v):
    with pytest.raises(ValueError, match="voxel_size"):
        _map().thin(voxel_size=v)


def test_abi_declares_the_crop_and_thin_entry_points():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    for name in ("sicp_map_crop", "sicp_map_thin"):
        assert re.search(rf"int32_t {name}\(", header) and name in _capi.SYMBOLS
