"""Map.insert without a device: the NumPy statement of the insert rule (checked against a plain
loop), the argument checks that fail before the engine is reached, and the ABI declarations.

The rule: C is the clouds concatenated in order; key(p) = floor(p / v) per axis (IEEE division,
compared as doubles); C[j] is added iff it is finite, no map point has its key and no finite
C[j'] with j' < j has it.  The new map is the old one followed by the added points in order."""
import math
import re

import numpy as np
import pytest

from conftest import REPO

from simpleicp_b200 import _capi, batch


def voxel_keys(P, v):
    """floor(P / v) per coordinate; + 0.0 makes a -0.0 key the +0.0 one, as a double compare does."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.floor(np.asarray(P, dtype=np.float64).reshape(-1, 3) / v) + 0.0


def insert_oracle(M, clouds, v):
    """(new map, points added per cloud) of inserting `clouds` (already moved) into map `M`."""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    C = np.concatenate([np.asarray(X, dtype=np.float64).reshape(-1, 3) for X in clouds])
    owner = np.repeat(np.arange(len(clouds)), [len(X) for X in clouds])
    fin = np.flatnonzero(np.isfinite(C).all(axis=1))
    # the first row of every distinct key over [map keys; new keys]: a new point is first of its
    # key exactly when no map point and no earlier new point has that key
    _, first = np.unique(np.concatenate([voxel_keys(M, v), voxel_keys(C[fin], v)]), axis=0, return_index=True)
    add = fin[np.sort(first[first >= len(M)]) - len(M)]
    return np.concatenate([M, C[add]]), np.bincount(owner[add], minlength=len(clouds)).astype(np.int64)


def _loop_oracle(M, clouds, v):
    def key(p):
        return tuple(float(math.floor(x / v)) if math.isfinite(x / v) else x / v for x in p)

    taken = {key(p) for p in M.tolist()}
    out, counts = M.tolist(), []
    for X in clouds:
        k = 0
        for p in np.asarray(X, dtype=np.float64).reshape(-1, 3).tolist():
            if all(math.isfinite(x) for x in p) and key(p) not in taken:
                taken.add(key(p))
                out.append(p)
                k += 1
        counts.append(k)
    return np.array(out, dtype=np.float64).reshape(-1, 3), np.array(counts, dtype=np.int64)


def designed_clouds(v, seed=0):
    """A map on a lattice of voxel corners and clouds with points on voxel faces and one ulp off
    them, negative coordinates, duplicates of map points, many points in one voxel, NaN / inf
    points, an empty cloud and points far outside the map."""
    rng = np.random.default_rng(seed)
    M = rng.integers(-6, 6, (40, 3)) * v + rng.uniform(0, v, (40, 3))
    faces = rng.integers(-8, 8, (60, 3)) * v
    lo = np.nextafter(faces, -np.inf)
    hi = np.nextafter(faces, np.inf)
    dup = M[rng.integers(0, len(M), 10)]
    crowd = np.full((12, 3), 2.5 * v) + rng.uniform(0, 0.4 * v, (12, 3))
    bad = rng.uniform(-3 * v, 3 * v, (6, 3))
    bad[0, 0], bad[1, 1], bad[2, 2], bad[3] = np.nan, np.inf, -np.inf, np.nan
    far = rng.uniform(-1, 1, (5, 3)) * v + 1e4 * v
    return M, [faces, lo, np.zeros((0, 3)), np.concatenate([hi, dup]), crowd, bad, far, -faces]


@pytest.mark.parametrize("v", [1.0, 0.3, 2.0 ** -7, 1e3])
def test_oracle_equals_a_plain_loop(v):
    M, clouds = designed_clouds(v)
    got, counts = insert_oracle(M, clouds, v)
    want, want_counts = _loop_oracle(M, clouds, v)
    assert np.array_equal(got, want) and np.array_equal(counts, want_counts)
    assert counts[2] == 0 and counts.sum() == len(got) - len(M)


def test_oracle_zero_and_overflowing_keys():
    # -0.0 has the map's key 0; at v = 1e10 the negative subnormal's quotient rounds to -0.0 (key
    # 0 too), at v = 1e-10 it does not (key -1) and the two large points' quotients overflow to
    # the same key (inf, 0, 0), so only the first of them is added
    M = np.array([[0.0, 0.0, 0.0]])
    C = np.array([[-0.0, 0.0, 0.0], [-5e-324, 0.0, 0.0], [1e308, 0.0, 0.0], [1.5e308, 0.0, 0.0]])
    for v, rows in ((1e10, [2, 3]), (1e-10, [1, 2])):
        got, counts = insert_oracle(M, [C], v)
        want, want_counts = _loop_oracle(M, [C], v)
        assert np.array_equal(got, want) and np.array_equal(counts, want_counts)
        assert np.array_equal(got, np.concatenate([M, C[rows]]))


class _NoEngine:
    """An engine that must not be reached: the arguments fail first."""

    alive = True

    def __getattr__(self, name):
        raise AssertionError(f"the engine was reached ({name}) before the arguments were checked")


def _map():
    m = batch.Map.__new__(batch.Map)
    m.device, m.n_points, m._engine = 0, 1000, _NoEngine()
    return m


CLOUDS = [np.zeros((5, 3)), np.ones((2, 3))]


@pytest.mark.parametrize("v", [0.0, -1.0, np.nan, np.inf, -np.inf])
def test_bad_voxel_size_raises(v):
    with pytest.raises(ValueError, match="voxel_size"):
        _map().insert(CLOUDS, voxel_size=v)


@pytest.mark.parametrize("H", [np.zeros((2, 4, 3)), np.zeros((1, 4, 4)), np.zeros((3, 4, 4)), np.zeros((2, 16))])
def test_bad_H_shape_raises(H):
    with pytest.raises(ValueError, match="shape"):
        _map().insert(CLOUDS, H, voxel_size=1.0)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_H_raises(bad):
    H = np.tile(np.eye(4), (2, 1, 1))
    H[1, 0, 3] = bad
    with pytest.raises(ValueError, match="finite"):
        _map().insert(CLOUDS, H, voxel_size=1.0)


@pytest.mark.parametrize("cloud", [np.zeros((5, 2)), np.zeros(6), np.zeros((2, 3, 1)), [1.0, 2.0, 3.0]])
def test_bad_cloud_raises(cloud):
    with pytest.raises(ValueError, match=r"\(n, 3\)"):
        _map().insert([np.zeros((4, 3)), cloud], voxel_size=1.0)


def test_no_cloud_raises():
    with pytest.raises(ValueError, match="at least one"):
        _map().insert([], voxel_size=1.0)


def test_abi_declares_the_insert_entry_points():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    for name in ("sicp_map_insert", "sicp_get_map"):
        assert re.search(rf"int32_t {name}\(", header) and name in _capi.SYMBOLS
    names = [n for n, _ in _capi.Timings._fields_]
    assert names[-1] == "overlap_candidates"
