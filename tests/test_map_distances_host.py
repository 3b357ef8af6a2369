"""Map.distances without a device: the argument checks that fail before the engine is reached,
fitness and RMSE against a plain loop, and the ABI declaration of sicp_map_distances."""
import math
import re

import numpy as np
import pytest

from conftest import REPO
from test_map_insert_host import CLOUDS, _map

from simpleicp_b200 import _capi, batch


@pytest.mark.parametrize("r", [0.0, -1.0, np.nan, np.inf, -np.inf])
def test_bad_max_distance_raises(r):
    with pytest.raises(ValueError, match="max_distance"):
        _map().distances(CLOUDS, max_distance=r)


@pytest.mark.parametrize("k", [0, 1, 65, 1001])  # the map of _map() has 1000 points
def test_bad_neighbors_raises(k):
    with pytest.raises(ValueError, match="neighbors"):
        _map().distances(CLOUDS, max_distance=1.0, neighbors=k)


@pytest.mark.parametrize("H", [np.zeros((2, 4, 3)), np.zeros((1, 4, 4)), np.zeros((3, 4, 4)), np.zeros((2, 16))])
def test_bad_H_shape_raises(H):
    with pytest.raises(ValueError, match="shape"):
        _map().distances(CLOUDS, H, max_distance=1.0)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_H_raises(bad):
    H = np.tile(np.eye(4), (2, 1, 1))
    H[0, 2, 1] = bad
    with pytest.raises(ValueError, match="finite"):
        _map().distances(CLOUDS, H, max_distance=1.0)


@pytest.mark.parametrize("cloud", [np.zeros((5, 2)), np.zeros(6), np.zeros((2, 3, 1)), [1.0, 2.0, 3.0]])
def test_bad_cloud_raises(cloud):
    with pytest.raises(ValueError, match=r"\(n, 3\)"):
        _map().distances([np.zeros((4, 3)), cloud], max_distance=1.0)


def test_no_cloud_raises():
    with pytest.raises(ValueError, match="at least one"):
        _map().distances([], max_distance=1.0, neighbors=10)


def _loop_fit(index, dist2):
    n, inside, total = len(index), 0, 0.0
    for i, d in zip(index.tolist(), dist2.tolist()):
        if i >= 0:
            inside += 1
            total += d
    fitness = inside / n if n else math.nan
    rmse = math.sqrt(total / inside) if inside else math.nan
    return inside, fitness, rmse


@pytest.mark.parametrize("seed", range(4))
def test_fitness_and_rmse_equal_a_plain_loop(seed):
    rng = np.random.default_rng(seed)
    for n in (0, 1, 7, 1000):
        index = rng.integers(-1, 50, n)
        index[rng.random(n) < 0.3] = -1
        dist2 = np.where(index >= 0, rng.uniform(0, 0.25, n), np.inf)
        dist2[(index < 0) & (rng.random(n) < 0.3)] = np.nan  # non-finite points
        inside, fitness, rmse = _loop_fit(index, dist2)
        got = batch.CloudDistances.of(index, dist2, None, None, inside)
        assert got.n_within == inside
        assert (math.isnan(fitness) and math.isnan(got.fitness)) or got.fitness == fitness
        assert (math.isnan(rmse) and math.isnan(got.rmse)) or got.rmse == pytest.approx(rmse, rel=1e-14)
        assert np.array_equal(got.distance, np.sqrt(dist2), equal_nan=True)
        assert np.all(np.isinf(got.distance[(index < 0) & ~np.isnan(dist2)]))


def test_no_within_point_gives_nan_rmse_and_zero_fitness():
    got = batch.CloudDistances.of(np.full(5, -1), np.full(5, np.inf), None, None, 0)
    assert got.fitness == 0.0 and math.isnan(got.rmse)


def test_abi_declares_map_distances():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    assert re.search(r"int32_t sicp_map_distances\(", header) and "sicp_map_distances" in _capi.SYMBOLS
    src = (REPO / "simpleicp_b200" / "_capi.py").read_text()
    decl = re.search(r'"sicp_map_distances": \[(.*?)\],\n', src, re.S).group(1)
    assert len([a for a in decl.split(",") if a.strip()]) == 12  # ctx, n_clouds, xyz, n, H, r, k, 4 arrays, n_within


class _RecordingEngine:
    """Answers map_distances with every point within (index 0, d2 0.25) and records the call."""

    alive = True

    def __init__(self):
        self.calls = []

    def map_distances(self, clouds, H, *, max_distance, neighbors):
        self.calls.append((clouds, H, max_distance, neighbors))
        n = [len(X) for X in clouds]
        return ([np.zeros(k, np.int64) for k in n], [np.full(k, 0.25) for k in n], None, None,
                np.array(n, dtype=np.int64))


def test_the_readme_call_shape_with_a_scan_that_failed(monkeypatch):
    import contextlib

    import torch

    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())  # no device needed here
    # the table of Map.register(..., on_error="nan"): scan 1 did not register, its record is NaN
    scans = [np.zeros((5, 3)), np.ones((4, 3)), np.full((3, 3), 2.0)]
    t = np.zeros((3, 20))
    t[:, :16] = np.eye(4).reshape(16)
    t[:, 16] = [7, -2, 9]
    t[1, :16] = np.nan
    t[1, 17:] = np.nan
    m = _map()
    with pytest.raises(ValueError, match="finite"):  # all rows: the failed scan's NaN H is refused
        m.distances(scans, t[:, :16].reshape(-1, 4, 4), max_distance=0.5)
    m._engine = _RecordingEngine()
    ok = [i for i in range(len(scans)) if t[i, 16] > 0]
    fit = m.distances([scans[i] for i in ok], t[ok, :16].reshape(-1, 4, 4), max_distance=0.5)
    ok = [i for i, d in zip(ok, fit) if d.fitness > 0.9]
    (clouds, H, r, k), = m._engine.calls
    assert ok == [0, 2] and [len(X) for X in clouds] == [5, 3] and r == 0.5 and k == 0
    assert H.shape == (2, 4, 4) and np.isfinite(H).all()
    assert [d.rmse for d in fit] == [0.5, 0.5] and [d.fitness for d in fit] == [1.0, 1.0]
