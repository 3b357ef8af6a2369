"""sb.Map and the map bindings without a device: argument and key checks, the 32-bit limit on
scans per library call, ABI declarations."""
import re

import numpy as np
import pytest

from conftest import REPO

from simpleicp_b200 import _capi, batch
from simpleicp_b200.simpleicp import SimpleICPException


class _NoEngine:
    """An engine that must not be reached: the arguments fail first."""

    alive = True

    def __getattr__(self, name):
        raise AssertionError(f"the engine was reached ({name}) before the arguments were checked")


def _map(n_points=1000):
    m = batch.Map.__new__(batch.Map)
    m.device, m.n_points, m._engine = 0, n_points, _NoEngine()
    return m


SCANS = [np.zeros((5, 3))] * 3


@pytest.mark.parametrize("key", ["want_normals", "mov_normals", "engine", "debug"])
def test_unsupported_keys_raise(key):
    with pytest.raises(TypeError, match=key):
        _map().register(SCANS, **{key: 1})


def test_too_many_correspondences_raise():
    with pytest.raises(ValueError, match="4096"):
        _map().register(SCANS, correspondences=5000)


@pytest.mark.parametrize("obs", [np.zeros((2, 6)), np.zeros((3, 5)), 0.0])
def test_bad_rows_raise(obs):
    with pytest.raises(SimpleICPException, match="shape"):
        _map().register(SCANS, rbp_observed_values=obs, max_overlap_distance=1.0)


def test_invalid_rows_and_mov_arguments_raise():
    rows = np.zeros((3, 6))
    rows[1, 2] = np.inf
    with pytest.raises(SimpleICPException, match="finite"):
        _map().register(SCANS, rbp_observed_values=rows)
    with pytest.raises(SimpleICPException):
        _map().register(SCANS, max_angle_between_normals=10.0)  # needs mov_neighbors
    with pytest.raises(SimpleICPException):
        _map().register(SCANS, mov_neighbors=1)


def test_map_keys_are_the_batch_keys_without_debug_output():
    assert batch._MAP_KEYS == batch._BATCH_KEYS - {"want_normals"}


@pytest.mark.parametrize("n_points,batch_size,expect", [(1000, 64, 64), (1 << 28, 64, 15), (1 << 31, 64, 1),
                                                       (1 << 26, 8, 8)])
def test_scans_per_call_keep_offsets_32_bit(monkeypatch, n_points, batch_size, expect):
    seen = {}

    def fake(get, mine, local, device, per_call, kw, messages, rows=None, map_engine=None):
        seen["per_call"] = per_call
        assert map_engine is not None

    monkeypatch.setattr(batch, "_run_batched", fake)
    _map(n_points).register(SCANS, batch_size=batch_size)
    assert seen["per_call"] == expect
    assert expect * n_points < 2 ** 32


def test_abi_declares_the_map_entry_points():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    for name in ("sicp_set_map", "sicp_register_to_map"):
        assert re.search(rf"int32_t {name}\(", header) and name in _capi.SYMBOLS
    # overlap_candidates is appended: every earlier field keeps its offset
    names = [n for n, _ in _capi.Timings._fields_]
    assert names[-1] == "overlap_candidates" and names[-2] == "mov_normals_ms"
    assert re.search(r"int64_t overlap_candidates;[^}]*\} sicp_timings;", header, re.S)
