"""Host-side tests of the overlap graph: the argument checks of sb.overlap_graph, the NumPy
statement of the rule (tests/overlap_graph_rule.py) against a plain double loop, the sampled /
fraction arithmetic and the cap handling of the wrapper, and the C ABI declaration of
sicp_overlap_graph."""
import contextlib
import re
from pathlib import Path

import numpy as np
import pytest

import simpleicp_b200 as sb
from simpleicp_b200 import _capi, batch

import overlap_graph_rule as G

REPO = Path(__file__).resolve().parents[1]


def _rot(rng):
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return q * np.sign(np.linalg.det(q))


def _pose(rng, t=2.0):
    H = np.eye(4)
    H[:3, :3] = _rot(rng)
    H[:3, 3] = rng.uniform(-t, t, 3)
    return H


def _clouds(n=3, m=50):
    rng = np.random.default_rng(3)
    return [rng.normal(size=(m, 3)) for _ in range(n)]


_I3 = np.tile(np.eye(4), (3, 1, 1))


def _bad_row():
    H = _I3.copy()
    H[1, 3, 0] = 1e-3
    return H


def _skewed():
    H = _I3.copy()
    H[2, 0, 1] = 1e-5
    return H


class _Huge:
    """An (n, 3) array stand-in too large to allocate: only its shape is read before the check."""

    def __init__(self, n):
        self.shape = (n, 3)


@pytest.mark.parametrize("clouds,kw,msg", [
    ([], {}, "at least one cloud"),
    ([np.zeros((4, 2))], {}, "shape"),
    (None, {"H": np.tile(np.eye(4), (2, 1, 1))}, "H must have shape"),
    (None, {"H": _I3 * np.array([1, np.nan, 1])[:, None, None]}, "finite"),
    (None, {"H": _bad_row()}, "bottom row"),
    (None, {"H": _skewed()}, "orthonormal"),
    (None, {"max_distance": 0.0}, "max_distance"),
    (None, {"max_distance": -1.0}, "max_distance"),
    (None, {"max_distance": np.inf}, "max_distance"),
    (None, {"max_distance": np.nan}, "max_distance"),
    (None, {"stride": 0}, "stride"),
    (None, {"stride": 1.5}, "stride"),
    (None, {"stride": True}, "stride"),
    ([_Huge(1 << 31), _Huge(1 << 31)], {}, "2\\^32"),
])
def test_overlap_graph_argument_checks(clouds, kw, msg):
    kw = {"max_distance": 1.0, **kw}
    with pytest.raises(ValueError, match=msg):
        sb.overlap_graph(_clouds() if clouds is None else clouds, **kw)


def test_rotations_orthonormal_to_1e_6_are_accepted_by_the_check():
    H = _I3.copy()
    H[2, 0, 1] = 4e-7
    batch._check_rigid(H)


def _loop(clouds, H, r, s):
    """The rule by a plain double loop: squared distances ((dx dx + dy dy) + dz dz) < r r."""
    pairs, counts = [], []
    n = len(clouds)
    for a in range(n):
        for b in range(a + 1, n):
            c = []
            for x, y in ((a, b), (b, a)):
                T = G.relative(H, x, y)
                k = 0
                for q in G.queries(clouds[x], T, s):
                    for m in clouds[y]:
                        d = q - m
                        if (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] < r * r:
                            k += 1
                            break
                c.append(k)
            if sum(c):
                pairs.append((a, b))
                counts.append(c)
    return np.array(pairs, dtype=np.int64).reshape(-1, 2), np.array(counts, dtype=np.int64).reshape(-1, 2)


@pytest.mark.parametrize("with_poses", [False, True])
@pytest.mark.parametrize("s", [1, 3, 100])
def test_rule_matches_a_plain_double_loop(with_poses, s):
    rng = np.random.default_rng(7 + s)
    clouds = [rng.uniform(-2, 2, size=(m, 3)) for m in (60, 0, 45, 70, 30)]
    H = np.array([_pose(rng, 0.5) for _ in clouds])
    H[:, 0, 3] += 2.5 * np.arange(len(clouds))
    if not with_poses:  # the same clouds moved into one frame
        clouds, H = [X @ h[:3, :3].T + h[:3, 3] for X, h in zip(clouds, H)], None
    pairs, counts = G.overlap_graph(clouds, H, 0.6, s)
    ref_pairs, ref_counts = _loop(clouds, H, 0.6, s)
    assert np.array_equal(pairs, ref_pairs) and np.array_equal(counts, ref_counts)
    assert len(pairs) > 0 and not np.any(pairs == 1)  # the empty cloud takes part in no pair


class _FakeEngine:
    """Engine.overlap_graph's contract with a fixed answer: the total, and the first cap rows."""

    def __init__(self, pairs, counts):
        self.pairs, self.counts, self.caps = pairs, counts, []

    def overlap_graph(self, clouds, H, *, max_distance, stride, cap):
        self.caps.append(cap)
        return len(self.pairs), self.pairs[:cap], self.counts[:cap]


def test_sampled_fraction_and_the_second_call(monkeypatch):
    clouds = [np.zeros((m, 3)) for m in (10, 11, 0, 1)]
    n_rows = 8 * len(clouds) + 5  # more rows than the first call's capacity
    rng = np.random.default_rng(5)
    pairs = np.array([(0, 1)] * (n_rows - 2) + [(0, 3), (1, 3)], dtype=np.int64)
    counts = np.column_stack((rng.integers(0, 4, n_rows), rng.integers(0, 2, n_rows))).astype(np.int64)
    fake = _FakeEngine(pairs, counts)
    monkeypatch.setattr(batch, "_batch_engine", lambda device: fake)
    import torch

    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    g = sb.overlap_graph(clouds, max_distance=1.0, stride=4)
    assert fake.caps == [8 * len(clouds), n_rows]
    assert np.array_equal(g.sampled, [3, 3, 0, 1])  # ceil(n / 4)
    assert np.array_equal(g.pairs, pairs) and np.array_equal(g.counts, counts)
    assert np.array_equal(g.fraction[:, 0], counts[:, 0] / g.sampled[pairs[:, 0]])
    assert np.array_equal(g.fraction[:, 1], counts[:, 1] / g.sampled[pairs[:, 1]])
    assert g.fraction.dtype == np.float64 and g.fraction.shape == (n_rows, 2)


def test_abi_declares_the_overlap_graph_entry_point():
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    decl = re.search(r"int32_t sicp_overlap_graph\(([^;]*)\);", header)
    assert decl and "sicp_overlap_graph" in _capi.SYMBOLS
    # one parameter per ctypes argument type
    assert re.sub(r"/\*.*?\*/", "", decl.group(1)).count(",") + 1 == 13
