"""Host-side checks of the movable-normals keywords (mov_neighbors, max_angle_between_normals):
batch routing and argument errors raised before any device work."""
import numpy as np
import pytest

import simpleicp_b200 as sb
from simpleicp_b200 import batch


def _pairs(n=3):
    rng = np.random.default_rng(3)
    return [(rng.uniform(0, 10, (200, 3)), rng.uniform(0, 10, (150, 3))) for _ in range(n)]


def test_batchable_accepts_the_movable_keys():
    assert batch._batchable({"mov_neighbors": 10})
    assert batch._batchable({"mov_neighbors": 10, "max_angle_between_normals": 20.0, "correspondences": 500})
    assert not batch._batchable({"mov_neighbors": 10, "mov_normals": None})


def _never(*a, **kw):
    raise AssertionError("a registration started")


@pytest.mark.parametrize("kw", [{"max_angle_between_normals": 20.0},
                                {"mov_neighbors": 1},
                                {"mov_neighbors": 65},
                                {"mov_neighbors": 2.5},
                                {"mov_neighbors": 10, "max_angle_between_normals": 91.0}])
def test_batch_checks_before_any_registration(kw):
    with pytest.raises(sb.SimpleICPException):
        sb.simpleicp_batch(_pairs(), register_fn=_never, **kw)
    with pytest.raises(sb.SimpleICPException):
        sb.simpleicp_batch(_pairs(), **kw)


def test_batch_message_names_mov_neighbors():
    with pytest.raises(sb.SimpleICPException, match="needs the normals of the movable.*mov_neighbors=k"):
        sb.simpleicp_batch(_pairs(), register_fn=_never, max_angle_between_normals=20.0)


def test_injected_register_fn_receives_the_keywords():
    seen = []

    class R:
        H = np.eye(4)
        iterations = 1
        records = [{"n_kept": 6, "mean_res": 0.0, "std_res": 0.0}]

    def fn(Xf, Xm, **kw):
        seen.append(kw)
        return R()

    sb.simpleicp_batch(_pairs(2), register_fn=fn, mov_neighbors=10, max_angle_between_normals=20.0)
    assert seen == [{"mov_neighbors": 10, "max_angle_between_normals": 20.0}] * 2


@pytest.mark.parametrize("kw,msg", [
    ({"mov_neighbors": 1}, "within \\[2, 64\\]"),
    ({"mov_neighbors": 65}, "within \\[2, 64\\]"),
    ({"mov_neighbors": 31}, "exceeds the number of points"),
    ({"mov_neighbors": 10, "mov_normals": (np.zeros(30),) * 4}, "either mov_normals or mov_neighbors"),
    ({"max_angle_between_normals": 10.0}, "needs the normals of the movable"),
    ({"mov_neighbors": 10, "max_angle_between_normals": 120.0}, "within \\[0, 90\\]"),
])
def test_facade_errors_before_device_work(kw, msg, monkeypatch):
    import importlib

    facade = importlib.import_module("simpleicp_b200.simpleicp")

    monkeypatch.setattr(facade, "default_engine", _never)
    Xf, Xm = _pairs(1)[0]
    Xm = Xm[:30]
    with pytest.raises(sb.SimpleICPException, match=msg):
        sb.register(Xf, Xm, **kw)
    with pytest.raises(sb.SimpleICPException, match=msg):
        sb.simpleicp(Xf, Xm, **kw)
