"""Movable-side attributes estimated on the device (sicp_register_params.mov_neighbors): the one
library call against the reference's class route (pc_mov.estimate_normals(k), then run()), against
the staged route with the same normals handed in, edge cases, and the batched engine against
sicp_register pair by pair."""
import numpy as np
import pytest

from conftest import load_golden, load_pair
from test_gpu_parity import _surface_pairs

import simpleicp_b200 as sb
from simpleicp_b200 import _capi, pointcloud
from simpleicp_b200.linearized import VARIANT_LINEARIZED
from simpleicp_b200.simpleicp import _observed_in_radians
from simpleicp_b200.synthetic import c3_pair

pytestmark = pytest.mark.gpu

_INPUTS = {}


def _input(name):
    """(X_fix, X_mov, register kwargs) of a test input."""
    if name not in _INPUTS:
        if name == "dragon":
            _INPUTS[name] = (*load_pair("dragon"), {})
        elif name == "bunny_overlap":
            _INPUTS[name] = (*load_pair("bunny"), {"max_overlap_distance": 1.0})
        else:  # the C3 geometry at 200 000 points
            X_fix, X_mov, _ = c3_pair(200_000)
            _INPUTS[name] = (X_fix, X_mov, {})
    return _INPUTS[name]


def _same(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def _assert_same_run(r, s, what):
    assert r.iterations == s.iterations and r.converged == s.converged, what
    assert len(r.records) == len(s.records), what
    for i, (a, b) in enumerate(zip(r.records, s.records)):
        for key in a:
            if key in ("lm_iterations", "n_bruteforce"):
                continue  # the staged loop reports them the same way; compared anyway below
            assert _same(a[key], b[key]), f"{what}: iteration {i} field {key}: {a[key]} vs {b[key]}"
        assert a["lm_iterations"] == b["lm_iterations"] and a["n_bruteforce"] == b["n_bruteforce"], what
    assert _same(r.H, s.H), what
    assert _same(r.residuals, s.residuals), what
    assert _same(np.asarray(r.X_mov_transformed), np.asarray(s.X_mov_transformed)), what


def test_one_call_equals_class_route(gpu):
    """simpleicp(..., mov_neighbors=10) is the reference's pc_mov.estimate_normals(10) + run()."""
    g = load_golden("dragon_movnormals")
    X_fix, X_mov = load_pair("dragon_movnormals")
    H, X_t, _, res = sb.simpleicp(X_fix, X_mov, mov_neighbors=10)
    pc_fix, pc_mov = sb.PointCloud(X_fix, columns=["x", "y", "z"]), sb.PointCloud(X_mov, columns=["x", "y", "z"])
    pc_mov.estimate_normals(10)
    icp = sb.SimpleICP(verbose=False)
    icp.add_point_clouds(pc_fix, pc_mov)
    H_c, X_c, _, res_c = icp.run()
    assert np.array_equal(H, H_c)
    assert np.array_equal(res, res_c)
    assert np.array_equal(np.asarray(X_t), np.asarray(X_c))
    r = sb.register(X_fix, X_mov, mov_neighbors=10, want_normals=False)
    kept = [rec["n_kept"] for rec in r.records]
    ref_kept = [int(k.sum()) for k in g["it_keep"]]
    dH = np.linalg.norm(r.H - g["H"])
    print(f"mov_neighbors=10: |dH|_F = {dH:.3e}, kept {kept} vs {ref_kept}, "
          f"mov_normals_ms {r.timings['mov_normals_ms']:.3f}")
    assert dH < 1e-5
    assert r.iterations == len(ref_kept)
    assert max(abs(a - b) for a, b in zip(kept, ref_kept)) <= 3
    assert r.timings["mov_normals_ms"] > 0


@pytest.mark.parametrize("k", [3, 10, 16, 17, 40])
@pytest.mark.parametrize("name", ["dragon", "bunny_overlap", "c3_200k"])
def test_one_call_equals_staged_route(gpu, name, k):
    """register(mov_neighbors=k) in one sicp_register call against register(mov_normals=<the
    same cloud's PointCloud.estimate_normals(k)>) through the stages: equal bit for bit, under
    every k-NN kernel choice, angle limit and reject/solve kernel."""
    X_fix, X_mov, kw = _input(name)
    mov = pointcloud.estimate_normals_of(X_mov, None, k)
    coops = (-1, 0, 1, 2) if k <= 16 else (-1, 0)
    angles = (None, 5.0, 20.0, 90.0)

    def run(e, **kwa):
        # a registration that runs out of correspondences (a narrow angle on a noisy small-k
        # estimate) must do so alike on both routes: the exception's message is compared
        try:
            return sb.register(X_fix, X_mov, max_angle_between_normals=kwa.pop("angle"), engine=e, **kw, **kwa)
        except sb.SimpleICPException as ex:
            return str(ex)

    staged = {}
    with _capi.Engine() as e:
        for angle in angles:
            for fused in (1, 0):
                e.reset_options()
                e.set_option("fused", fused)
                staged[angle, fused] = run(e, mov_normals=mov, angle=angle)
        for coop in coops:
            for angle in angles:
                for fused in (1, 0):
                    e.reset_options()
                    e.set_option("fused", fused)
                    e.set_option("knn_coop", coop)
                    r = run(e, mov_neighbors=k, angle=angle, want_normals=False)
                    what = f"{name} k={k} knn_coop={coop} angle={angle} fused={fused}"
                    s = staged[angle, fused]
                    if isinstance(s, str):
                        assert r == s, what
                        continue
                    assert not isinstance(r, str), f"{what}: {r}"
                    assert e.timings()["mov_normals_ms"] > 0
                    _assert_same_run(r, s, what)
    kept = {a: staged[a, 1].records[0]["n_kept"] for a in angles if not isinstance(staged[a, 1], str)}
    print(f"{name} k={k}: first-iteration kept by angle limit {kept}")
    assert None in kept and 90.0 in kept and kept[90.0] <= kept[None]


def test_duplicate_points_are_rejected_alike(gpu):
    """k copies of one movable point: planarity NaN there (l_max = 0), which fails the planarity
    test on both routes.  The point is rounded to 2^-10 and k = 16 so that the neighbourhood's mean
    is the point itself in floating point and the covariance is exactly zero."""
    X_fix, X_mov = load_pair("bunny")
    X_mov = X_mov.copy()
    X_mov[100:120] = np.round(X_mov[100] * 1024.0) / 1024.0
    k = 16
    mov = pointcloud.estimate_normals_of(X_mov, None, k)
    assert np.isnan(mov[3][100:120]).all()
    with _capi.Engine() as e:
        a = sb.register(X_fix, X_mov, mov_neighbors=k, want_normals=False, engine=e)
        b = sb.register(X_fix, X_mov, mov_normals=mov, engine=e)
    _assert_same_run(a, b, "duplicates")


def test_bad_mov_neighbors(gpu):
    X_fix, X_mov = load_pair("bunny")
    with _capi.Engine() as e:
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        params = e.run_params(0.3, 1.0, 100, lsq)
        for k in (1, 65, -3):
            with pytest.raises(_capi.SicpError) as ei:
                e.register_fused(X_fix, X_mov, 1000, 10, -1.0, params, mov_neighbors=k)
            assert ei.value.code == _capi.SICP_ERR_BAD_ARG
        with pytest.raises(_capi.SicpError) as ei:
            e.register_fused(X_fix, X_mov[:5], 1000, 10, -1.0, params, mov_neighbors=6)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG
        with pytest.raises(_capi.SicpError) as ei:
            e.register_fused(X_fix, X_mov, 1000, 10, -1.0, params, mov_neighbors=10, max_angle_rad=2.0)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG
        e.set_option("variant", VARIANT_LINEARIZED)
        with pytest.raises(_capi.SicpError) as ei:
            e.register_fused(X_fix, X_mov, 1000, 10, -1.0, params, mov_neighbors=10)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG
        with pytest.raises(_capi.SicpError) as ei:
            e.register_batch([(X_fix, X_mov)], 1000, 10, params, mov_neighbors=10)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG
        # the context is still usable after the refusals
        e.reset_options()
        r = sb.register(X_fix, X_mov, mov_neighbors=10, want_normals=False, engine=e)
        assert r.iterations >= 1
    with pytest.raises(sb.SimpleICPException):
        sb.simpleicp(X_fix, X_mov, mov_neighbors=10, mov_normals=pointcloud.estimate_normals_of(X_mov, None, 10))


def _ragged_pairs():
    """Ragged surface pairs cropped so that 20-80 % of each fixed cloud overlaps the movable
    one, plus the bunny."""
    sizes = [40_000, 25_000, 60_000, 8_000, 30_000, 12_345, 50_000, 20_000]
    pairs = []
    for i, (Xf, Xm) in enumerate(_surface_pairs(len(sizes), sizes, seed0=60_000)):
        frac = 0.2 + 0.6 * i / (len(sizes) - 1)
        pairs.append((np.ascontiguousarray(Xf), np.ascontiguousarray(Xm[Xm[:, 0] > 30.0 * (1.0 - frac)])))
    pairs.append(load_pair("bunny"))
    return pairs


def _priors(n):
    rng = np.random.default_rng(7)
    return np.column_stack((rng.uniform(-0.5, 0.5, (n, 3)), rng.uniform(-0.05, 0.05, (n, 3))))


@pytest.mark.parametrize("priors", [False, True])
@pytest.mark.parametrize("mod", [-1.0, 1.0])
@pytest.mark.parametrize("angle", [None, 20.0])
def test_batch_equals_register(gpu, angle, mod, priors):
    pairs = _ragged_pairs()
    rows = _priors(len(pairs)) if priors else None
    rad = None if rows is None else np.array([_observed_in_radians(r) for r in rows])
    ang = -1.0 if angle is None else float(np.deg2rad(angle))
    with _capi.Engine() as e:
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        params = e.run_params(0.3, 1.0, 100, lsq)
        res = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=mod, observed=rad,
                               mov_neighbors=10, max_angle_rad=ang)
        assert e.timings()["mov_normals_ms"] > 0
        plain = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=mod, observed=rad)
        fewer = 0
        for i, (Xf, Xm) in enumerate(pairs):
            kw = {} if rows is None else {"rbp_observed_values": rows[i]}
            r = sb.register(Xf, Xm, engine=e, want_normals=False, max_overlap_distance=mod if mod > 0 else np.inf,
                            mov_neighbors=10, max_angle_between_normals=angle, **kw)
            what = f"angle {angle} mod {mod} priors {priors} pair {i}"
            b = res[i]
            assert b.status == 0, what
            assert b.iterations == r.iterations and bool(b.converged) == r.converged, what
            assert b.n_kept == r.records[-1]["n_kept"], what
            assert int(res.n_selected[i]) == len(r.idx_selected), what
            np.testing.assert_allclose(np.array(b.H).reshape(4, 4), r.H, rtol=0, atol=1e-12, err_msg=what)
            fewer += b.n_kept < plain[i].n_kept
        assert fewer > 0  # the movable-side tests did reject something


def test_batch_pair_with_too_few_movable_points(gpu):
    pairs = _ragged_pairs()[:3]
    pairs[1] = (pairs[1][0], pairs[1][1][:9])
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
        with pytest.raises(_capi.SicpError) as ei:
            e.register_batch(pairs, 1000, 10, params, mov_neighbors=10)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG


def test_front_end_takes_the_batched_engine(gpu, monkeypatch):
    from simpleicp_b200 import batch

    pairs = _ragged_pairs()[:6]
    calls = []
    orig = batch._run_batched

    def spy(*a, **kw):
        calls.append(1)
        return orig(*a, **kw)

    monkeypatch.setattr(batch, "_run_batched", spy)
    table = sb.simpleicp_batch(pairs, mov_neighbors=10, max_angle_between_normals=20.0)
    assert calls == [1]
    pool = sb.simpleicp_batch(pairs, mov_neighbors=10, max_angle_between_normals=20.0, engine="pool")
    assert calls == [1]
    np.testing.assert_allclose(table[:, :16], pool[:, :16], rtol=0, atol=1e-12)
    assert np.array_equal(table[:, 16:18], pool[:, 16:18])
