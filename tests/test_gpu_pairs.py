"""Pairs drawn from one set of clouds (sicp_register_pairs, sb.simpleicp_edges): bit for bit
against sicp_register_batch on the expanded pairs -- results, n_selected and the batch outputs --
for scan chains, several priors of one pair, clouds in both roles, self pairs and unreferenced
NULL clouds, with and without the overlap filter and movable attributes."""
import ctypes as C

import numpy as np
import pytest

from oracle import simpleicp_oracle as O
from test_gpu_batch_overlap import _lsq, _same_as_register, _same_bits

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200.linearized import VARIANT_LINEARIZED
from simpleicp_b200.simpleicp import _observed_in_radians

pytestmark = pytest.mark.gpu


def _chain(n=8, seed=80_000):
    """n ragged scans of one surface (extent 40 m, 12 000-30 000 points), scan i sampled over
    x in [2 i, 2 i + 26) and moved by a small rigid transform, with a noisy prior per edge
    (degrees) for the edges (i, i + 1) and (i, i + 2)."""
    rng = np.random.default_rng(seed)
    scans, poses = [], []
    for i in range(n):
        S = O.surface(int(rng.integers(12_000, 30_000)), seed + 1 + i, extent=40.0)
        S = S[(S[:, 0] >= 2.0 * i) & (S[:, 0] < 2.0 * i + 26.0)]
        x = np.concatenate((rng.uniform(-1, 1, 3), rng.uniform(-0.3, 0.3, 3)))
        scans.append(np.ascontiguousarray(O.transform_by_H(S, np.linalg.inv(O.rbp_to_H(_observed_in_radians(x))))))
        poses.append(x)
    edges = np.array([(i, i + 1) for i in range(n - 1)] + [(i, i + 2) for i in range(n - 2)])
    # the relative prior of edge (a, b), as degrees / metres, plus noise
    rows = np.array([poses[b] - poses[a] + np.concatenate((rng.normal(0, 0.05, 3), rng.normal(0, 0.02, 3)))
                     for a, b in edges])
    return scans, edges, rows


_DATA = {}


def _data():
    if "chain" not in _DATA:
        _DATA["chain"] = _chain()
    return _DATA["chain"]


def _geometries():
    """(clouds, edges, rows in degrees) of every geometry: the chain; a star (one pair under 6
    priors); a cloud fixed in one edge and movable in another; a self edge; an unreferenced
    cloud passed as None (NULL)."""
    scans, edges, rows = _data()
    yaws = [-3.0, -1.0, 0.0, 0.5, 2.0, 4.0]
    star_rows = np.array([[0, 0, y, 0.1 * k, -0.05 * k, 0] for k, y in enumerate(yaws)], dtype=float)
    return {
        "chain": (scans, edges, rows),
        "star": (scans[:2], np.tile([[0, 1]], (6, 1)), star_rows),
        "both_roles": (scans[:3], np.array([[0, 1], [1, 2], [2, 0]]), np.vstack((rows[0], rows[1], -rows[7]))),
        "self": (scans[:2], np.array([[0, 0], [0, 1], [1, 1]]), np.vstack((np.zeros(6), rows[0], np.zeros(6)))),
        "null": ([scans[0], None, scans[2], None], np.array([[0, 2], [2, 0]]), np.vstack((rows[7], -rows[7]))),
    }


def _rad(rows):
    return np.array([_observed_in_radians(r) for r in rows])


def _assert_outputs_equal(oa, ob, what):
    """batch_outputs of two calls' results, pair by pair: X_t, residuals, the log's bytes, T."""
    for i, (x, y) in enumerate(zip(oa, ob)):
        assert (x is None) == (y is None), f"{what} pair {i}"
        if x is None:
            continue
        assert np.array_equal(x[0], y[0]), f"{what} pair {i}: X_t"
        assert np.array_equal(x[1], y[1]), f"{what} pair {i}: residuals"
        assert b"".join(bytes(r) for r in x[2]) == b"".join(bytes(r) for r in y[2]), f"{what} pair {i}: log"
        assert np.array_equal(x[3], y[3]), f"{what} pair {i}: T"


def _compare(e, clouds, edges, rows, opts, what):
    params = e.run_params(0.3, 1.0, 60, _lsq(e))
    a = e.register_pairs(clouds, edges, 1000, 10, params, observed=_rad(rows), **opts)
    oa = e.batch_outputs(a)
    b = e.register_batch([(clouds[f], clouds[m]) for f, m in edges], 1000, 10, params, observed=_rad(rows), **opts)
    ob = e.batch_outputs(b)
    assert np.array_equal(a.n_selected, b.n_selected), f"{what}: {a.n_selected} vs {b.n_selected}"
    assert np.array_equal(a.n_mov, b.n_mov)
    for i in range(len(edges)):
        assert _same_bits(a[i], b[i]), f"{what} pair {i}"
    _assert_outputs_equal(oa, ob, what)
    return a


OPTS = {"plain": {}, "overlap": dict(max_overlap_distance=1.0),
        "mov": dict(mov_neighbors=10, max_angle_rad=np.deg2rad(20.0)),
        "both": dict(max_overlap_distance=1.0, mov_neighbors=10, max_angle_rad=np.deg2rad(20.0))}


@pytest.mark.parametrize("opts", list(OPTS))
@pytest.mark.parametrize("variant", [0, VARIANT_LINEARIZED])
def test_bits_equal_the_batch_on_the_expanded_pairs(gpu, variant, opts):
    with _capi.Engine() as e:
        e.set_option("variant", variant)
        for name, (clouds, edges, rows) in _geometries().items():
            if variant != 0 and "mov_neighbors" in OPTS[opts]:
                # the linearised variants have no movable-side attributes, here as in the batch
                params = e.run_params(0.3, 1.0, 60, _lsq(e))
                with pytest.raises(_capi.SicpError) as err:
                    e.register_pairs(clouds, edges, 1000, 10, params, observed=_rad(rows), **OPTS[opts])
                assert err.value.code == _capi.SICP_ERR_BAD_ARG
                continue
            a = _compare(e, clouds, edges, rows, OPTS[opts], f"variant {variant} {opts} {name}")
            if name == "chain":
                assert sum(r.status == 0 for r in a) >= len(edges) - 1, [r.status for r in a]


def test_pair_without_overlap_fails_alone(gpu):
    scans, edges, rows = _data()
    far = scans[3] + np.array([1e4, 0.0, 0.0])
    clouds = scans + [far]
    bad = np.vstack((edges, [[2, len(scans)], [len(scans), 4]]))
    bad_rows = np.vstack((rows, np.zeros((2, 6))))
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 60, _lsq(e))
        a = e.register_pairs(scans, edges, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        b = e.register_pairs(clouds, bad, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(bad_rows))
    assert b[len(edges)].status == b[len(edges) + 1].status == _capi.SICP_ERR_NO_OVERLAP
    assert b.n_selected[len(edges)] == b.n_selected[len(edges) + 1] == 0
    for i in range(len(edges)):
        assert _same_bits(a[i], b[i]), f"pair {i}"
        assert a.n_selected[i] == b.n_selected[i]


def test_edges_agree_with_register(gpu):
    scans, edges, rows = _data()
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        res = e.register_pairs(scans, edges, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        for i in (0, 3, len(edges) - 1):
            f, m = edges[i]
            r = sb.register(scans[f], scans[m], engine=e, want_normals=False, max_overlap_distance=1.0,
                            rbp_observed_values=rows[i])
            _same_as_register(res[i], int(res.n_selected[i]), r, f"edge {i}")


def test_memory_kinds_give_the_same_bits(gpu):
    import torch

    scans, edges, rows = _data()
    mixed = []
    for j, S in enumerate(scans):
        if j % 3 == 0:
            mixed.append(torch.from_numpy(S).cuda())
        elif j % 3 == 1:
            mixed.append(torch.from_numpy(S).pin_memory().numpy())
        else:
            mixed.append(S.copy())
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 60, _lsq(e))
        a = e.register_pairs(scans, edges, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        oa = e.batch_outputs(a)
        b = e.register_pairs(mixed, edges, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        ob = e.batch_outputs(b)
    for i in range(len(edges)):
        assert _same_bits(a[i], b[i]), f"pair {i}"
    _assert_outputs_equal(oa, ob, "memory kinds")


def test_call_order(gpu):
    scans, edges, rows = _data()
    X = np.concatenate(scans[:4])
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 60, _lsq(e))
        e.set_map(X)
        m0 = e.register_to_map(scans[4:], 1000, 10, params, max_overlap_distance=1.0)
        om0 = e.batch_outputs(m0)
        a = e.register_pairs(scans, edges, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        oa = e.batch_outputs(a)
        assert all(o is not None for o in oa[:3])
        # the map is untouched: the same register_to_map bits and outputs as before
        m1 = e.register_to_map(scans[4:], 1000, 10, params, max_overlap_distance=1.0)
        for i in range(len(m0)):
            assert _same_bits(m0[i], m1[i]), f"scan {i}"
        _assert_outputs_equal(om0, e.batch_outputs(m1), "map after pairs")
        with pytest.raises(_capi.SicpError):  # the pairs' outputs are gone: n_pairs differs now
            e.batch_outputs(a)
        # a batched call that fails on its arguments clears them too
        e.register_pairs(scans, edges, 1000, 10, params, max_overlap_distance=1.0, observed=_rad(rows))
        with pytest.raises(_capi.SicpError):
            e.register_pairs(scans, edges, 4097, 10, params)
        with pytest.raises(_capi.SicpError) as err:
            e.batch_outputs(a)
        assert err.value.code == _capi.SICP_ERR_STATE


def _raw(e, xyz, n, fix, mov, corr=1000, neighbors=10):
    lib = _capi.load_library()
    k = len(xyz)
    params = e.run_params(0.3, 1.0, 20, _lsq(e))
    rp = e._register_params(corr, neighbors, params, -1.0, 0, -1.0)
    out = (_capi.PairResult * len(fix))()
    return lib.sicp_register_pairs(e._h, k, (C.c_void_p * k)(*xyz), (C.c_int64 * k)(*n), len(fix),
                                   (C.c_int32 * len(fix))(*fix), (C.c_int32 * len(fix))(*mov), C.byref(rp), None,
                                   out, None)


def test_bad_arguments(gpu):
    scans, _, _ = _data()
    small = np.ascontiguousarray(scans[0][:5])
    ptrs = [scans[0].ctypes.data, scans[1].ctypes.data, None, small.ctypes.data]
    n = [len(scans[0]), len(scans[1]), 100, len(small)]
    with _capi.Engine() as e:
        assert _raw(e, ptrs, n, [0, 1], [1, 0]) == _capi.SICP_OK
        assert _raw(e, ptrs, n, [0, 4], [1, 0]) == _capi.SICP_ERR_BAD_ARG        # id out of range
        assert _raw(e, ptrs, n, [0, -1], [1, 0]) == _capi.SICP_ERR_BAD_ARG
        assert _raw(e, ptrs, n, [0, 2], [1, 0]) == _capi.SICP_ERR_BAD_ARG        # a referenced NULL cloud
        assert _raw(e, ptrs, n, [0, 3], [1, 0]) == _capi.SICP_ERR_BAD_ARG        # fixed cloud below neighbors
        assert _raw(e, ptrs, n, [0, 1], [3, 0]) == _capi.SICP_OK                 # as a movable cloud it is fine
        assert _raw(e, ptrs, n, [0, 1], [1, 0], corr=4097) == _capi.SICP_ERR_BAD_ARG
        assert _raw(e, ptrs[:0], n[:0], [0], [0]) == _capi.SICP_ERR_BAD_ARG     # n_clouds 0


def test_simpleicp_edges_equals_simpleicp_batch(gpu):
    scans, edges, rows = _data()
    kw = dict(max_overlap_distance=1.0, rbp_observed_values=rows, max_iterations=60)
    pairs = [(scans[f], scans[m]) for f, m in edges]
    for bs in (64, 3):
        t_e, r_e = sb.simpleicp_edges(scans, edges, batch_size=bs, full_output=True, on_error="nan", **kw)
        t_b, r_b = sb.simpleicp_batch(pairs, batch_size=bs, full_output=True, on_error="nan", **kw)
        assert np.array_equal(t_e, t_b, equal_nan=True), bs
        for i, (x, y) in enumerate(zip(r_e, r_b)):
            assert (x is None) == (y is None), (bs, i)
            if x is None:
                continue
            for f in ("H", "X_mov_transformed", "residuals"):
                assert np.array_equal(getattr(x, f), getattr(y, f)), (bs, i, f)
            assert repr(x.records) == repr(y.records) and x.iterations == y.iterations, (bs, i)
            assert np.array_equal(x.rbp.get_parameter_attributes_as_list("estimated_uncertainty"),
                                  y.rbp.get_parameter_attributes_as_list("estimated_uncertainty"), equal_nan=True)
    # movable attributes through the front end, chunks straddling the clouds
    kw = dict(mov_neighbors=10, max_angle_between_normals=20.0, max_iterations=30)
    assert np.array_equal(sb.simpleicp_edges(scans, edges, batch_size=3, on_error="nan", **kw),
                          sb.simpleicp_batch(pairs, batch_size=3, on_error="nan", **kw), equal_nan=True)
