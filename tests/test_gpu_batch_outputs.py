"""sicp_get_batch_outputs and the full_output front ends: transformed clouds, final residuals,
iteration logs and applied transforms of sicp_register_batch / sicp_register_to_map, against
sicp_register pair by pair, bit for bit within the batch, through every memory kind, and across
the call order that makes them valid or stale.  Every movable cloud has an odd point count, so
pair offsets alternate between 16-byte aligned and not."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_gpu_batch_overlap import _cropped_pairs, _lsq
from test_gpu_map import _map_and_scans, _rad
from test_gpu_memory_kinds import Buf, _same

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200.linearized import VARIANT_LINEARIZED, VARIANT_LINEARIZED_CPP

pytestmark = pytest.mark.gpu

_DATA = {}


def _odd(X):
    return np.ascontiguousarray(X if len(X) % 2 else X[:-1])


def _pairs():
    if "pairs" not in _DATA:
        _DATA["pairs"] = [(Xf, _odd(Xm)) for Xf, Xm in _cropped_pairs()]
    return _DATA["pairs"]


def _map():
    if "map" not in _DATA:
        X, scans, rows = _map_and_scans(n_map=60_000, extent=60.0, seed=73_000)
        _DATA["map"] = X, [_odd(S) for S in scans], rows
    return _DATA["map"]


def _two_pass(r, sample):
    m = r.sum() / r.size
    return m, np.sqrt(((r - m) ** 2).sum() / (r.size - (1 if sample else 0)))


def _log_rows(log):
    return np.array([[rec.n_kept, rec.median, rec.mad, rec.mean_dist, rec.std_dist, *rec.x, rec.mean_res, rec.std_res]
                     for rec in log])


def _records_match(log, records, what):
    """Iteration count, per-iteration n_kept and x, and the record statistics (to 1e-9 m where they
    are near zero: the transforms differ from register's by up to 1e-12)."""
    assert len(log) == len(records), what
    for j, (a, b) in enumerate(zip(log, records)):
        assert a.n_kept == b["n_kept"], f"{what}: iteration {j}"
        np.testing.assert_allclose(np.array(a.x), b["x"], rtol=0, atol=1e-12, err_msg=f"{what}: x, iteration {j}")
        np.testing.assert_allclose([a.median, a.mad, a.mean_dist, a.std_dist, a.mean_res, a.std_res],
                                   [b[k] for k in ("median", "mad", "mean_dist", "std_dist", "mean_res", "std_res")],
                                   rtol=1e-9, atol=1e-9, err_msg=f"{what}: statistics, iteration {j}")


CONFIGS = [(0, -1.0, {}), (0, 1.0, {}), (VARIANT_LINEARIZED, -1.0, {}), (VARIANT_LINEARIZED, 1.0, {}),
           (VARIANT_LINEARIZED_CPP, -1.0, {}), (VARIANT_LINEARIZED_CPP, 1.0, {}),
           (0, 1.0, dict(mov_neighbors=10, max_angle_rad=np.deg2rad(20.0)))]


@pytest.mark.parametrize("variant,mod,mov", CONFIGS)
def test_outputs_equal_register_per_pair(gpu, variant, mod, mov):
    pairs = _pairs()
    with _capi.Engine() as e, _capi.Engine() as t:
        e.set_option("variant", variant)
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        res = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=mod, **mov)
        outs = e.batch_outputs(res)
        extra = {} if not mov else dict(mov_neighbors=mov["mov_neighbors"],
                                         max_angle_between_normals=float(np.rad2deg(mov["max_angle_rad"])))
        for i, (Xf, Xm) in enumerate(pairs):
            what = f"variant {variant} mod {mod} {mov} pair {i}"
            b = res[i]
            assert b.status == 0, what
            X_t, resid, log, T = outs[i]
            r = sb.register(Xf, Xm, engine=e, want_normals=False, max_overlap_distance=mod if mod > 0 else np.inf,
                            **extra)
            # against register
            assert resid.shape == r.residuals.shape, what
            _records_match(log, r.records, what)
            np.testing.assert_allclose(resid, r.residuals, rtol=0, atol=1e-9, err_msg=what)
            np.testing.assert_allclose(X_t, r.X_mov_transformed, rtol=0, atol=1e-9, err_msg=what)
            # within the batch, bit for bit
            t.set_clouds(Xf, Xm)
            _same(X_t, t.transform(T), f"{what}: sicp_transform under T")
            if variant == VARIANT_LINEARIZED_CPP:
                assert not np.array_equal(T, np.array(b.H).reshape(4, 4)), what
            else:
                _same(T, np.array(b.H).reshape(4, 4), f"{what}: T vs H")
            m, s = _two_pass(resid, variant != 0)
            np.testing.assert_allclose([m, s], [b.mean_res, b.std_res], rtol=1e-12, atol=1e-18, err_msg=what)
            assert log[-1].n_kept == b.n_kept == resid.size, what
            assert (log[-1].mean_res, log[-1].std_res) == (b.mean_res, b.std_res), what


def _all_outputs(e, res):
    """Every output of the last call as bytes (pageable NumPy), for bit comparisons."""
    return [None if o is None else (o[0].tobytes(), o[1].tobytes(), _log_rows(o[2]).tobytes(), o[3].tobytes())
            for o in e.batch_outputs(res)]


@pytest.mark.parametrize("opts", [dict(max_overlap_distance=1.0), dict(),
                                  dict(max_overlap_distance=1.0, mov_neighbors=10, max_angle_rad=np.deg2rad(20.0))])
def test_map_outputs_equal_the_batch_with_the_map_repeated(gpu, opts):
    X, scans, rows = _map()
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        e.set_map(X)
        a = e.register_to_map(scans, 1000, 10, params, observed=_rad(rows), **opts)
        oa = _all_outputs(e, a)
        b = e.register_batch([(X, S) for S in scans], 1000, 10, params, observed=_rad(rows), **opts)
        ob = _all_outputs(e, b)
    assert [r.status for r in a] == [r.status for r in b]
    assert any(o is not None for o in oa)
    for i, (x, y) in enumerate(zip(oa, ob)):
        assert x == y, f"{opts} scan {i}"


# ------------------------------------------------------------------------- memory kinds, state
def _raw(e, n, xyz=None, resid=None, log=None, T=None):
    """sicp_get_batch_outputs with raw addresses (None: NULL array or NULL entry)."""
    arr = (lambda a: None if a is None else (C.c_void_p * n)(*a))
    return e._lib.sicp_get_batch_outputs(e._h, n, arr(xyz), arr(resid), log, T)


def _other_device_buf(n, device):
    return torch.full((n,), np.nan, dtype=torch.float64, device=f"cuda:{device}")


def test_every_memory_kind_gives_the_same_bits(gpu):
    pairs = _pairs()[:6]
    pairs = pairs[:2] + [(pairs[2][0], pairs[2][1] + 1e4)] + pairs[3:]  # pair 2: no overlap
    n = len(pairs)
    skip = 4  # a NULL entry in every array
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 60, _lsq(e))
        res = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=1.0)
        assert res[2].status == _capi.SICP_ERR_NO_OVERLAP
        assert all(res[i].status == 0 for i in range(n) if i != 2)
        want = e.batch_outputs(res)
        kinds = ["P", "P+", "H", "D", "D+"] + (["other"] if torch.cuda.device_count() > 1 else [])
        for kind in kinds:
            def buf(count):
                if kind == "other":
                    return _other_device_buf(count, 1)
                return Buf(kind, count, np.float64)

            xs = [buf(3 * int(res.n_mov[i])) for i in range(n)]
            rs = [buf(max(int(res[i].n_kept), 1)) for i in range(n)]
            addr = (lambda b: b.data_ptr() if isinstance(b, torch.Tensor) else b.addr)
            log = (_capi.IterRecord * (n * 60))()
            for k in range(n * 60):
                log[k].n_kept = -7  # sentinel
            T = (C.c_double * (16 * n))(*([np.nan] * 16 * n))
            rc = _raw(e, n, [None if i == skip else addr(b) for i, b in enumerate(xs)],
                      [None if i == skip else addr(b) for i, b in enumerate(rs)], log, T)
            assert rc == 0, e._lib.sicp_last_error(e._h)
            get = (lambda b: b.cpu().numpy() if isinstance(b, torch.Tensor) else b.get())
            for i in range(n):
                what = f"{kind} pair {i}"
                X, R = get(xs[i]), get(rs[i])
                if i in (2, skip):
                    assert np.isnan(X).all() and np.isnan(R).all(), f"{what}: written"
                    if i == 2:
                        assert np.isnan(np.array(T[16 * i:16 * i + 16])).all(), what
                        assert all(log[i * 60 + j].n_kept == -7 for j in range(60)), what
                    continue
                _same(X.reshape(-1, 3), want[i][0], f"{what}: cloud")
                _same(R, want[i][1], f"{what}: residuals")
                _same(np.array(T[16 * i:16 * i + 16]).reshape(4, 4), want[i][3], f"{what}: T")
                _same(_log_rows([log[i * 60 + j] for j in range(res[i].iterations)]), _log_rows(want[i][2]),
                      f"{what}: log")
                assert not any(log[i * 60 + j].n_kept for j in range(res[i].iterations, 60)), what


def test_validity_follows_the_call_order(gpu):
    pairs = _pairs()
    first, second = pairs[:4], pairs[3:8]
    with _capi.Engine() as e, _capi.Engine() as ref:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        assert _raw(e, 1) == _capi.SICP_ERR_STATE  # fresh context
        e.register_batch(first, 1000, 10, params)
        res = e.register_batch(second, 1000, 10, params, max_overlap_distance=1.0)
        assert _raw(e, len(second) + 1) == _capi.SICP_ERR_BAD_ARG
        assert _raw(e, len(second) - 1) == _capi.SICP_ERR_BAD_ARG
        a, b = _all_outputs(e, res), _all_outputs(e, res)  # twice: the same bits
        assert a == b
        # the outputs are the second call's: a context that only ran it gives the same
        assert _all_outputs(ref, ref.register_batch(second, 1000, 10, params, max_overlap_distance=1.0)) == a
        # a refused call clears them
        with pytest.raises(_capi.SicpError) as ex:
            e.register_batch(second, 5000, 10, params)
        assert ex.value.code == _capi.SICP_ERR_BAD_ARG
        assert _raw(e, len(second)) == _capi.SICP_ERR_STATE
        # so does sicp_set_map
        res = e.register_batch(second, 1000, 10, params, max_overlap_distance=1.0)
        assert _all_outputs(e, res) == a
        e.set_map(pairs[0][0])
        assert _raw(e, len(second)) == _capi.SICP_ERR_STATE


# ------------------------------------------------------------------------- front ends
def test_simpleicp_batch_full_output(gpu):
    pairs = _pairs()[:6]
    pairs = pairs[:2] + [(pairs[2][0], pairs[2][1] + 1e4)] + pairs[3:]  # pair 2: no overlap
    kw = dict(max_overlap_distance=1.0, on_error="nan")
    table = sb.simpleicp_batch(pairs, **kw)
    t2, results = sb.simpleicp_batch(pairs, full_output=True, **kw)
    assert np.array_equal(table, t2, equal_nan=True)
    assert results[2] is None and table[2, 16] == -_capi.SICP_ERR_NO_OVERLAP
    for i, (Xf, Xm) in enumerate(pairs):
        if i == 2:
            continue
        what = f"pair {i}"
        got = results[i]
        r = sb.register(Xf, Xm, want_normals=False, max_overlap_distance=1.0)
        np.testing.assert_allclose(got.H, r.H, rtol=0, atol=1e-12, err_msg=what)
        _same(got.H.reshape(16), table[i, :16], what)
        assert got.iterations == r.iterations and got.converged == r.converged, what
        assert got.residuals.shape == r.residuals.shape, what
        np.testing.assert_allclose(got.residuals, r.residuals, rtol=0, atol=1e-9, err_msg=what)
        np.testing.assert_allclose(got.X_mov_transformed, r.X_mov_transformed, rtol=0, atol=1e-9, err_msg=what)
        for attr, rtol, atol in (("estimated_value", 0, 1e-12), ("estimated_uncertainty", 1e-9, 0),
                                 ("initial_value", 0, 1e-12), ("observed_value", 0, 0),
                                 ("observation_weight", 0, 0)):
            np.testing.assert_allclose(got.rbp.get_parameter_attributes_as_list(attr),
                                       r.rbp.get_parameter_attributes_as_list(attr), rtol=rtol, atol=atol,
                                       err_msg=f"{what}: {attr}")
        assert len(got.records) == len(r.records), what
        for j, (a, b) in enumerate(zip(got.records, r.records)):
            assert a["n_kept"] == b["n_kept"], what
            np.testing.assert_allclose(a["x"], b["x"], rtol=0, atol=1e-12, err_msg=f"{what}: iteration {j}")
            np.testing.assert_allclose([a[k] for k in ("median", "mad", "mean_res", "std_res")],
                                       [b[k] for k in ("median", "mad", "mean_res", "std_res")],
                                       rtol=1e-9, atol=1e-9, err_msg=f"{what}: iteration {j}")
        assert got.idx_selected is None and got.normals is None and got.timings is None, what
    with pytest.raises(sb.BatchError) as ex:
        sb.simpleicp_batch(pairs, max_overlap_distance=1.0, full_output=True)
    assert ex.value.failed.tolist() == [2] and ex.value.results[2] is None
    assert ex.value.results[0] is not None
    # the per-pair engines give register's own objects
    _, pool = sb.simpleicp_batch(pairs, full_output=True, engine="pool", **kw)
    assert pool[2] is None and pool[0].normals is None and pool[0].timings is not None


def _result_bytes(r):
    return (r.H.tobytes(), np.asarray(r.X_mov_transformed).tobytes(), r.residuals.tobytes(),
            repr([sorted((k, np.asarray(v).tobytes()) for k, v in rec.items()) for rec in r.records]),
            np.array(r.rbp.get_parameter_attributes_as_list("estimated_uncertainty")).tobytes(),
            r.iterations, r.converged)


def test_map_full_output_does_not_depend_on_the_call_split(gpu):
    X, scans, rows = _map()
    assert len(scans) == 7
    kw = dict(max_overlap_distance=1.0, rbp_observed_values=rows, on_error="nan", full_output=True)
    with sb.Map(X) as m:
        ta, ra = m.register(scans, batch_size=2, **kw)
        tb, rb = m.register(scans, batch_size=64, **kw)
        plain = m.register(scans, max_overlap_distance=1.0, rbp_observed_values=rows, on_error="nan")
    assert np.array_equal(ta, tb, equal_nan=True) and np.array_equal(ta, plain, equal_nan=True)
    assert ra[-1] is None and rb[-1] is None
    for i in range(len(scans) - 1):
        assert _result_bytes(ra[i]) == _result_bytes(rb[i]), f"scan {i}"
