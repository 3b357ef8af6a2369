"""The batched engine with the overlap filter and one prior per pair (sicp_register_batch with
max_overlap_distance and `observed`), against sicp_register pair by pair."""
import numpy as np
import pytest

from conftest import load_pair
from oracle import simpleicp_oracle as O
from test_gpu_nn_exact import ORIGINS, U, exact_knn, perm_H, rigid_apply, to_xyz
from test_gpu_parity import _surface_pairs

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200.linearized import VARIANT_LINEARIZED
from simpleicp_b200.simpleicp import _observed_in_radians

pytestmark = pytest.mark.gpu


def _cropped_pairs():
    """Ragged surface pairs (extent 30 m) cropped so that 20-80 % of each fixed cloud overlaps
    the movable one, plus the bunny."""
    sizes = [40_000, 25_000, 60_000, 8_000, 30_000, 12_345, 50_000, 20_000]
    pairs = []
    for i, (Xf, Xm) in enumerate(_surface_pairs(len(sizes), sizes, seed0=20_000)):
        frac = 0.2 + 0.6 * i / (len(sizes) - 1)
        pairs.append((np.ascontiguousarray(Xf), np.ascontiguousarray(Xm[Xm[:, 0] > 30.0 * (1.0 - frac)])))
    pairs.append(load_pair("bunny"))
    return pairs


def _same_bits(a, b):
    """Every field of two PairResults bit for bit (NaN sigmas of fixed parameters included)."""
    return all(np.array(getattr(a, f)).tobytes() == np.array(getattr(b, f)).tobytes() for f, _ in _capi.PairResult._fields_)


def _lsq(e, w=np.zeros(6), dw=1.0):
    return e.lsq_params(np.zeros(6), np.zeros(6), w, dw)


def _same_as_register(b, nsel, r, what):
    assert b.status == 0, f"{what}: status {b.status}"
    assert b.iterations == r.iterations and bool(b.converged) == r.converged, what
    assert b.n_kept == r.records[-1]["n_kept"], what
    assert nsel == len(r.idx_selected), what
    np.testing.assert_allclose(np.array(b.H).reshape(4, 4), r.H, rtol=0, atol=1e-12, err_msg=what)
    np.testing.assert_allclose(np.array(b.x), r.rbp.get_parameter_attributes_as_list("estimated_value"),
                               rtol=0, atol=1e-12, err_msg=what)
    np.testing.assert_allclose(np.array(b.sigma), r.rbp.get_parameter_attributes_as_list("estimated_uncertainty"),
                               rtol=1e-9, err_msg=what)
    np.testing.assert_allclose([b.mean_res, b.std_res], [r.records[-1]["mean_res"], r.records[-1]["std_res"]],
                               rtol=1e-9, atol=1e-15, err_msg=what)


@pytest.mark.parametrize("variant", [0, VARIANT_LINEARIZED])
def test_filtered_batch_equals_register_per_pair(gpu, variant):
    pairs = _cropped_pairs()
    with _capi.Engine() as e:
        e.set_option("variant", variant)
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        for mod in (0.5, 1.0):
            res = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=mod)
            for i, (Xf, Xm) in enumerate(pairs):
                r = sb.register(Xf, Xm, engine=e, want_normals=False, max_overlap_distance=mod)
                _same_as_register(res[i], int(res.n_selected[i]), r, f"variant {variant} mod {mod} pair {i}")


def _boundary_pair(origin, s):
    """test_gpu_nn_exact.test_overlap_filter_boundary's geometry: neighbours at exactly r U, at
    the largest d^2 below it, and far queries; the movable cloud sits at X_fix's place moved by -s
    lattice units, so the prior translation s U brings it back."""
    rng = np.random.default_rng(11)
    r = 300
    mk = np.stack(np.meshgrid(*[np.arange(0, 20 * 1024, 1024)] * 2, [0], indexing="ij"), -1).reshape(-1, 3)
    offs = []
    for target in range(r * r - 40, r * r + 41):
        a = rng.integers(0, r + 1)
        b2 = target - a * a
        if b2 < 0:
            continue
        b = int(np.sqrt(b2))
        cc = int(np.sqrt(b2 - b * b))
        if cc * cc == b2 - b * b:
            offs.append([a, b, cc])
    offs += [[r, 0, 0], [0, r, 0], [0, 0, r], [0, 0, r - 1], [r - 1, 1, 0]]
    inside = max(a * a + b * b + c * c for a in range(r) for b in range(40) for c in range(40)
                 if a * a + b * b + c * c < r * r)
    offs += [[a, b, c] for a in range(r - 2, r) for b in range(40) for c in range(40)
             if a * a + b * b + c * c == inside][:4]
    offs = np.array(offs)
    base = mk[rng.integers(0, len(mk), len(offs))]
    far = np.array([[-40 * 1024, 5000, 0], [5000, 30 * 1024, 9000], [3000, 3000, 60 * 1024]])
    qk = np.concatenate((base + offs * rng.choice([-1, 1], offs.shape), far))
    _, d2 = exact_knn(mk, qk, 1)
    assert (d2[:, 0] == r * r).any() and (d2[:, 0] == inside).any() and (d2[:, 0] > r * r).any()
    Xf, Xm = to_xyz(qk + s, origin), to_xyz(mk, origin)
    H0 = perm_H(np.eye(3), s, origin)
    oracle = O.select_in_range(Xf, np.arange(len(qk)), rigid_apply(H0, Xm), r * U)
    return Xf, Xm, r * U, int((d2[:, 0] < r * r).sum()), oracle


def test_filter_counts_are_exact(gpu):
    """n_selected of boundary pairs with their own dyadic prior, beside ordinary pairs: the
    integer reference and the oracle's select_in_range, whatever the loop does with the pair."""
    cases = [(o, s) for o in ORIGINS.values() for s in ([5, -3, 2], [-7, 1, 4])]
    boundary = [_boundary_pair(o, np.array(s)) for o, s in cases]
    max_range = boundary[0][2]
    others = _surface_pairs(2, 4000, seed0=30_000)
    pairs = [(b[0], b[1]) for b in boundary] + others
    rows = np.zeros((len(pairs), 6))
    for i, (_, s) in enumerate(cases):
        rows[i, 3:] = np.array(s) * U
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 20, _lsq(e))
        res = e.register_batch(pairs, 4096, 10, params, max_overlap_distance=max_range, observed=rows)
    for i, (Xf, Xm, _, n_ref, oracle) in enumerate(boundary):
        assert n_ref == len(oracle) < 4096
        assert res.n_selected[i] == n_ref, f"pair {i}: {res.n_selected[i]} vs {n_ref}"


def _far_batch():
    pairs = _cropped_pairs()[:5]
    far = (pairs[2][0], pairs[2][1] + 1e4)
    return pairs, pairs[:2] + [far] + pairs[2:]


def test_pair_without_overlap_fails_alone(gpu):
    pairs, with_far = _far_batch()
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        a = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=1.0)
        b = e.register_batch(with_far, 1000, 10, params, max_overlap_distance=1.0)
    assert b[2].status == _capi.SICP_ERR_NO_OVERLAP and b.n_selected[2] == 0
    for i, j in enumerate([0, 1, 3, 4, 5]):
        assert a[i].status == 0
        assert _same_bits(a[i], b[j]), f"pair {i}"
        assert a.n_selected[i] == b.n_selected[j]
    table = sb.simpleicp_batch(with_far, max_overlap_distance=1.0, on_error="nan")
    pool = sb.simpleicp_batch(with_far, max_overlap_distance=1.0, on_error="nan", engine="pool")
    assert table[2, 16] == pool[2, 16] == -_capi.SICP_ERR_NO_OVERLAP
    ok = [0, 1, 3, 4, 5]
    np.testing.assert_allclose(table[ok, :16], pool[ok, :16], rtol=0, atol=1e-12)
    assert np.array_equal(table[ok, 16:18], pool[ok, 16:18])


def _displaced_pairs():
    """Surface pairs moved by yaws from -60 to +120 degrees and translations of metres, which the
    identity start cannot undo; row i (degrees) undoes pair i's displacement.  The last pair is
    100 m away: no overlap at all under the identity."""
    pairs = _surface_pairs(6, [30_000, 20_000, 40_000, 25_000, 30_000, 15_000], seed0=40_000)
    yaws = [-60.0, -20.0, 15.0, 45.0, 90.0, 120.0]
    shifts = [(3.0, -2.0, 0.5), (-4.0, 1.0, -1.0), (2.5, 2.5, 0.0), (-1.5, 3.0, 0.25), (5.0, -5.0, 1.0),
              (100.0, 0.0, 0.0)]
    out, rows = [], []
    for (Xf, Xm), yaw, t in zip(pairs, yaws, shifts):
        row = np.array([0.0, 0.0, yaw, *t])
        D = O.rbp_to_H(_observed_in_radians(row))
        out.append((Xf, O.transform_by_H(Xm, np.linalg.inv(D))))
        rows.append(row)
    return out, np.array(rows)


@pytest.mark.parametrize("weights", [(0, 0, 0, 0, 0, 0), (np.inf, np.inf, 0, 5, 0, 0)])
def test_per_pair_priors(gpu, weights):
    pairs, rows = _displaced_pairs()
    rad = np.array([_observed_in_radians(r) for r in rows])
    w = np.array(weights, dtype=float)
    with _capi.Engine() as e:
        params = e.run_params(0.3, 1.0, 100, _lsq(e, w))
        res = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=1.0, observed=rad)
        for i, (Xf, Xm) in enumerate(pairs):
            r = sb.register(Xf, Xm, engine=e, want_normals=False, max_overlap_distance=1.0,
                            rbp_observed_values=rows[i], rbp_observation_weights=weights)
            _same_as_register(res[i], int(res.n_selected[i]), r, f"weights {weights} pair {i}")
            assert np.linalg.norm(r.H[:3, :3] - O.rbp_to_H(rad[i])[:3, :3]) < 0.1  # the prior was needed
        # the filter runs under each pair's prior: under the identity the last pair has no overlap
        ident = e.register_batch(pairs, 1000, 10, params, max_overlap_distance=1.0)
        assert ident[5].status == _capi.SICP_ERR_NO_OVERLAP and ident.n_selected[5] == 0


def test_no_behaviour_change_without_rows(gpu):
    """observed rows all equal to the common values give exactly the results of observed = NULL,
    with and without the filter."""
    pairs = _surface_pairs(5, [30_000, 12_000, 45_000, 30_000, 8_000], seed0=50_000)
    obs = np.array([0.001, 0, 0, 0, 0, 0.01])
    with _capi.Engine() as e:
        lsq = e.lsq_params(obs, obs, np.array([np.inf, 0, 0, 5.0, 0, 0]), None)
        params = e.run_params(0.3, 1.0, 50, lsq)
        for mod in (-1.0, 1.0):
            a = e.register_batch(pairs, 700, 10, params, max_overlap_distance=mod)
            b = e.register_batch(pairs, 700, 10, params, max_overlap_distance=mod, observed=np.tile(obs, (5, 1)))
            assert np.array_equal(a.n_selected, b.n_selected)
            for i in range(len(pairs)):
                assert a[i].status == 0
                assert _same_bits(a[i], b[i]), f"{mod} pair {i}"


def test_front_end_takes_the_batched_engine(gpu, monkeypatch):
    pairs, rows = _displaced_pairs()
    calls = []
    orig = _capi.Engine.register_batch

    def spy(self, *a, **kw):
        calls.append(len(a[0]))
        return orig(self, *a, **kw)

    monkeypatch.setattr(_capi.Engine, "register_batch", spy)
    table = sb.simpleicp_batch(pairs, max_overlap_distance=1.0, rbp_observed_values=rows, batch_size=4)
    assert calls == [4, 2]
    monkeypatch.setattr(_capi.Engine, "register_batch", orig)
    pool = sb.simpleicp_batch(pairs, max_overlap_distance=1.0, rbp_observed_values=rows, engine="pool")
    np.testing.assert_allclose(table[:, :16], pool[:, :16], rtol=0, atol=1e-12)
    assert np.array_equal(table[:, 16:18], pool[:, 16:18])
