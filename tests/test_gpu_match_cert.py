"""The certificate of the warm-started one-pair match (nn.cu: MatchCert, DESIGN §3.2).

A search that finishes in the warm sphere scan leaves a radius rho around the query it searched,
inside which its neighbour provably stays the strict nearest record; the next match answers a
query from that certificate, without a search, while the moved query stays inside the ball.
The answer must be exactly the search's: these tests compare with the exact integer reference
of test_gpu_nn_exact (dyadic coordinates, signed-permutation transforms) and with
warm_start = 0, which never reads a certificate.
"""
from __future__ import annotations

import numpy as np
import pytest

from simpleicp_b200 import _capi
from test_gpu_nn_exact import (DEFAULTS, ORIGINS, _same, _utm_c3, cases, check_match, exact_knn,
                               rigid_apply, set_paths, to_xyz)

WALK = 12   # one-unit steps per walk


def _engine(name, where, occ=3.0):
    c = cases()[name]
    origin = ORIGINS[where]
    e = _capi.Engine()
    e.set_option("grid_target_occupancy", occ)
    _, pk = c.H(origin)
    e.set_clouds(to_xyz(pk, origin), to_xyz(c.mk, origin))
    e.set_selected(None)
    K = len(c.qk)
    z = np.zeros(K, dtype=np.float32)
    e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
    set_paths(e, {})
    return e


def _walk(step):
    """Shifts 0, s, 2 s, ... with s one unit along a mix of axes: the moved queries cross cell
    faces and equal-distance faces one unit at a time, and the moves add up across calls."""
    return [tuple(int(v) for v in np.asarray(step) * t) for t in range(WALK)]


@pytest.mark.gpu
@pytest.mark.parametrize("where", list(ORIGINS))
@pytest.mark.parametrize("name,step", [("sheet", (1, 0, 0)), ("sheet", (1, -1, 1)), ("ties", (0, 1, 0)),
                                       ("ties", (1, 1, -1))])
def test_walk_is_exact_and_certifies(gpu, name, step, where):
    """After every one-unit step the indices and distances equal the exact reference, and from
    the second warm match on some queries are answered from their certificate."""
    c = cases()[name]
    origin = ORIGINS[where]
    with _engine(name, where) as e:
        counts = []
        for t, shift in enumerate(_walk(step)):
            check_match(e, c, origin, shift, f"{name}@{where} step {t} shift {shift}")
            counts.append(e.match_counts())
        assert counts[0] == 0 and counts[1] == 0, counts     # no certificate yet: cold, then warm scan
        if name == "sheet":
            assert all(n > 0 for n in counts[2:]), counts
        else:
            # on the lattice of ties a step can put every query within one unit of an
            # equal-distance face, farther than any certificate reaches
            assert sum(counts[2:]) > 0, counts
        assert max(counts) < len(c.qk), counts


def _scattered():
    """A sparse volumetric cloud: ~3 points per cell, so a query's nearest competitor often lies
    in a neighbouring cell that the skinned sphere scan never visits, nearer than the second
    point of the cells it does visit.  Only the skip limit of L bounds such a competitor.  Queries
    start a few units from a cloud point, so their first certificates are tight."""
    rng = np.random.default_rng(271828)
    mk = rng.integers(0, 2 ** 13, size=(20_000, 3))
    src = rng.choice(len(mk), 3000, replace=False)
    qk = mk[src] + rng.integers(-6, 7, size=(3000, 3))
    from test_gpu_nn_exact import Case

    return Case("scattered", mk, qk)


@pytest.mark.gpu
@pytest.mark.parametrize("where", list(ORIGINS))
def test_walk_past_unvisited_competitors(gpu, where):
    """Walk the scattered queries a quarter cell along a diagonal in steps of h / 64: many cross
    the equal-distance face to a competitor the certifying scans skipped, and every call must
    equal the exact reference while a good share of the answers come from certificates."""
    c = _scattered()
    origin = ORIGINS[where]
    e = _capi.Engine()
    try:
        _, pk = c.H(origin)
        e.set_clouds(to_xyz(pk, origin), to_xyz(c.mk, origin))
        e.set_selected(None)
        K = len(c.qk)
        z = np.zeros(K, dtype=np.float32)
        e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
        set_paths(e, {})
        _, h, _ = e.grid_params("mov")
        step = max(1, int(round(h / 2 ** -10 / 64)))
        counts, changed = [], 0
        ref0 = exact_knn(c.mk, c.qk, 1)[0][:, 0]
        for t in range(17):
            shift = np.array([1, -1, 1]) * step * t
            H, pk = c.H(origin, shift)
            idx, d = e.match(H)
            ref = exact_knn(c.mk, c.qk - shift, 1)[0][:, 0]
            bad = np.flatnonzero(idx != ref)
            assert bad.size == 0, f"{where} step {t}: {bad.size} of {K} differ"
            M = to_xyz(c.mk, origin)
            d_host = rigid_apply(H, M)[ref, 2] - to_xyz(pk, origin)[:, 2]
            assert np.array_equal(d, d_host), f"{where} step {t}: distances"
            counts.append(e.match_counts())
            changed = int((ref != ref0).sum())
        assert changed >= 100, changed          # the walk does cross faces
        # every query moves alike, so their certificates run out on the same steps: count over
        # the walk, not per step
        assert sum(counts[2:]) > K * len(counts[2:]) // 4, counts
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("where", list(ORIGINS))
def test_tied_queries_are_never_certified(gpu, where):
    """Queries with two or more nearest points at the same distance get no certificate: with only
    those selected, repeated matches at the same transform answer none from a certificate, while
    the untied queries are certified."""
    c = cases()["ties"]
    origin = ORIGINS[where]
    _, d2 = exact_knn(c.mk, c.qk, 2)
    tied = np.flatnonzero(d2[:, 0] == d2[:, 1])
    untied = np.flatnonzero(d2[:, 0] != d2[:, 1])
    assert len(tied) >= 1000
    with _engine("ties", where) as e:
        H, _ = c.H(origin)
        for sel, certified in ((tied, False), (untied, True)):
            e.set_selected(sel)
            K = len(sel)
            z = np.zeros(K, dtype=np.float32)
            e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
            ref = exact_knn(c.mk, c.qk[sel], 1)[0][:, 0]
            for it in range(4):
                idx, _ = e.match(H)
                assert np.array_equal(idx, ref), f"{where} call {it}"
                n = e.match_counts()
                if not certified:
                    assert n == 0, f"{where} call {it}: {n} tied queries certified"
                elif it >= 2:
                    assert n > K // 2, f"{where} call {it}: {n} of {K}"


@pytest.mark.gpu
def test_invalidation(gpu):
    """Every change that ends the warm start ends the certificates: a new selection, new clouds,
    another cell size, the brute-force engine and back, and a match without distance
    (select_in_range) are each followed by exact matches; so is an iteration from a far pose,
    where the certificates stay but no moved query is inside its ball."""
    c = cases()["sheet"]
    origin = ORIGINS["utm"]
    with _engine("sheet", "utm") as e:
        def warm(shift=(0, 0, 0)):
            for _ in range(3):
                check_match(e, c, origin, shift, "warm-up")
            assert e.match_counts() > 0

        H, pk = c.H(origin)
        warm()
        # a selection of every second query: query i of the new selection is query 2 i before
        sel = np.arange(0, len(c.qk), 2)
        e.set_selected(sel)
        K = len(sel)
        z = np.zeros(K, dtype=np.float32)
        e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
        idx, _ = e.match(H)
        assert np.array_equal(idx, exact_knn(c.mk, c.qk[sel], 1)[0][:, 0]), "set_selected"
        e.set_selected(None)
        K = len(c.qk)
        z = np.zeros(K, dtype=np.float32)
        e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
        warm()
        # new movable cloud: every point moved by 3 units along z (the same K)
        mk2 = c.mk + [0, 0, 3]
        e.set_clouds(to_xyz(pk, origin), to_xyz(mk2, origin))
        e.set_selected(None)
        e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
        idx, _ = e.match(H)
        assert np.array_equal(idx, exact_knn(mk2, c.qk, 1)[0][:, 0]), "set_clouds"
        # another cell size, the original cloud back
        e.set_option("grid_target_occupancy", 0.25)
        e.set_clouds(to_xyz(pk, origin), to_xyz(c.mk, origin))
        e.set_selected(None)
        e.set_normals(z, z, np.ones(K, dtype=np.float32), np.full(K, 0.9, dtype=np.float32))
        warm()
        e.set_option("nn_engine", _capi.NN_BRUTE)
        check_match(e, c, origin, (5, 0, 0), "brute")
        assert e.match_counts() == 0
        e.set_option("nn_engine", DEFAULTS["nn_engine"])
        check_match(e, c, origin, (0, 0, 0), "grid after brute")
        warm()
        e.select_in_range(c.H(origin, (40, 0, 0))[0], 1.0)
        check_match(e, c, origin, (0, 0, 0), "after select_in_range")
        # an iteration from a far pose (3000 units along x; zero angles keep it exact), then the
        # matches at that pose and back at the start
        warm()
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), [np.inf] * 5 + [0.0], 1.0)
        params = e.run_params(0.0, 1.0, 1, lsq)
        H_far, _ = c.H(origin, (3000, 0, 0))
        e.iterate(params, x_in=list(np.zeros(3)) + list(H_far[:3, 3]))
        check_match(e, c, origin, (3000, 0, 0), "at the far pose of iterate")
        check_match(e, c, origin, (0, 0, 0), "back from the far pose")


def _runs(Xf, Xm, **kw):
    """register with min_change = 0 and 40 iterations, warm start on and off: bit-identical."""
    import simpleicp_b200 as sb

    out = []
    with _capi.Engine() as e:
        for warm in (1, 0):
            e.reset_options()
            e.set_option("warm_start", warm)
            r = sb.register(Xf, Xm, engine=e, want_normals=False, min_change=0.0, max_iterations=40, **kw)
            out.append((np.array(r.H), r.records, np.array(r.residuals), np.array(r.X_mov_transformed)))
            if warm:
                n_last = e.match_counts()
    return out, n_last


@pytest.mark.gpu
@pytest.mark.parametrize("pair", ["dragon", "bunny", "airborne", "c3_utm"])
def test_registration_equals_warm_start_off(gpu, pair):
    if pair == "c3_utm":
        Xf, Xm = _utm_c3()
    else:
        from conftest import load_pair

        Xf, Xm = load_pair(pair)
    (a, b), n_last = _runs(Xf, Xm)
    _same(a, b, pair)
    assert n_last > 0, pair


@pytest.mark.gpu
def test_registration_with_movable_attributes(gpu):
    from conftest import load_pair

    Xf, Xm = load_pair("dragon")
    (a, b), n_last = _runs(Xf, Xm, mov_neighbors=10, max_angle_between_normals=30.0)
    _same(a, b, "dragon mov_neighbors angle")
    assert n_last > 0
