"""Exact median / MAD of every device selection path on adversarial distance distributions.

Each iteration keeps the correspondences with |d - median| <= 3 MAD, where median and MAD are
taken over the planarity survivors.  Three device implementations compute these two order
statistics, and which one runs depends on K, the iteration, the option "fused" and how good
the predictor was (reject_solve.cu):

  radix select                  radix_median (k_reject_solve): iteration 0, the stage API, every fallback
  per-bin key store             fused_select (k_rs_fused, k_rs_batch)
  in-kernel radix fallback      rs_fused_body, G == 1 (K <= 4096 or a batched pair)

Slot 29 of Engine.phase_times() names the path that produced the last record; slot 30 holds
the outcome of the last predictor attempt of the barrier-free kernel.  Engine.seed_predictor sets the predictor directly, so that any distance distribution
can be paired with any prediction.

The harness makes every device distance reproducible on the host bit for bit: a fixed lattice
on the plane z = z0, the same lattice moved by designed z offsets |s_i| < 0.3 (the nearest
neighbour of fixed point i is movable point i), normals injected as exactly (0, 0, 1), and the
rotations and tx, ty fixed by infinite observation weights.  R is then the identity, and the
distance is d = fl(fl(m_z + t_z) - p_z).  The reference is the oracle's reject (np.median and the
unscaled MAD) on the reconstructed distances, compared with ==.
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import numpy as np
import pytest
from scipy.spatial import cKDTree

from oracle import linearized_oracle as LO
from oracle import simpleicp_oracle as O

from simpleicp_b200 import _capi, linearized

A = 1e-2                               # spread of the designed offsets
MIN_PL = float(np.float32(0.3))        # representable in float32: a planarity can equal it exactly
PL_BELOW = float(np.nextafter(np.float32(MIN_PL), np.float32(0)))  # one float32 ulp below
Z0 = (0.0, 1e6)                        # 1e6: cancellation in d as in UTM-scale lidar
DIMS = {1000: (40, 25), 4096: (64, 64), 4097: (241, 17), 20000: (200, 100), 120000: (400, 300)}
SHAPES = ("gauss", "expo", "gap_narrow", "gap_wide", "tie_mass", "tie_majority", "peaked", "grid",
          "negative", "zeros", "planarity")
PINNED = ("negative", "zeros")  # tz held by a stiff observation so the distances keep their sign
GRID_Q = 2.0 ** -14


def bin_cap(K: int) -> int:
    """Members per predictor-histogram bin the key store holds (nn.cu: bin_cap_for)."""
    cap = 32
    while cap < K // 192 and cap < 2048:
        cap *= 2
    return cap


@dataclass
class Case:
    name: str
    K: int
    z0: float
    fix: np.ndarray      # K x 3
    mov: np.ndarray      # K x 3
    nrm: tuple           # three float32 arrays
    pl: np.ndarray       # float32 planarity
    pinned: bool

    @property
    def obs_weight(self):
        return [np.inf] * 5 + [1e8 if self.pinned else 0.0]


def offsets(name: str, K: int, seed: int):
    """Designed z offsets, planarities and normal signs of one distribution shape."""
    rng = np.random.default_rng(seed)
    pl = np.full(K, 0.9, dtype=np.float32)
    flip = np.zeros(K, dtype=bool)
    cap = bin_cap(K)
    if name == "gauss":
        s = A * rng.standard_normal(K)
    elif name == "expo":  # median and mean differ
        s = A * (rng.exponential(1.0, K) - 0.5)
    elif name in ("gap_narrow", "gap_wide"):
        # two halves; the natural predictor bin is ~ 0.8 std / 512 ~ 1e-3 A, so the narrow gap
        # spans ~ 2 bins and the wide one hundreds.  n1 is even: the two middle ranks straddle it.
        gap = A * (2e-3 if name == "gap_narrow" else 0.3)
        w = A * rng.uniform(0.0, 1.0, K)
        s = np.where(np.arange(K) < K // 2, -gap / 2 - w, gap / 2 + w)
        if K % 2:
            pl[K - 1] = np.nan  # the odd one out leaves the statistics set
    elif name == "tie_mass":  # more exact ties at the median than a key-store bin holds
        s = A * rng.standard_normal(K)
        s[: int(1.5 * cap) + 8] = 0.0
    elif name == "tie_majority":  # > 50 % exact ties: MAD = 0, only the ties are kept
        s = A * rng.standard_normal(K)
        s[: int(0.6 * K)] = 0.0
    elif name == "peaked":  # a cluster of (384, bin_cap] members inside one natural predictor bin
        s = A * rng.standard_normal(K)
        n_peak = 600 if cap >= 1024 else max(cap // 2, 8)
        s[:n_peak] = A * 1e-5 * rng.uniform(-1.0, 1.0, n_peak)
    elif name == "grid":  # quantised, symmetric: ties everywhere, on bin edges of power-of-two seeds
        h = GRID_Q * np.round(A * rng.standard_normal(K // 2) / GRID_Q)
        s = np.concatenate((h, -h, np.zeros(K - 2 * h.size)))
    elif name == "negative":
        s = -A * (0.05 + rng.exponential(1.0, K))
    elif name == "zeros":  # exact zeros; a quarter of them through the normal -e_z, i.e. -0.0
        s = A * rng.standard_normal(K)
        nz = K // 2
        s[:nz] = 0.0
        flip[: nz // 4] = True
    elif name == "planarity":  # NaN, exactly the bound (kept), one ulp below (dropped)
        s = A * rng.standard_normal(K)
        m = K // 20
        pl[:m] = np.nan
        pl[m: 2 * m] = np.float32(MIN_PL)
        pl[2 * m: 3 * m] = np.float32(PL_BELOW)
    else:
        raise ValueError(name)
    perm = rng.permutation(K)  # spread ties and special values over every block
    return np.clip(s, -0.29, 0.29)[perm], pl[perm], flip[perm]


def make_case(name: str, K: int, z0: float, seed: int = 7) -> Case:
    nx, ny = DIMS[K]
    ix, iy = np.meshgrid(np.arange(nx, dtype=np.float64), np.arange(ny, dtype=np.float64), indexing="ij")
    x, y = ix.ravel(), iy.ravel()
    s, pl, flip = offsets(name, K, seed + K)
    fix = np.column_stack((x, y, np.full(K, z0)))
    mov = np.column_stack((x, y, z0 + s))
    nz = np.where(flip, np.float32(-1.0), np.float32(1.0)).astype(np.float32)
    nxy = np.where(flip, np.float32(-0.0), np.float32(0.0)).astype(np.float32)
    return Case(name, K, z0, fix, mov, (nxy.copy(), nxy.copy(), nz), pl, name in PINNED)


def distances(case: Case, tz: float) -> np.ndarray:
    """The match kernel's point-to-plane distance at R = I, t = (0, 0, tz): rigid_apply
    (common.cuh) gives (m_x, m_y, fl(m_z + tz)); then (dx nx + dy ny) + dz nz, no FMA."""
    n = [v.astype(np.float64) for v in case.nrm]
    dx = (case.mov[:, 0] + 0.0) - case.fix[:, 0]
    dy = (case.mov[:, 1] + 0.0) - case.fix[:, 1]
    dz = (case.mov[:, 2] + tz) - case.fix[:, 2]
    return (dx * n[0] + dy * n[1]) + dz * n[2]


def reference(case: Case, tz: float, variant: int = 0):
    """(d, keep, median, mad) of one iteration matched at tz."""
    d = distances(case, tz)
    if variant == 0:
        keep, med, mad = O.reject(d, case.pl, MIN_PL)
        return d, keep, med, mad
    # linearised variants: statistics over every correspondence with a planarity (NaN compares
    # false), upper middle elements, limit 3 (1.4826 MAD) (corrpts.cpp:61-66)
    pop = ~np.isnan(case.pl)
    med = LO.median_upper(d[pop])
    mad = LO.mad_upper(d[pop])
    keep = (case.pl.astype(np.float64) >= MIN_PL) & (np.abs(d - med) <= 3.0 * (1.4826 * mad))
    return d, keep, med, mad


def run_params(e, case: Case, max_iterations: int):
    lsq = e.lsq_params(np.zeros(6), np.zeros(6), case.obs_weight, 1.0)
    return e.run_params(MIN_PL, 0.0, max_iterations, lsq)


# --------------------------------------------------------------------------- host-only checks
@pytest.mark.parametrize("K", [1000, 4097, 20000])
@pytest.mark.parametrize("name", SHAPES)
def test_case_design(name, K):
    """The catalogue does what its comments say, and the reconstruction follows the device's
    operation order (checked against an element-by-element Python evaluation)."""
    for z0 in Z0:
        c = make_case(name, K, z0)
        s = c.mov[:, 2] - c.fix[:, 2]
        assert np.all(np.abs(s) < 0.3)
        # nearest neighbour of fixed point i is movable point i, with a margin
        dist, idx = cKDTree(c.mov).query(c.fix, k=2)
        assert np.array_equal(idx[:, 0], np.arange(K)) and np.all(dist[:, 1] > 0.9)
        d = distances(c, 0.0)
        for i in np.random.default_rng(0).choice(K, 50, replace=False):
            n = [float(v[i]) for v in c.nrm]
            dz = (float(c.mov[i, 2]) + 0.0) - float(c.fix[i, 2])
            ref = (0.0 * n[0] + 0.0 * n[1]) + dz * n[2]
            assert np.float64(ref).view(np.int64) == d[i].view(np.int64)
        surv = ~np.isnan(c.pl) & (c.pl.astype(np.float64) >= MIN_PL)
        keep, med, mad = O.reject(d, c.pl, MIN_PL)
        srt = np.sort(d[surv])
        n1 = srt.size
        assert med == 0.5 * (srt[(n1 - 1) // 2] + srt[n1 // 2])
        dev = np.sort(np.abs(d[surv] - med))
        assert mad == 0.5 * (dev[(n1 - 1) // 2] + dev[n1 // 2])
        assert np.array_equal(keep, surv & (np.abs(d - med) <= 3 * mad))
        if name.startswith("gap"):
            assert n1 % 2 == 0 and srt[n1 // 2] - srt[n1 // 2 - 1] >= A * 2e-3
        if name == "tie_mass":
            assert np.sum(d[surv] == med) > bin_cap(K)
        if name == "tie_majority":
            assert mad == 0.0 and keep.sum() == np.sum(d[surv] == med) > n1 // 2
        if name == "negative":
            assert np.all(d < 0)
        if name == "zeros" and z0 == 0.0:
            z = d == 0.0
            assert np.any(z & np.signbit(d)) and np.any(z & ~np.signbit(d))
        if name == "planarity":
            assert np.any(c.pl == np.float32(MIN_PL)) and np.any(c.pl == np.float32(PL_BELOW))
            assert np.all(surv[c.pl == np.float32(MIN_PL)]) and not np.any(surv[c.pl == np.float32(PL_BELOW)])


# --------------------------------------------------------------------------- device harness
def new_engine(case: Case) -> _capi.Engine:
    e = _capi.Engine()
    e.set_clouds(case.fix, case.mov)
    e.set_selected(None)
    e.set_normals(*case.nrm, case.pl)
    return e


def assert_match_reproduced(e, case: Case, tz: float):
    """The host formula against the match kernel, bit for bit (before anything relies on it)."""
    idx, d = e.match(O.rbp_to_H([0.0, 0.0, 0.0, 0.0, 0.0, tz]))
    assert np.array_equal(idx, np.arange(case.K))
    assert np.array_equal(d.view(np.int64), distances(case, tz).view(np.int64)), \
        f"{case.name} K={case.K} z0={case.z0}: device distances differ from fl(fl(m_z + tz) - p_z)"


def assert_record(rec, case: Case, tz_in: float, what: str, check_step: bool = True):
    d, keep, med, mad = reference(case, tz_in)
    n = int(keep.sum())
    assert rec.n_kept == n, f"{what}: n_kept {rec.n_kept} vs {n}"
    assert rec.median == med and rec.mad == mad, f"{what}: median/MAD {rec.median!r}/{rec.mad!r} vs {med!r}/{mad!r}"
    if check_step and not case.pinned and n >= 6:
        # one free parameter and a residual linear in it: the solve is the mean of the kept
        # distances.  The re-centred model carries the translation as fl(c_m + t) - c_f with the
        # movable box centre c_m ~ z0, which rounds it to a few ulps of z0.
        dk = d[keep]
        spread = max(float(dk.max() - dk.min()), A)
        step = -math.fsum(dk) / n
        tol = 1e-15 * spread + 8 * float(np.spacing(np.abs(case.mov[:, 2]).max()))
        assert abs((rec.x[5] - tz_in) - step) <= tol, f"{what}: tz step {rec.x[5] - tz_in!r} vs {step!r}"
    return keep


@functools.lru_cache(maxsize=None)
def cached_case(name, K, z0):
    return make_case(name, K, z0)


# --------------------------------------------------------------------------- a. stage API
@pytest.mark.gpu
@pytest.mark.parametrize("K", [1000, 4096, 4097, 20000, 120000])
@pytest.mark.parametrize("name", SHAPES)
def test_radix_lockstep_stage_api(gpu, name, K):
    """match + reject (radix select: one block for K <= 4096, the cooperative grid above),
    default and linearised variant: keep mask, n_kept, median and MAD exact."""
    for z0 in Z0:
        case = cached_case(name, K, z0)
        with new_engine(case) as e:
            assert_match_reproduced(e, case, 0.0)
            for variant in (0, linearized.VARIANT_LINEARIZED):
                e.set_option("variant", variant)
                e.match(np.eye(4))
                keep, n_kept, st = e.reject(MIN_PL)
                _, keep_o, med, mad = reference(case, 0.0, variant)
                what = f"{name} K={K} z0={z0} variant {variant}"
                assert np.array_equal(keep, keep_o), what
                assert n_kept == int(keep_o.sum()), what
                assert st[0] == med and st[1] == mad, f"{what}: {st[:2]} vs {med!r}, {mad!r}"
                assert e.selection()["path"] == _capi.SEL_PATH_RADIX


# --------------------------------------------------------------------------- b. seeded sweep
U_GRID = (-6.0, -3.0, -0.5, 0.0, 0.5, 3.0, 6.0)
V_GRID = (-9, -6, -3, 0, 2, 4, 6)
SWEEP_K = (1000, 20000, 120000)
# codes the predictor select can return (reject_solve.cuh: SelectOutcome)
FUSED_CODES = {"SEL_OK", "SEL_NO_PREDICTION", "SEL_MEDIAN_OUTSIDE", "SEL_MEDIAN_GAP", "SEL_MEDIAN_CANDIDATES",
               "SEL_MAD_BRACKET", "SEL_MAD_WINDOW", "SEL_MAD_CANDIDATES", "SEL_BIN_CAP"}


@functools.lru_cache(maxsize=None)
def seeded_sweep(name, K, z0):
    """Run the whole seeded grid for one case; return what was observed."""
    case = cached_case(name, K, z0)
    obs = {"fused": set(), "paths": set(), "cnt_med_store": [], "cells": 0}
    x0 = np.zeros(6)
    with new_engine(case) as e:
        assert_match_reproduced(e, case, 1.5e-3)
        p = run_params(e, case, 2)
        results = {}
        for fused in (1, 0):
            e.set_option("fused", fused)
            for u in U_GRID:
                for v in V_GRID:
                    r0 = e.iterate(p, x_in=x0, want_record=True)
                    note(obs, e.selection(), fused and K <= 4096)
                    tz1 = r0.x[5]
                    d1, keep1, m, s = reference(case, tz1)
                    scale = s if s > 0 else A * 2.0 ** -10  # MAD = 0: seeds of a positive width
                    e.seed_predictor(m + u * scale, scale * 2.0 ** v, MIN_PL)
                    r1 = e.iterate(p, want_record=True)
                    sel = e.selection()
                    note(obs, sel, fused)
                    what = f"{name} K={K} z0={z0} fused={fused} u={u} v={v} sel={sel}"
                    assert_record(r1, case, tz1, what)
                    if fused and sel["path"] == _capi.SEL_PATH_BINSTORE:
                        obs["cnt_med_store"].append(sel["cnt_med"])
                    results[(fused, u, v)] = (tz1, r1.n_kept, r1.median, r1.mad)
                    obs["cells"] += 1
        for u in U_GRID:
            for v in V_GRID:
                a, b = results[(1, u, v)], results[(0, u, v)]
                if a[0] == b[0]:  # same iteration-0 solve (different kernels for K <= 4096)
                    assert a == b, f"{name} K={K} z0={z0} u={u} v={v}: fused {a} vs cooperative {b}"
    return obs


def note(obs, sel, fused):
    """Record the fresh diagnostics of the last iterate(): the path, and slot 30 after a
    barrier-free launch.  fused: the iteration ran in the barrier-free kernel."""
    obs["paths"].add(sel["path"])
    if fused:
        obs["fused"].add(sel["fused"])


@pytest.mark.gpu
@pytest.mark.parametrize("K", SWEEP_K)
@pytest.mark.parametrize("name", SHAPES)
def test_seeded_predictor_sweep(gpu, name, K):
    """Any finite prediction with MAD > 0 gives NumPy's order statistics exactly, through the
    barrier-free and the cooperative kernel alike."""
    for z0 in Z0:
        obs = seeded_sweep(name, K, z0)
        assert obs["cells"] == 2 * len(U_GRID) * len(V_GRID)


@pytest.mark.gpu
def test_seeded_sweep_reaches_every_outcome(gpu):
    """The sweep reaches every reason code and the success of the predictor select, every
    selection path, and both selections inside fused_select (rank_select for <= 384 median
    candidates, block_select above)."""
    fused, paths, cnt = set(), set(), []
    for name in SHAPES:
        for K in SWEEP_K:
            for z0 in Z0:
                obs = seeded_sweep(name, K, z0)
                fused |= obs["fused"]
                paths |= obs["paths"]
                cnt += obs["cnt_med_store"]
    inv = {v: k for k, v in _capi.SEL_OUTCOMES.items()}
    seen_f = {inv[c] for c in fused}
    print(f"barrier-free outcomes {sorted(seen_f)}\n"
          f"paths {sorted(paths)}, key-store cnt_med range {min(cnt)}..{max(cnt)}")
    assert seen_f == FUSED_CODES
    assert set(_capi.SEL_OUTCOMES) == FUSED_CODES
    assert paths == {_capi.SEL_PATH_RADIX, _capi.SEL_PATH_BINSTORE}
    assert min(cnt) <= 384 < max(cnt)


# --------------------------------------------------------------------------- c. minpl mismatch
@pytest.mark.gpu
@pytest.mark.parametrize("K", [1000, 20000])
def test_seeded_minpl_mismatch_falls_back(gpu, K):
    """A predictor made for another planarity bound is not used; the statistics stay exact."""
    case = cached_case("planarity", K, 0.0)
    with new_engine(case) as e:
        p = run_params(e, case, 2)
        for fused in (1, 0):
            e.set_option("fused", fused)
            r0 = e.iterate(p, x_in=np.zeros(6), want_record=True)
            _, _, m, s = reference(case, r0.x[5])
            e.seed_predictor(m, s, PL_BELOW)  # would be a perfect prediction for the other bound
            r1 = e.iterate(p, want_record=True)
            sel = e.selection()
            assert_record(r1, case, r0.x[5], f"K={K} fused={fused}")
            assert sel["path"] == _capi.SEL_PATH_RADIX
            if fused:
                assert sel["fused"] == _capi.SEL_NO_PREDICTION
            # the same seed with the right bound passes the guard (whether the plan then brackets
            # the ranks depends on the sample: at K = 1000 the two middle elements of an even n1
            # are often more than 4 bins of MAD / 512 apart)
            e.iterate(p, x_in=np.zeros(6), want_record=True)
            e.seed_predictor(m, s, MIN_PL)
            r1 = e.iterate(p, want_record=True)
            sel = e.selection()
            assert_record(r1, case, r0.x[5], f"K={K} fused={fused} matching bound")
            if fused:
                assert sel["fused"] != _capi.SEL_NO_PREDICTION


# --------------------------------------------------------------------------- d. whole runs
def run_and_check(e, case: Case, max_iterations: int = 8):
    out, recs, res = e.run(run_params(e, case, max_iterations))
    assert out.iterations == max_iterations  # min_change = 0: the stop rule never fires
    tz = 0.0
    keep = None
    for it, r in enumerate(recs):
        keep = assert_record(r, case, tz, f"{case.name} K={case.K} z0={case.z0} it {it}")
        tz = r.x[5]
    d = distances(case, tz)  # the residuals at the final transform, kept order
    assert np.array_equal(res.view(np.int64), d[keep].view(np.int64))
    return out, recs, res


def rec_tuple(r):
    return (r.n_kept, r.median, r.mad, tuple(r.x), r.mean_res, r.std_res)


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1000, 20000])
@pytest.mark.parametrize("name", SHAPES)
def test_whole_runs_natural_prediction(gpu, name, K):
    """Engine.run with the predictor the iterations leave behind: every record against the host
    reference, barrier-free kernel against the cooperative kernel record by record."""
    for z0 in Z0:
        case = cached_case(name, K, z0)
        with new_engine(case) as e:
            a = run_and_check(e, case)
            ta = e.timings()
            e.set_option("fused", 0)
            b = run_and_check(e, case)
        # the two kernels sum the moments in different orders: the solves agree to rounding, and
        # records taken at the same transform agree exactly
        tz_a = tz_b = 0.0
        for ra, rb in zip(a[1], b[1]):
            if tz_a == tz_b:
                assert (ra.n_kept, ra.median, ra.mad) == (rb.n_kept, rb.median, rb.mad)
            np.testing.assert_allclose(ra.x[5], rb.x[5], rtol=0, atol=1e-15 + 8 * np.spacing(z0))
            tz_a, tz_b = ra.x[5], rb.x[5]
        if tz_a == tz_b:
            assert np.array_equal(a[2], b[2])
        if K > 4096 and name in ("tie_mass", "tie_majority"):
            assert ta["rerun_iterations"] > 0, f"{name} z0={z0}: {ta}"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tie_mass", "tie_majority"])
def test_missed_prediction_with_queued_iterations(gpu, name):
    """A missed prediction parks the pipeline and the host repeats the iteration through the
    general kernel; with iterations queued behind the miss the outcome must not depend on how
    many there were."""
    for z0 in Z0:
        case = cached_case(name, 20000, z0)
        runs = []
        with new_engine(case) as e:
            for every in (1, 4, 7):
                e.set_option("host_sync_every", every)
                out, recs, res = run_and_check(e, case)
                runs.append((out.iterations, tuple(out.H), [rec_tuple(r) for r in recs], res.tobytes(),
                             e.timings()["rerun_iterations"]))
        print(f"{name} z0={z0}: re-run iterations {[r[4] for r in runs]}")
        assert all(r[4] > 0 for r in runs)
        assert all(r[:4] == runs[0][:4] for r in runs)


# --------------------------------------------------------------------------- e. small counts
@pytest.mark.gpu
@pytest.mark.parametrize("K", [1000, 4097])
def test_small_and_boundary_counts(gpu, K):
    """n1 planarity survivors in {0, 1, 2, 3, 5, 6, 7, 8}: fewer than 6 kept correspondences
    raise SICP_ERR_TOO_FEW_CORR, six or more run, with exact statistics."""
    seen = {}
    base = make_case("gauss", K, 0.0)
    for n1 in (0, 1, 2, 3, 5, 6, 7, 8):
        pl = np.full(K, np.nan, dtype=np.float32)
        sel = np.random.default_rng(n1).choice(K, n1, replace=False)
        pl[sel] = 0.9
        mov = base.mov.copy()
        mov[sel, 2] = A * (np.arange(n1) - (n1 - 1) / 2)  # symmetric: every survivor is kept
        case = Case("small", K, 0.0, base.fix, mov, base.nrm, pl, False)
        n_kept = int(reference(case, 0.0)[1].sum())
        with new_engine(case) as e:
            for fused in (1, 0):
                e.set_option("fused", fused)
                if n_kept < 6:
                    with pytest.raises(_capi.SicpError) as ex:
                        e.run(run_params(e, case, 8))
                    assert ex.value.code == _capi.SICP_ERR_TOO_FEW_CORR
                    assert f"correspondences is {n_kept}." in ex.value.message
                else:
                    run_and_check(e, case)
            # the engine stays usable after the error
            ok = make_case("gauss", K, 0.0)
            e.set_clouds(ok.fix, ok.mov)
            e.set_selected(None)
            e.set_normals(*ok.nrm, ok.pl)
            run_and_check(e, ok, 2)
        seen[n_kept] = n1
    assert 5 in seen and 6 in seen and 0 in seen


# --------------------------------------------------------------------------- f. batched engine
@pytest.mark.gpu
def test_batched_engine_on_lattices(gpu):
    """register_batch on lattice pairs (normals estimated on the device) against per-pair
    registration, and the per-pair records against the host reference.  tie_mass at K = 1000
    misses its key-store bin every iteration, so the in-kernel radix fallback runs."""
    names = ["gauss", "tie_mass", "gap_wide", "planarity"]
    cases = [cached_case(n, 1000, 0.0) for n in names]
    with _capi.Engine() as e:
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), [np.inf] * 5 + [0.0], 1.0)
        params = e.run_params(MIN_PL, 0.0, 6, lsq)
        res = e.register_batch([(c.fix, c.mov) for c in cases], 1000, 10, params)
        for c, b in zip(cases, res):
            e.set_clouds(c.fix, c.mov)
            e.set_selected(None)
            nx, ny, nz, pl = e.estimate_normals(10)
            ez = (nx == 0) & (ny == 0) & (np.abs(nz) == 1)
            print(f"{c.name}: estimated normals exactly +-e_z: {ez.mean():.4f}")
            out, recs, resid, _ = e.register_fused(c.fix, c.mov, 1000, 10, -1.0, params)
            sel = e.selection()
            assert b.status == 0
            assert (b.iterations, b.n_kept) == (out.iterations, out.n_residuals)
            np.testing.assert_allclose(np.array(b.H), np.array(out.H), rtol=0, atol=1e-12)
            if c.name == "tie_mass":
                assert sel["fused"] == _capi.SEL_BIN_CAP and sel["path"] == _capi.SEL_PATH_RADIX
            if ez.all():
                host = Case(c.name, c.K, c.z0, c.fix, c.mov, (nx, ny, nz), pl, False)
                tz = 0.0
                for it, r in enumerate(recs):
                    assert_record(r, host, tz, f"batch {c.name} it {it}")
                    tz = r.x[5]
