"""Host-side tests of the joint registration with relative pose observations (DESIGN.md §6.13):
simpleicp_joint's argument checks, the C entry point and its declaration, and the NumPy restatement
with observations (joint_relative_oracle.py, on top of joint_prior_oracle.py): no observation read,
the linearisation against finite differences, a huge weight from a fixed cloud against holding the
relative pose, and the s0 rule with observations."""
import re
from pathlib import Path

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import simpleicp_b200 as sb
from oracle import joint_oracle as J
from simpleicp_b200 import _capi
from simpleicp_b200.batch import _joint_relative, relative_misclosure

import joint_prior_cov_rule
import joint_prior_oracle as JPO
import joint_relative_cov_rule
import joint_relative_oracle as JRO
from test_joint_host import ring

REPO = Path(__file__).resolve().parents[1]


def _clouds(n=4, m=200):
    rng = np.random.default_rng(1)
    return [rng.normal(size=(m, 3)) for _ in range(n)]


def _eye(n=2):
    return np.tile(np.eye(4), (n, 1, 1))


def _w(n=2, v=1.0):
    return np.full((n, 6), v)


def _set(a, idx, v):
    a = a.copy()
    a[idx] = v
    return a


_P = [(1, 2), (2, 3)]


@pytest.mark.parametrize("kw,msg", [
    ({"relative_pairs": _P}, "given together"),
    ({"relative_pairs": _P, "relative_poses": _eye()}, "given together"),
    ({"relative_poses": _eye(), "relative_weights": _w()}, "given together"),
    ({"relative_pairs": [1, 2], "relative_poses": _eye(), "relative_weights": _w()}, r"shape \(n_rel, 2\)"),
    ({"relative_pairs": [(1.0, 2.0)], "relative_poses": _eye(1), "relative_weights": _w(1)}, "integers"),
    ({"relative_pairs": [(1, 4)], "relative_poses": _eye(1), "relative_weights": _w(1)}, "index the 4 clouds"),
    ({"relative_pairs": [(-1, 2)], "relative_poses": _eye(1), "relative_weights": _w(1)}, "index the 4 clouds"),
    ({"relative_pairs": [(1, 2), (2, 2)], "relative_poses": _eye(), "relative_weights": _w()},
     r"join two clouds: observation 1"),
    ({"edges": [(0, 1), (1, 2)], "relative_pairs": [(1, 3)], "relative_poses": _eye(1), "relative_weights": _w(1)},
     "observation 0 joins a cloud that no edge references"),
    ({"relative_pairs": _P, "relative_poses": _eye(3), "relative_weights": _w()},
     r"relative_poses must have shape \(2, 4, 4\)"),
    ({"relative_pairs": _P, "relative_poses": _eye(), "relative_weights": _w()[:, :5]},
     r"relative_weights must have shape \(2, 6\)"),
    ({"relative_pairs": _P, "relative_poses": _eye(), "relative_weights": _set(_w(), (1, 2), -1.0)}, "finite and >= 0"),
    ({"relative_pairs": _P, "relative_poses": _eye(), "relative_weights": _set(_w(), (0, 4), np.nan)},
     "finite and >= 0"),
    ({"relative_pairs": _P, "relative_poses": _eye(), "relative_weights": _set(_w(), (0, 0), np.inf)},
     "finite and >= 0"),
    # the weights of an observation that is not read are checked all the same
    ({"relative_pairs": _P, "relative_poses": _eye(), "relative_weights": _set(_set(_w(), 1, 0.0), (1, 0), -2.0)},
     "finite and >= 0"),
    ({"relative_pairs": _P, "relative_poses": _set(_eye(), (1, 0, 3), np.nan), "relative_weights": _w()},
     r"relative_poses\[1\] has non-finite"),
    ({"relative_pairs": _P, "relative_poses": _set(_eye(), (1, 0, 0), 1.0 + 1e-5), "relative_weights": _w()},
     "orthonormal"),
    ({"relative_pairs": _P, "relative_poses": _set(_eye(), (0, 3, 1), 1e-3), "relative_weights": _w()}, "bottom row"),
    ({"relative_pairs": np.zeros((65536, 2), dtype=np.int64), "relative_poses": _eye(65536),
      "relative_weights": _w(65536)}, "at most 65535"),
    # fixed=() is accepted with observations, but they anchor nothing
    ({"fixed": (), "relative_pairs": _P, "relative_poses": _eye(), "relative_weights": _w()},
     "free cloud 0 has no path to a fixed cloud over the edges and the relative observations with six non-zero"),
    # clouds 2 and 3 are tied to the rest only by a position-only observation: no link
    ({"edges": [(0, 1), (2, 3)], "relative_pairs": [(1, 2)], "relative_poses": _eye(1),
      "relative_weights": _set(_w(1), (0, slice(0, 3)), 0.0)},
     "free cloud 2 has no path to a fixed cloud over the edges and the relative observations"),
])
def test_relative_argument_checks(kw, msg):
    kw = dict(kw)
    edges = kw.pop("edges", [(0, 1), (1, 2), (2, 3)])
    with pytest.raises(ValueError, match=msg):
        sb.simpleicp_joint(_clouds(), edges, **kw)


def test_without_observations_the_messages_are_unchanged():
    with pytest.raises(ValueError, match=r"^fixed must be a sequence of at least one integer cloud index$"):
        sb.simpleicp_joint(_clouds(), [(0, 1)], fixed=())
    with pytest.raises(ValueError, match=r"^free cloud 2 has no path to a fixed cloud over the edges$"):
        sb.simpleicp_joint(_clouds(), [(0, 1), (2, 3)])
    with pytest.raises(ValueError, match=r"^free cloud 1 has no path to a fixed cloud over the edges and no pose prior "
                                         r"with six non-zero weights in its component$"):
        sb.simpleicp_joint(_clouds(), [(1, 2)], prior_poses=_eye(4), prior_weights=_w(4, 0.0))


def test_observations_that_are_not_read_may_hold_nan():
    """Observation 0 joins two fixed clouds, observation 1 has zero weights: their poses are not
    read.  Observation 2 (six weights > 0) links its clouds, observation 3 (rotation only) does not;
    a rotation inside 1e-6 of orthonormal passes."""
    used = np.array([True, True, True, True, False])
    free = np.array([False, False, True, True, False])
    pairs = [(0, 1), (2, 3), (1, 2), (3, 0)]
    Z = _eye(4)
    Z[[0, 1]] = np.nan
    Z[2, :3, :3] *= 1.0 + 4e-7
    W = np.ones((4, 6))
    W[1] = 0.0
    W[3, 3:] = 0.0
    p, Zc, Wc, link = _joint_relative(pairs, Z, W, used, free)
    assert list(link) == [False, False, True, False]
    assert p.dtype == np.int64 and Zc.dtype == Wc.dtype == np.float64
    with pytest.raises(ValueError, match="no edge references"):
        _joint_relative([(1, 4)], _eye(1), _w(1), used, free)


def test_c_entry_point_and_declaration():
    """sicp_register_joint_relative is sicp_register_joint_priors plus five parameters after
    prior_w; the priors' declaration keeps its 15 parameters and the ABI version stays 5."""
    header = (REPO / "include" / "sicp_b200.h").read_text()
    assert int(re.search(r"#define SICP_ABI_VERSION (\d+)", header).group(1)) == _capi.ABI_VERSION == 5
    params = {}
    for name in ("sicp_register_joint_priors", "sicp_register_joint_relative"):
        decl = re.search(rf"int32_t {name}\(([^;]*)\);", header)
        assert decl and name in _capi.SYMBOLS
        params[name] = [p.split()[-1].lstrip("*") for p in re.sub(r"/\*.*?\*/", "", decl.group(1)).split(",")]
    pri, rel = params["sicp_register_joint_priors"], params["sicp_register_joint_relative"]
    assert len(pri) == 15 and len(rel) == 20
    assert rel[:11] == pri[:11] and rel[16:] == pri[11:]
    assert rel[11:16] == ["n_rel", "rel_a", "rel_b", "rel_H", "rel_w"]
    lib = _capi.load_library()
    assert len(lib.sicp_register_joint_relative.argtypes) == 20
    args = [None, 1, None, None, 1, None, None, None, None, None, None, 0, None, None, None, None, None, None, None,
            None]
    assert lib.sicp_register_joint_relative(*args) == _capi.SICP_ERR_BAD_ARG
    assert b"NULL" in lib.sicp_last_error(None)


def _rel_ring(truth, seed=3, rot_deg=0.02, pos_m=0.01):
    """Odometry along the ring: (i, i + 1) from the truth with seeded noise, weights for rows of 5 mm;
    and one observation (2, 6) between clouds no edge joins, position only."""
    rng = np.random.default_rng(seed)
    pairs, Z = [], []
    for a, b in [(i, i + 1) for i in range(len(truth) - 1)] + [(2, 6)]:
        dx = np.concatenate((np.deg2rad(rng.normal(0, rot_deg, 3)), rng.normal(0, pos_m, 3)))
        E = np.eye(4)
        E[:3, :3] = Rotation.from_rotvec(dx[:3]).as_matrix()
        E[:3, 3] = dx[3:]
        Z.append(np.linalg.inv(truth[a]) @ truth[b] @ E)
        pairs.append((a, b))
    W = np.tile([0.005 ** 2 / np.deg2rad(rot_deg) ** 2] * 3 + [0.005 ** 2 / pos_m ** 2] * 3, (len(pairs), 1))
    W[-1, :3] = 0.0
    return np.array(pairs), np.array(Z), W


def test_oracle_without_observations_read_gives_the_prior_restatement_bit_for_bit():
    scans, truth, H0, edges = ring()
    kw = dict(fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    pairs, Z, W = _rel_ring(truth)
    for solver in ("dense", "sparse"):
        a = JPO.simpleicp_joint(scans, edges, solver=solver, **kw)
        unread = [dict(),
                  dict(relative_pairs=pairs, relative_poses=np.full_like(Z, np.nan), relative_weights=np.zeros_like(W)),
                  # both ends fixed
                  dict(relative_pairs=[(0, 0)], relative_poses=np.full((1, 4, 4), np.nan), relative_weights=_w(1))]
        for obs in unread:
            b = JRO.simpleicp_joint(scans, edges, solver=solver, **obs, **kw)
            assert np.array_equal(a.H, b.H) and len(a.log) == len(b.log) and a.converged == b.converged
            for ra, rb in zip(a.log, b.log):
                assert [(e.n_kept, e.mean, e.std) for e in ra] == [(e.n_kept, e.mean, e.std) for e in rb]


def _exact_l(Ta, Tb, Z):
    """l(T_a, T_b) from its definition, with SciPy's rotation vector."""
    Rab = Ta[:3, :3].T @ Tb[:3, :3]
    tab = Ta[:3, :3].T @ (Tb[:3, 3] - Ta[:3, 3])
    return np.concatenate((Rotation.from_matrix(Z[:3, :3] @ Rab.T).as_rotvec(), Z[:3, 3] - tab))


@pytest.mark.parametrize("origin", [(0.0, 0.0, 0.0), (4.5e5, 5.4e6, 300.0)])
def test_linearisation_against_finite_differences(origin):
    """u = B_b x_b - B_a x_a with B_c = G_c J_c is the first-order change of T_a^-1 T_b under the
    increments x_c (about the world origin, T_c <- dH(x_c) T_c), so dl/dx_b = -B_b and dl/dx_a = B_a
    at an observation whose rotation equals R_ab (its translation is arbitrary).  Central
    differences on random poses, near the origin and at UTM coordinates."""
    rng = np.random.default_rng(11)
    for _ in range(5):
        T = []
        for _ in range(2):
            H = np.eye(4)
            H[:3, :3] = Rotation.from_rotvec(rng.normal(0, 1.0, 3)).as_matrix()
            H[:3, 3] = np.asarray(origin) + rng.uniform(-50, 50, 3)
            T.append(H)
        Ta, Tb = T
        Z = np.linalg.inv(Ta) @ Tb
        Z[:3, 3] += rng.normal(0, 0.5, 3)
        Ba, Bb = JRO.jacobians(Ta, Tb)
        assert np.allclose(JRO.observe(Ta, Tb, Z), _exact_l(Ta, Tb, Z), rtol=0, atol=1e-9)
        h = 1e-6
        for side, B, sg in ((0, Ba, 1.0), (1, Bb, -1.0)):
            D = np.zeros((6, 6))
            for j in range(6):
                x = np.zeros(6)
                x[j] = h
                Tp, Tm = list(T), list(T)
                Tp[side] = J.rigid_from_x(x) @ T[side]
                Tm[side] = J.rigid_from_x(-x) @ T[side]
                D[:, j] = (_exact_l(*Tp, Z) - _exact_l(*Tm, Z)) / (2 * h)
            scale = max(1.0, np.abs(B).max())
            assert np.abs(D - sg * B).max() <= 1e-6 * scale, (side, np.abs(D - sg * B).max(), scale)


def test_oracle_huge_weight_from_a_fixed_cloud_holds_the_relative_pose():
    """An observation (0, 3) from fixed cloud 0 with Z = H0[0]^-1 H0[3] and weights 1e12 against
    cloud 3 in fixed: the same bound as test_joint_prior_host's huge prior, 1e3 |N| / w."""
    scans, truth, H0, edges = ring()
    kw = dict(H0=H0, max_iterations=30, max_overlap_distance=1.0)
    fixed = J.simpleicp_joint(scans, edges, fixed=(0, 3), **kw)
    Z = (np.linalg.inv(H0[0]) @ H0[3])[None]
    rel = JRO.simpleicp_joint(scans, edges, fixed=(0,), relative_pairs=[(0, 3)], relative_poses=Z,
                              relative_weights=_w(1, 1e12), **kw)
    s = J.first_iteration_sums(scans, edges, fixed=(0,), H0=H0, max_overlap_distance=1.0)
    Nnorm = max(np.linalg.norm(J.ad_world_to_frame(Ta).T @ N @ J.ad_world_to_frame(Ta), 2)
                for N, Ta in zip(s.N, s.T_a))
    assert 1e4 < Nnorm < 1e6
    assert len(rel.log) == len(fixed.log)
    for ra, rb in zip(rel.log, fixed.log):
        assert [e.n_kept for e in ra] == [e.n_kept for e in rb]
    assert np.abs(rel.H - fixed.H).max() < 1e3 * Nnorm / 1e12


def test_oracle_odometry_links_two_components():
    """Edges (0, 1), (1, 2) and (3, 4), (4, 5) of the ring's scans with no edge across: one
    full-weight observation (2, 3) from the truth brings the second component to the truth.  (Edge
    (3, 4)'s kept count keeps changing by one or two rows, so its stop rule is not met in 30
    iterations.)"""
    scans, truth, H0, _ = ring()
    edges = [(0, 1), (1, 2), (3, 4), (4, 5)]
    Z = (np.linalg.inv(truth[2]) @ truth[3])[None]
    res = JRO.simpleicp_joint(scans, edges, fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0,
                              relative_pairs=[(2, 3)], relative_poses=Z, relative_weights=_w(1, 1e4))
    assert np.abs(res.H[:6] - truth[:6]).max() < 1e-2  # measured: 3.6 mm


def test_s0_rule_with_observations():
    """Zero weights give joint_prior_cov_rule's N, s0 and covariances; with observations s0 counts
    their residuals and weights, and N holds their off-diagonal block of clouds 2 and 6, which no
    edge joins."""
    scans, truth, H0, edges = ring()
    kw = dict(fixed=(0,), H0=H0, max_iterations=30, max_overlap_distance=1.0)
    res = JPO.simpleicp_joint(scans, edges, **kw)
    base = joint_prior_cov_rule.final_iteration(scans, edges, res, **kw)
    pairs, Z, W = _rel_ring(truth)
    zero = joint_relative_cov_rule.final_iteration(scans, edges, res, relative_pairs=pairs,
                                                   relative_poses=np.full_like(Z, np.nan),
                                                   relative_weights=np.zeros_like(W), **kw)
    assert np.array_equal(zero.N, base.N) and zero.s0 == base.s0 and np.array_equal(zero.cov, base.cov)
    resr = JRO.simpleicp_joint(scans, edges, relative_pairs=pairs, relative_poses=Z, relative_weights=W, **kw)
    fi = joint_relative_cov_rule.final_iteration(scans, edges, resr, relative_pairs=pairs, relative_poses=Z,
                                                 relative_weights=W, **kw)
    assert np.abs(fi.H - resr.H).max() < 1e-12
    assert len(fi.rels) == len(pairs) and np.isfinite(fi.s0)
    i2, i6 = 6 * fi.slot[2], 6 * fi.slot[6]
    assert np.abs(fi.N[i6:i6 + 6, i2:i2 + 6]).max() > 0 and np.array_equal(fi.N[i6:i6 + 6, i2:i2 + 6],
                                                                            fi.N[i2:i2 + 6, i6:i6 + 6].T)


def test_misclosure_against_a_statement():
    """relative_misclosure: (rotvec(R_Z R_ab^T), t_Z - t_ab), with rotations up to pi."""
    rng = np.random.default_rng(4)
    H = np.tile(np.eye(4), (3, 1, 1))
    for c in range(3):
        H[c, :3, :3] = Rotation.from_rotvec(rng.normal(0, 1, 3)).as_matrix()
        H[c, :3, 3] = rng.normal(0, 100, 3)
    pairs = np.array([(0, 1), (1, 2), (2, 0), (0, 2)])
    Z = np.tile(np.eye(4), (4, 1, 1))
    angles = [0.3, 2.5, np.pi - 1e-9, 0.0]
    for k, (a, b) in enumerate(pairs):
        axis = rng.normal(size=3)
        E = Rotation.from_rotvec(angles[k] * axis / np.linalg.norm(axis)).as_matrix()
        Rab = H[a, :3, :3].T @ H[b, :3, :3]
        Z[k, :3, :3] = E @ Rab
        Z[k, :3, 3] = rng.normal(0, 1, 3)
    m = relative_misclosure(H, pairs, Z)
    for k, (a, b) in enumerate(pairs):
        ref = _exact_l(H[a], H[b], Z[k])
        if angles[k] > 3.0:  # near pi the sign of the vector is free: compare the rotations
            Rm, Rr = Rotation.from_rotvec(m[k, :3]).as_matrix(), Rotation.from_rotvec(ref[:3]).as_matrix()
            assert np.abs(Rm - Rr).max() < 1e-9
        else:
            assert np.abs(m[k, :3] - ref[:3]).max() < 1e-12
        assert np.abs(m[k, 3:] - ref[3:]).max() < 1e-9
