"""CPU: the eigen-solver of the normal kernel (csrc/eig3.cuh, compiled here with g++) against
np.linalg.eig — values to 1e-12, and LAPACK dgeev's eigenvector SIGNS, which the reference
inherits (pointcloud.py:191-197) and which decide the sign of every point-to-plane distance."""
import ctypes as C
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

from conftest import REPO, load_pair


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("eig3") / "libeig3_host.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                    str(REPO / "tests" / "native" / "eig3_host.cpp"), "-o", str(out)], check=True)
    lib = C.CDLL(str(out))
    lib.eig3_dgeev_host.restype = C.c_int
    return lib


def covariances(name, k, n=2000):
    X_fix, _ = load_pair(name)
    idx = np.round(np.linspace(0, len(X_fix) - 1, n)).astype(int)
    _, nn = cKDTree(X_fix).query(X_fix[idx], k=k)
    return [np.cov(X_fix[row].T) for row in nn]


def dgeev(lib, Cm):
    A = np.ascontiguousarray(Cm, dtype=np.float64)
    wr = np.zeros(3)
    vr = np.zeros((3, 3))
    assert lib.eig3_dgeev_host(A.ctypes.data_as(C.c_void_p), wr.ctypes.data_as(C.c_void_p),
                               vr.ctypes.data_as(C.c_void_p)) == 1
    return wr, vr


def smallest(lib, Cm, mode=0):
    """eig3_smallest as the normal kernels store it: float32 normal, float32 planarity."""
    c6 = np.array([Cm[0, 0], Cm[0, 1], Cm[0, 2], Cm[1, 1], Cm[1, 2], Cm[2, 2]], dtype=np.float64)
    w = np.zeros(3)
    n = np.zeros(3)
    lib.eig3_smallest_host(c6.ctypes.data_as(C.c_void_p), C.c_int(mode), w.ctypes.data_as(C.c_void_p),
                           n.ctypes.data_as(C.c_void_p))
    return n.astype(np.float32), np.float32((w[1] - w[2]) / w[0])


def numpy_normal(Cm):
    """The reference's normal and planarity (pointcloud.py:190-198)."""
    w, v = np.linalg.eig(Cm)
    o = w.argsort()[::-1]
    w, v = w[o], v[:, o]
    with np.errstate(invalid="ignore"):
        return v[:, 2].astype(np.float32), np.float32((w[1] - w[2]) / w[0])


def same_f32(a, b):
    """Bit for bit; NaN equals NaN whatever its payload."""
    a, b = np.atleast_1d(a), np.atleast_1d(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


# slot / vector mismatches measured with NumPy 2.3 on OpenBLAS 0.3.30 (see the test)
RESIDUE_BOUND = {"dragon": 2, "bunny": 6, "webots": 6, "terrestrial": 4}


@pytest.mark.parametrize("name,k", [("dragon", 10), ("bunny", 10), ("webots", 40), ("terrestrial", 10)])
def test_dgeev_emulation_matches_numpy(lib, name, k):
    bound = RESIDUE_BOUND[name]
    n_bad = n_bad32 = n_tot = 0
    for Cm in covariances(name, k, 4000 if name == "terrestrial" else 2000):
        if not np.isfinite(Cm).all() or np.abs(Cm).max() == 0:
            continue
        w, v = np.linalg.eig(Cm)
        wr, vr = dgeev(lib, Cm)
        # eigenvalues as a set, eigenvectors up to sign: always
        np.testing.assert_allclose(np.sort(wr), np.sort(w), rtol=1e-9, atol=1e-18)
        order = [int(np.argmin(np.abs(w - x))) for x in wr]
        for c in range(3):
            assert abs(abs(np.dot(vr[:, c], v[:, order[c]])) - 1.0) < 1e-6
        n_tot += 1
        n_bad += int(not (np.allclose(wr, w, rtol=1e-9, atol=1e-18) and np.allclose(vr, v, atol=1e-7)))
        n_bad32 += int(not same_f32(smallest(lib, Cm)[0], numpy_normal(Cm)[0]))
    # slot order AND sign agree except where a deflation test sits within rounding of its
    # threshold (DESIGN.md "normal sign"); canonical-sign agreement would be ~50 %.  The bound is
    # the measured count (NumPy 2.3 on OpenBLAS 0.3.30): dragon 2, bunny 6, webots 6, terrestrial
    # 4.  Float32 normals that differ in a last bit (values equal to 1e-7) are printed, not bounded.
    print(f"{name}: {n_bad} of {n_tot} slot/vector mismatches, {n_bad32} float32 normals differ")
    assert n_bad <= bound, (n_bad, n_tot)


# --------------------------------------------------------------------------- designed covariances
# Every family below is built so that LAPACK's dgebal (called by dgeev with job 'B') takes a
# known permutation: `hi` is the last row of the block the QR runs on, `perm` the rows dgebal
# swapped into positions hi + 1 .. 2 (0-based).  Exact zeros come from exact constructions: zero
# entries set in the matrix, or points whose deviations from their mean are exactly zero in one
# coordinate or pair up symmetrically.  Not here: a rank-1 covariance without a zero entry (a
# line along (1, -1, 2)).  Its two zero eigenvalues come out of the QR as rounding noise (NumPy
# even returns a complex pair for some), so neither the slots nor the float32 normal are
# reproducible bit for bit; its planarity is noise / l_max in the reference too.
def _spd(rng, zeros=()):
    """Random symmetric matrix, diagonally dominant, with the listed off-diagonals exactly zero."""
    M = rng.normal(size=(3, 3))
    M = M + M.T
    for i, j in zeros:
        M[i, j] = M[j, i] = 0.0
    M[np.diag_indices(3)] = np.abs(M).sum(1) + rng.uniform(0.1, 2.0, 3)
    return M * 10.0 ** rng.integers(-6, 3)


def _cov(P):
    return np.cov(np.asarray(P, dtype=np.float64).T, bias=False)


def _points(rng, kind, k=10, origin=(0.0, 0.0, 0.0)):
    """Neighbourhoods of k points on 2^-10 m lattices (dyadic: np.cov's zeros are exact)."""
    U = 2.0 ** -10
    q = rng.integers(-2000, 2001, size=(k, 3))
    if kind.startswith("wall_"):                  # one coordinate constant
        q[:, "xyz".index(kind[-1])] = 17
    elif kind in ("line_x", "line_y", "line_z"):  # all but one coordinate constant
        a = "xyz".index(kind[-1])
        q[:, [b for b in range(3) if b != a]] = [5, -9]
    elif kind.startswith("line_diag_"):           # diagonal in a coordinate plane
        t = rng.integers(-2000, 2001, k)
        q = np.full((k, 3), 3)
        q[:, "xyz".index(kind[-2])] = t
        q[:, "xyz".index(kind[-1])] = -2 * t
    elif kind == "mirror_x":                      # (x, y, z) and (-x, y, z): c01 = c02 = 0
        h = q[: k // 2]
        q = np.concatenate((h, h * [-1, 1, 1]))
    elif kind == "mirror_y":
        h = q[: k // 2]
        q = np.concatenate((h, h * [1, -1, 1]))
    elif kind == "mirror_z":
        h = q[: k // 2]
        q = np.concatenate((h, h * [1, 1, -1]))
    elif kind == "square":                        # repeated in-plane eigenvalue, rank 2
        q = np.array([[1, 1, 0], [1, -1, 0], [-1, 1, 0], [-1, -1, 0]] * (k // 4)) * rng.integers(1, 500)
    elif kind == "cube":                          # 3-fold repeated
        q = np.array([[a, b, c] for a in (-1, 1) for b in (-1, 1) for c in (-1, 1)] * (k // 8)) * rng.integers(1, 500)
    elif kind == "octahedron":                    # 3-fold repeated
        q = np.concatenate((np.eye(3, dtype=np.int64), -np.eye(3, dtype=np.int64))) * rng.integers(1, 500)
    elif kind == "coincident":                    # rank 0
        q = np.tile(q[:1], (k, 1))
    return np.asarray(origin) + q * U


# (family, builder, hi, perm): the dgebal outcome the design must produce
_O_UTM = (612345.25, 5432109.875, 310.5)   # easting / northing / height; 2^-10 lattice exact there
FAMILIES = [
    ("row0_decoupled", lambda r: _spd(r, [(0, 1), (0, 2)]), 1, [0]),
    ("row1_decoupled", lambda r: _spd(r, [(0, 1), (1, 2)]), 1, [1]),
    ("row2_decoupled", lambda r: _spd(r, [(0, 2), (1, 2)]), 1, [2]),
    ("zero01", lambda r: _spd(r, [(0, 1)]), 2, []),
    ("zero02", lambda r: _spd(r, [(0, 2)]), 2, []),
    ("zero12", lambda r: _spd(r, [(1, 2)]), 2, []),
    ("diagonal", lambda r: _spd(r, [(0, 1), (0, 2), (1, 2)]), 0, [1, 2]),
    ("wall_x", lambda r: _cov(_points(r, "wall_x")), 1, [0]),
    ("wall_y", lambda r: _cov(_points(r, "wall_y")), 1, [1]),
    ("wall_z", lambda r: _cov(_points(r, "wall_z")), 1, [2]),
    ("wall_x_utm", lambda r: _cov(_points(r, "wall_x", 16, _O_UTM)), 1, [0]),
    ("wall_y_utm", lambda r: _cov(_points(r, "wall_y", 16, _O_UTM)), 1, [1]),
    ("wall_z_utm", lambda r: _cov(_points(r, "wall_z", 16, _O_UTM)), 1, [2]),
    ("mirror_x", lambda r: _cov(_points(r, "mirror_x", 16)), 1, [0]),
    ("mirror_y", lambda r: _cov(_points(r, "mirror_y", 16)), 1, [1]),
    ("mirror_z", lambda r: _cov(_points(r, "mirror_z", 16)), 1, [2]),
    ("line_x", lambda r: _cov(_points(r, "line_x")), 0, [1, 2]),
    ("line_y", lambda r: _cov(_points(r, "line_y")), 0, [1, 2]),
    ("line_z", lambda r: _cov(_points(r, "line_z")), 0, [1, 2]),
    ("line_diag_xy", lambda r: _cov(_points(r, "line_diag_xy")), 1, [2]),
    ("line_diag_xz", lambda r: _cov(_points(r, "line_diag_xz")), 1, [1]),
    ("line_diag_yz", lambda r: _cov(_points(r, "line_diag_yz")), 1, [0]),
    ("square", lambda r: _cov(_points(r, "square", 8)), 0, [1, 2]),
    ("cube", lambda r: _cov(_points(r, "cube", 8)), 0, [1, 2]),
    ("octahedron", lambda r: _cov(_points(r, "octahedron", 6)), 0, [1, 2]),
]
N_DESIGNED = 300


def _family(name):
    for f in FAMILIES:
        if f[0] == name:
            return f
    raise KeyError(name)


def _instances(name):
    _, build, _, _ = _family(name)
    rng = np.random.default_rng(sum(map(ord, name)))
    n = 4 if name in ("square", "cube", "octahedron") else N_DESIGNED
    return [build(rng) for _ in range(n)]


@pytest.mark.parametrize("name", [f[0] for f in FAMILIES])
def test_designed_covariances_take_the_intended_dgebal_permutation(name):
    """LAPACK's own dgebal on every instance: the designed permutation and block, unit scaling."""
    from scipy.linalg import lapack

    _, _, hi_want, perm_want = _family(name)
    for Cm in _instances(name):
        assert np.array_equal(Cm, Cm.T)
        _, lo, hi, ps, info = lapack.dgebal(Cm, permute=1, scale=1)
        assert info == 0 and lo == 0 and hi == hi_want, (name, lo, hi, Cm)
        assert (ps[lo:hi + 1] == 1.0).all(), (name, ps)                 # no scaling
        assert [int(p) - 1 for p in ps[hi + 1:]] == perm_want, (name, ps)


@pytest.mark.parametrize("name", [f[0] for f in FAMILIES])
def test_designed_covariances_match_numpy_eig(lib, name):
    """Eigenvalue slots and eigenvectors as np.linalg.eig returns them, and the float32 normal and
    planarity of eig3_smallest equal to the reference's bit for bit."""
    for i, Cm in enumerate(_instances(name)):
        w, v = np.linalg.eig(Cm)
        wr, vr = dgeev(lib, Cm)
        s = np.abs(Cm).max()
        np.testing.assert_allclose(wr, w, rtol=0, atol=1e-13 * s, err_msg=f"{name} #{i} slots")
        np.testing.assert_allclose(vr, v, rtol=0, atol=1e-12, err_msg=f"{name} #{i} vectors")
        n, pl = smallest(lib, Cm)
        n_ref, pl_ref = numpy_normal(Cm)
        assert same_f32(n, n_ref), f"{name} #{i}: normal {n} vs {n_ref}"
        assert same_f32(pl, pl_ref), f"{name} #{i}: planarity {pl} vs {pl_ref}"


def test_rank_zero_matches_numpy(lib):
    """All points coincide: covariance 0, NumPy's normal (1, 0, 0) (identity eigenvectors, ties
    in slot order) and planarity 0/0 = NaN."""
    rng = np.random.default_rng(1)
    for origin in ((0.0, 0.0, 0.0), _O_UTM):
        Cm = _cov(_points(rng, "coincident", 16, origin))
        assert (Cm == 0).all()
        n, pl = smallest(lib, Cm)
        n_ref, pl_ref = numpy_normal(Cm)
        assert same_f32(n, n_ref) and np.isnan(pl) and np.isnan(pl_ref), (n, n_ref, pl, pl_ref)


def test_smallest_eigenvector_modes(lib):
    rng = np.random.default_rng(0)
    for _ in range(200):
        B = rng.normal(size=(3, 3))
        Cm = B @ B.T
        c6 = np.array([Cm[0, 0], Cm[0, 1], Cm[0, 2], Cm[1, 1], Cm[1, 2], Cm[2, 2]])
        w_ref = np.sort(np.linalg.eigvalsh(Cm))[::-1]
        for mode in (0, 1):
            w = np.zeros(3)
            n = np.zeros(3)
            lib.eig3_smallest_host(c6.ctypes.data_as(C.c_void_p), C.c_int(mode),
                                   w.ctypes.data_as(C.c_void_p), n.ctypes.data_as(C.c_void_p))
            np.testing.assert_allclose(w, w_ref, rtol=1e-10, atol=1e-13 * w_ref[0])
            np.testing.assert_allclose(Cm @ n, w[2] * n, atol=1e-10 * w_ref[0])
            assert abs(np.linalg.norm(n) - 1) < 1e-12
            if mode == 1:
                assert n[np.argmax(np.abs(n))] > 0
    # degenerate neighbourhood -> planarity 0/0
    w = np.zeros(3)
    n = np.zeros(3)
    z6 = np.zeros(6)
    lib.eig3_smallest_host(z6.ctypes.data_as(C.c_void_p), C.c_int(0), w.ctypes.data_as(C.c_void_p),
                           n.ctypes.data_as(C.c_void_p))
    assert (w == 0).all() and np.isnan((w[1] - w[2]) / w[0])
