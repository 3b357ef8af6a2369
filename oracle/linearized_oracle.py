"""CPU oracle for the LINEARISED simpleICP variant: the C++ driver's algorithm (the Rust / Julia /
MATLAB ports share its structure; where they differ is listed below).

TEST INFRASTRUCTURE ONLY (same rule as simpleicp_oracle.py: only tests/, smoke() and bench.py's
CPU legs may import it; the product package never does).

What differs from the Python package's algorithm (SURVEY.md section 8f rank 3), with the C++
source lines each function follows (paths relative to /root/reference/c++/src/):

  * normals and planarity stay float64 (pointcloud.cpp:107-147; no float32 store);
  * rejection uses sigma = 1.4826 * MAD and the UPPER middle element as the median
    (corrpts.cpp:59-72, simpleicp.cpp:157-188: std::nth_element at size/2);
  * one linear least-squares solve A x = l per iteration (corrpts.cpp:113-156), the movable cloud
    is moved by dH = H(euler(x[0:3]), x[3:6]) and the printed residuals are A x - l;
  * sample standard deviation (n - 1) and a stop rule on the relative change of mean AND std of
    those residuals, checked from the second iteration on (simpleicp.cpp:64-80, 190-216);
  * no parameter uncertainties, no observed/fixed parameters.

Composition of the reported matrix: the C++ driver accumulates ``H_new = H_old * dH``
(simpleicp.cpp:66) while the Rust and MATLAB drivers accumulate ``dH * H`` (rust/src/icp.rs:164,
matlab/simpleicp.m:55).  Both are offered (``compose="post"`` is the C++ one); the cloud itself is
always moved by dH on the left, as all of them do.  Beyond the composition order the Rust, Julia
and MATLAB ports (a) build dH from the linearised matrix I + [x]_x instead of the Euler product
(rust/src/icp.rs:339-344, julia/simpleicp.jl:162-178, matlab/simpleicp.m:140-152) -- the
``rotation="small_angle"`` switch below -- and (b) average the two middle elements of an
even-sized sample in median / MAD (rust/src/icp.rs:392-409) where the C++ takes the upper one.
Neither the product's linearised variants nor the default settings of this file reproduce (a)
or (b): they follow the C++ sources, which is what can be compiled and pinned here.

Parity status: PINNED to the reference's own C++ sources, modulo their three third-party
libraries.  oracle/Makefile compiles the UNMODIFIED /root/reference/c++/src/{simpleicp,pointcloud,
corrpts,simpleicp-cli}.cpp where they lie into oracle/_ref/, against stand-in headers
(oracle/cpp_standin/) for Eigen, nanoflann and cxxopts -- none of which is in this image -- the way
oracle/lmfit_standin stands in for the Python package's lmfit.  oracle/make_golden_cpp.py runs the
reference CLI with the command lines of c++/run_simpleicp.sh (dragon, airborne, terrestrial, bunny)
plus two flag variations and stores screen output and a full-precision per-iteration dump in
tests/golden/cppref_*.npz; tests/test_cpp_reference_pin.py checks this restatement against them:
selection exact, normals / planarity 1e-9, and -- with the reference run's eigenvector signs handed
over -- every iteration's kept set exact, residual statistics, dH and H to 1e-11, the printed
table character by character; when /root/reference is present it also re-runs the recipe and
compares bit for bit.  What the stand-ins leave unpinned (stated in their headers): the
eigenvector SIGN convention (Eigen's SelfAdjointEigenSolver there, a Jacobi sweep in the stand-in,
LAPACK dsyevd through numpy.linalg.eigh here -- the solution is invariant to it, the sign of
individual residuals, and through the median the rejection path, is not), the pick among
EQUIDISTANT neighbours, last-ulp summation order, and nanoflann >= 1.5's reading of the
reference's ``SearchParameters(10)`` as eps = 10 (an approximate search whose misses depend on
nanoflann's own tree; every other port of the reference searches exactly, and so do the stand-in
and this file).

The older golden vector, the C++ screen output for the Dragon pair printed in
/root/reference/README.md:141-160 (iteration table to 4 decimals, H to 6 decimals), is kept in
tests/golden/cpp_readme_dragon.json and checked by tests/test_linearized_oracle.py under
``rotation="small_angle"``: that output predates the current sources (see
``simpleicp_linearized``).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Optional

import numpy as np
from scipy import spatial


def euler_angles_to_rotation_matrix(a1: float, a2: float, a3: float) -> np.ndarray:
    """corrpts.cpp:92-111 -- the same R = Rx Ry Rz element formulas as the Python package."""
    c1, s1 = np.cos(a1), np.sin(a1)
    c2, s2 = np.cos(a2), np.sin(a2)
    c3, s3 = np.cos(a3), np.sin(a3)
    return np.array(
        [
            [c2 * c3, -c2 * s3, s2],
            [c1 * s3 + s1 * s2 * c3, c1 * c3 - s1 * s2 * s3, -s1 * c2],
            [s1 * s3 - c1 * s2 * c3, s1 * c3 + c1 * s2 * s3, c1 * c2],
        ]
    )


def select_in_range(X_fix: np.ndarray, X_mov: np.ndarray, max_range: float, workers: int = -1) -> np.ndarray:
    """pointcloud.cpp:33-76 -- keep fixed points whose nearest movable point is within range
    (deselect when dist > max_range, i.e. keep dist <= max_range).  `workers` only splits the
    exact query over threads (1 for small clouds, where starting threads costs more than it saves)."""
    d, _ = spatial.cKDTree(X_mov).query(X_fix, k=1, workers=workers)
    return np.flatnonzero(d <= max_range)


def select_n_points(idx_sel: np.ndarray, n: int) -> np.ndarray:
    """pointcloud.cpp:78-98 -- LinSpaced(n, 0, m-1), C round() (half away from zero)."""
    m = idx_sel.shape[0]
    if n >= m:
        return idx_sel
    lin = np.linspace(0.0, float(m - 1), n)
    picks = np.floor(lin + 0.5).astype(np.int64)
    return idx_sel[np.unique(picks)]


def estimate_normals(X: np.ndarray, idx_sel: np.ndarray, neighbors: int):
    """pointcloud.cpp:100-147 -- k-NN covariance (n-1), eigenvector of the smallest eigenvalue,
    planarity (l1 - l0) / l2 with ascending eigenvalues; everything float64."""
    _, nn = spatial.cKDTree(X).query(X[idx_sel], k=neighbors, workers=-1)
    P = X[nn]  # (K, k, 3)
    c = P - P.mean(axis=1, keepdims=True)
    C = np.einsum("kni,knj->kij", c, c) / float(neighbors - 1)
    w, v = np.linalg.eigh(C)
    normals = v[:, :, 0].copy()
    planarity = (w[:, 1] - w[:, 0]) / w[:, 2]
    return normals, planarity


def median_upper(v: np.ndarray) -> float:
    """simpleicp.cpp:157-171 -- nth_element at size/2: the upper of the two middle elements."""
    return float(np.partition(v, v.shape[0] // 2)[v.shape[0] // 2])


def mad_upper(v: np.ndarray) -> float:
    """simpleicp.cpp:173-182."""
    return median_upper(np.abs(v - median_upper(v)))


def sample_std(v: np.ndarray) -> float:
    """simpleicp.cpp:184-188."""
    return float(np.sqrt(np.sum((v - v.mean()) ** 2) / (v.shape[0] - 1)))


def change(new: float, old: float) -> float:
    """simpleicp.cpp:190-197."""
    if old == 0.0:
        return 0.0 if new == 0.0 else float("inf")
    return abs((new - old) / old * 100.0)


@dataclass
class LinIteration:
    n_kept: int = 0
    mean: float = 0.0
    std: float = 0.0
    x: Optional[np.ndarray] = None  # the six increments of this iteration
    idx_mov: Optional[np.ndarray] = None
    dists: Optional[np.ndarray] = None
    keep: Optional[np.ndarray] = None
    T_before: Optional[np.ndarray] = None  # cumulative cloud transform the iteration started from
    idx_mov_own: Optional[np.ndarray] = None  # cKDTree's pick when ``matches`` forced another one


@dataclass
class LinResult:
    H: np.ndarray = field(default_factory=lambda: np.eye(4))  # reported matrix (compose rule)
    T: np.ndarray = field(default_factory=lambda: np.eye(4))  # transform actually applied to the cloud
    orig: Optional[LinIteration] = None
    iterations: List[LinIteration] = field(default_factory=list)
    converged: bool = False
    idx_fix: Optional[np.ndarray] = None
    normals: Optional[np.ndarray] = None
    planarity: Optional[np.ndarray] = None


def simpleicp_linearized(
    X_fix: np.ndarray,
    X_mov: np.ndarray,
    correspondences: int = 1000,
    neighbors: int = 10,
    min_planarity: float = 0.3,
    max_overlap_distance: float = np.inf,
    min_change: float = 1.0,
    max_iterations: int = 100,
    compose: str = "post",
    normals: Optional[np.ndarray] = None,
    planarity: Optional[np.ndarray] = None,
    keep_arrays: bool = False,
    rotation: str = "euler",
    matches=None,
) -> LinResult:
    """simpleicp.cpp:8-129 (driver) with corrpts.cpp:6-156 inlined.  ``normals``/``planarity``
    (per selected fixed point) replace the estimation, for lock-step comparisons.

    ``rotation="small_angle"`` builds dH with R = I + [alpha]x instead of the Euler product.  The
    current C++ sources use the Euler product (corrpts.cpp:92-111, 148-151), but the screen output
    printed in README.md:141-160 -- the only golden vector the reference holds for this variant --
    shows a matrix whose rows are not unit length (|row 0|^2 = 1.0013) and a residual std that
    floors at 0.0022 on noise-free data: it was produced by an earlier revision with the
    small-angle matrix.  With this switch the restatement reproduces that output (see
    tests/test_linearized_oracle.py); without it, it follows the sources as they are.

    ``matches`` (a sequence of index arrays, one per iteration) replaces the nearest-neighbour
    pick of that iteration: which of several EQUIDISTANT movable points a k-d tree returns is
    unspecified (mm-quantised scans tie in a few per cent of the queries), so a lock-step
    comparison hands over the other side's picks -- after checking that they are nearest
    neighbours too (tests/test_cpp_reference_pin.py) -- the way ``normals`` hands over its
    eigenvector signs."""
    X_fix = np.ascontiguousarray(X_fix, dtype=np.float64)
    X_mov0 = np.ascontiguousarray(X_mov, dtype=np.float64)
    res = LinResult()

    idx = np.arange(X_fix.shape[0])
    # the C++ CLI passes -1 for "no overlap filter" (simpleicp-cli.cpp:27); inf means the same here
    if np.isfinite(max_overlap_distance) and max_overlap_distance > 0:
        idx = select_in_range(X_fix, X_mov0, max_overlap_distance)
        if idx.size == 0:
            raise RuntimeError("Point clouds do not overlap within max_overlap_distance")
    idx = select_n_points(idx, correspondences)
    if normals is None:
        normals, planarity = estimate_normals(X_fix, idx, neighbors)
    res.idx_fix, res.normals, res.planarity = idx, normals, planarity
    P1 = X_fix[idx]

    T = np.eye(4)
    H = np.eye(4)
    X = X_mov0.copy()
    means: List[float] = []
    stds: List[float] = []
    for i in range(max_iterations):
        # corrpts.cpp:6-57 -- match in the MOVED cloud, signed distance along the fixed normal
        _, nn = spatial.cKDTree(X).query(P1, k=1, workers=-1)
        nn_own = nn
        if matches is not None and i < len(matches):
            nn = np.asarray(matches[i], dtype=np.int64)
        P2 = X[nn]
        d = np.einsum("ij,ij->i", P2 - P1, normals)
        # corrpts.cpp:59-90
        med = median_upper(d)
        sig = 1.4826 * mad_upper(d)
        keep = ~((np.abs(d - med) > 3.0 * sig) | (planarity < min_planarity))
        p1, p2, n = P1[keep], P2[keep], normals[keep]
        if i == 0:
            dk = d[keep]
            res.orig = LinIteration(int(keep.sum()), float(dk.mean()), sample_std(dk))
        # corrpts.cpp:113-156
        A = np.empty((p1.shape[0], 6))
        A[:, 0] = -p2[:, 2] * n[:, 1] + p2[:, 1] * n[:, 2]
        A[:, 1] = p2[:, 2] * n[:, 0] - p2[:, 0] * n[:, 2]
        A[:, 2] = -p2[:, 1] * n[:, 0] + p2[:, 0] * n[:, 1]
        A[:, 3:6] = n
        l = np.einsum("ij,ij->i", n, p1 - p2)
        x = np.linalg.lstsq(A, l, rcond=None)[0]
        dH = np.eye(4)
        if rotation == "small_angle":
            dH[:3, :3] = np.array([[1.0, -x[2], x[1]], [x[2], 1.0, -x[0]], [-x[1], x[0], 1.0]])
        else:
            dH[:3, :3] = euler_angles_to_rotation_matrix(x[0], x[1], x[2])
        dH[:3, 3] = x[3:6]
        r = A @ x - l

        it = LinIteration(int(keep.sum()), float(r.mean()), sample_std(r), x=x)
        if keep_arrays:
            it.idx_mov, it.dists, it.keep, it.T_before, it.idx_mov_own = nn, d, keep, T.copy(), nn_own
        # simpleicp.cpp:62-80
        X = X @ dH[:3, :3].T + dH[:3, 3]
        T = dH @ T
        H = H @ dH if compose == "post" else dH @ H
        means.append(it.mean)
        stds.append(it.std)
        res.iterations.append(it)
        if i > 0 and change(means[-1], means[-2]) < min_change and change(stds[-1], stds[-2]) < min_change:
            res.converged = True
            break
    res.H, res.T = H, T
    return res


def format_table(res: LinResult) -> str:
    """simpleicp.cpp:82-101 -- the rows the C++ driver prints (the converging iteration is not
    printed: the break comes first)."""
    rows = ["%9s | %15s | %15s | %15s" % ("Iteration", "correspondences", "mean(residuals)", "std(residuals)")]
    rows.append("%9s | %15d | %15.4f | %15.4f" % ("orig:0", res.orig.n_kept, res.orig.mean, res.orig.std))
    its = res.iterations[:-1] if res.converged else res.iterations
    for k, it in enumerate(its):
        rows.append("%9d | %15d | %15.4f | %15.4f" % (k + 1, it.n_kept, it.mean, it.std))
    return "\n".join(rows)
