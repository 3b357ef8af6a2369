"""SimpleICP facade: the reference's driver API (python/simpleicp/simpleicp.py:41-380) on top of
the H100 library, plus the functional form ``simpleicp(X_fix, X_mov, **kwargs)`` (shape of
julia/simpleicp.jl:216-222 and python/simpleicp/tests/test_simpleicp.py:18-32).

What runs where
  host (this file) : argument checks, degree->radian, linspace subsampling, logging, exceptions
  GPU (libsicp_b200): overlap filter, normals, every iteration of match / reject / solve, the
                      stop rule, parameter sigmas, the final transform
The whole iteration loop is one C call (sicp_run); nothing is transferred per iteration except a
176-byte record.
"""
from __future__ import annotations

import logging
import time
from dataclasses import fields
from pathlib import Path
from typing import Optional, Sequence, Tuple

import numpy as np

from . import _capi, mathutils, optimization, pointcloud

_log = logging.getLogger(__name__)
_NORMAL_COLUMNS = ("nx", "ny", "nz", "planarity")


class SimpleICPException(Exception):
    """Raised when SimpleICP is misused or cannot proceed (reference: simpleicp.py:382)."""


def _enable_verbose_logging() -> None:
    """Attach (once) a stdout handler to the package logger, like the reference's verbose=True."""
    pkg_log = logging.getLogger(__package__)
    pkg_log.setLevel(logging.INFO)
    for h in pkg_log.handlers:
        if getattr(h, "_simpleicp_verbose", False):
            return
    handler = logging.StreamHandler()
    handler.setFormatter(logging.Formatter("%(message)s"))
    handler._simpleicp_verbose = True
    pkg_log.addHandler(handler)


def _check_arguments(distance_weights, rbp_observed_values, rbp_observation_weights) -> None:
    """Same checks and messages as the reference (simpleicp.py:326-353)."""
    if distance_weights is not None and distance_weights <= 0:
        raise SimpleICPException("distance_weights must be > 0.")
    if len(rbp_observed_values) != 6:
        raise SimpleICPException("rbp_observed_values must have exactly 6 elements.")
    if len(rbp_observation_weights) != 6:
        raise SimpleICPException("rbp_observation_weights must have exactly 6 elements.")
    if not all(w >= 0 for w in rbp_observation_weights):
        raise SimpleICPException("All elements of rbp_observation_weights must be >= 0.")
    if not any(np.isfinite(rbp_observation_weights)):
        raise SimpleICPException("At least one element in rbp_observation_weights must be finite.")


def _check_mov_arguments(mov_neighbors, max_angle_between_normals, mov_normals=None, n_mov=None) -> None:
    """The movable-side keywords: ``mov_neighbors`` (k of pc_mov.estimate_normals(k)) in [2, 64] and
    at most the movable point count, not together with ``mov_normals``; ``max_angle_between_normals``
    within [0, 90] degrees and only with movable normals."""
    if mov_neighbors is not None:
        if mov_normals is not None:
            raise SimpleICPException("Give either mov_normals or mov_neighbors, not both.")
        if isinstance(mov_neighbors, bool) or int(mov_neighbors) != mov_neighbors or not 2 <= int(mov_neighbors) <= 64:
            raise SimpleICPException("mov_neighbors must be an integer within [2, 64].")
        if n_mov is not None and int(mov_neighbors) > n_mov:
            raise SimpleICPException("mov_neighbors exceeds the number of points in the movable point cloud.")
    if max_angle_between_normals is not None:
        if mov_normals is None and mov_neighbors is None:
            raise SimpleICPException(
                "max_angle_between_normals needs the normals of the movable point cloud "
                "(mov_neighbors=k, PointCloud.estimate_normals on pc_mov, or mov_normals=...)."
            )
        if not 0.0 <= float(max_angle_between_normals) <= 90.0:
            raise SimpleICPException("max_angle_between_normals must be within [0, 90] degrees.")


def _observed_in_radians(rbp_observed_values) -> np.ndarray:
    # The reference converts in place inside np.array(rbp_observed_values) (simpleicp.py:146-148),
    # i.e. an all-integer tuple stays an integer array; kept for drop-in behaviour.
    obs = np.array(rbp_observed_values)
    for i in range(3):
        obs[i] = obs[i] * np.pi / 180
    return obs


def _change(new: float, old: float) -> float:
    if old == 0:
        return 0.0 if new == 0 else np.inf
    return np.abs((new - old) / old * 100)


# One engine (CUDA context state, stream, ~250 MB of device buffers at 1M-point clouds) per
# (device, thread) is kept for calls that do not bring their own: creating and destroying it per
# call costs more than a small registration.  Engines are not thread-safe, hence the thread key.
_DEFAULT_ENGINES: dict = {}


def default_engine(device: Optional[int] = None) -> _capi.Engine:
    import threading

    if device is None:
        device = _capi.current_device()
    key = (int(device), threading.get_ident())
    eng = _DEFAULT_ENGINES.get(key)
    if eng is None or not eng.alive:
        eng = _capi.Engine(int(device))
        _DEFAULT_ENGINES[key] = eng
    else:
        eng.reset_options()
    return eng


def close_default_engines() -> None:
    """Release the engines kept for register()/simpleicp()/SimpleICP.run calls without `engine=`."""
    for eng in list(_DEFAULT_ENGINES.values()):
        eng.close()
    _DEFAULT_ENGINES.clear()


import atexit as _atexit  # noqa: E402

_atexit.register(close_default_engines)


def _host_xyz(X) -> np.ndarray:
    """Host float64 view of a cloud given as NumPy array or (CUDA) torch tensor."""
    if hasattr(X, "detach"):
        X = X.detach().cpu().numpy()
    return np.asarray(X, dtype=np.float64)


class _Result:
    """Everything one registration produces."""

    __slots__ = ("H", "X_mov_transformed", "rbp", "residuals", "_idx", "normals",
                 "records", "iterations", "converged", "timings", "loop_ms", "initial_stats")

    @property
    def idx_selected(self):
        """Indices of the selected fixed points (computed on first use after a fused run)."""
        if callable(self._idx):
            self._idx = self._idx()
        return self._idx

    @idx_selected.setter
    def idx_selected(self, v):
        self._idx = v


def _wrap_error(e: _capi.SicpError, max_overlap_distance: float):
    if e.code == _capi.SICP_ERR_NO_OVERLAP:
        return SimpleICPException(
            "Point clouds do not overlap within max_overlap_distance = "
            f"{max_overlap_distance:.5f}! Consider increasing the value of max_overlap_distance."
        )
    if e.code in (_capi.SICP_ERR_TOO_FEW_CORR, _capi.SICP_ERR_BAD_ARG, _capi.SICP_ERR_SINGULAR):
        return SimpleICPException(e.message)
    return e


def register(
    X_fix,
    X_mov,
    *,
    correspondences: int = 1000,
    neighbors: int = 10,
    min_planarity: float = 0.3,
    max_overlap_distance: float = np.inf,
    min_change: float = 1.0,
    max_iterations: int = 100,
    distance_weights: Optional[float] = 1,
    rbp_observed_values: Sequence[float] = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
    rbp_observation_weights: Sequence[float] = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
    debug_dirpath: str = "",
    idx_selected: Optional[np.ndarray] = None,
    normals: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]] = None,
    engine: Optional[_capi.Engine] = None,
    transform_out=None,
    stepwise: bool = False,
    on_normals=None,
    want_normals: bool = True,
    mov_normals: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]] = None,
    max_angle_between_normals: Optional[float] = None,
    mov_neighbors: Optional[int] = None,
) -> _Result:
    """Core of both front ends: one registration on one GPU.

    ``idx_selected`` restricts the candidate fixed points (the reference's ``selected`` column),
    ``normals=(nx, ny, nz, planarity)`` are full-length (n_fix) arrays supplied instead of being
    estimated (the reference's pre-computed-columns hook, simpleicp.py:176-178).

    ``mov_normals=(nx, ny, nz, planarity)``: full-length (n_mov) attributes of the movable cloud
    in its own frame, NaN where not estimated.  With them a correspondence must also pass
    ``min_planarity`` on the movable side — what the reference does when ``pc_mov`` carries a
    planarity column (corrpts.py:157-162).  ``max_angle_between_normals`` (degrees, needs
    ``mov_normals``) additionally drops correspondences whose normals differ by more than that
    angle after the distance rejection: the reference declares this step
    (``reject_wrt_to_angle_between_normals``, simpleicp.py:207) but leaves it unimplemented.

    ``mov_neighbors=k`` has the effect of ``pc_mov.estimate_normals(k)`` before the run: the
    movable attributes are estimated from k neighbours (inside the one library call when the
    registration is fused, through ``PointCloud.estimate_normals``'s code otherwise).
    """
    _check_arguments(distance_weights, rbp_observed_values, rbp_observation_weights)
    _check_mov_arguments(mov_neighbors, max_angle_between_normals, mov_normals, int(np.shape(X_mov)[0]))
    if debug_dirpath:
        _log.info(f'Write debug files to directory "{debug_dirpath}"')
        Path(debug_dirpath).mkdir(parents=True, exist_ok=True)
        stepwise = True
    obs = _observed_in_radians(rbp_observed_values)
    w_obs = [float(w) for w in rbp_observation_weights]
    H0 = mathutils.create_homogeneous_transformation_matrix(
        mathutils.euler_angles_to_rotation_matrix(obs[0], obs[1], obs[2]), obs[3:]
    )
    eng = engine if engine is not None else default_engine()
    fused = (idx_selected is None and normals is None and not stepwise and on_normals is None
             and not want_normals and mov_normals is None)
    try:  # noqa: PLR1702
        if fused:
            # the whole of SimpleICP.run as one library call: nothing but the clouds goes in,
            # nothing but the results comes back (simpleicp_b200/_capi.py::register_fused)
            return _register_fused(eng, X_fix, X_mov, correspondences, neighbors, min_planarity,
                                   max_overlap_distance, min_change, max_iterations, distance_weights,
                                   obs, w_obs, rbp_observation_weights, transform_out, mov_neighbors,
                                   max_angle_between_normals)
        if mov_neighbors is not None:
            mov_normals = pointcloud.estimate_normals_of(X_mov, None, int(mov_neighbors))
        eng.set_clouds(X_fix, X_mov)
        n_fix = eng.n_fix
        if mov_normals is not None:
            eng.set_mov_normals(*mov_normals, max_angle_deg=max_angle_between_normals)
        idx = None if idx_selected is None else np.asarray(idx_selected, dtype=np.int64)

        if np.isfinite(max_overlap_distance):
            _log.info("Consider partial overlap of point clouds ...")
            eng.set_selected(idx)
            try:
                keep = eng.select_in_range(H0, max_overlap_distance)
            except _capi.SicpError as e:
                raise _wrap_error(e, max_overlap_distance) from None
            idx = (np.arange(n_fix, dtype=np.int64) if idx is None else idx)[keep]

        _log.info("Select points for correspondences in fixed point cloud ...")
        m = n_fix if idx is None else idx.size
        if m > correspondences:
            # rint(linspace(0, m-1, n)) with m > n has a step > 1, so the picks are strictly
            # increasing: already the sorted, duplicate-free index set the reference ends up with
            pick = pointcloud.subsample_indices(m, correspondences)
            idx = (pick if idx is None else idx[pick]).astype(np.int64)
        eng.set_selected(idx)
        if idx is None:
            idx = np.arange(n_fix, dtype=np.int64)

        if normals is None:
            _log.info("Estimate normals of selected points ...")
            # the normals stay on the device for the loop; they are only downloaded when someone
            # wants to look at them (the class facade stores them as columns of pc_fix)
            nrm = eng.estimate_normals(neighbors, download=want_normals or on_normals is not None)
        else:
            nrm = tuple(np.asarray(a, dtype=np.float32)[idx] for a in normals)
            eng.set_normals(*nrm)
        if on_normals is not None:
            on_normals(idx, nrm)

        _log.info("Start iterations ...")
        lsq = eng.lsq_params(obs, obs, w_obs, distance_weights)
        params = eng.run_params(min_planarity, min_change, max_iterations, lsq)
        try:
            if stepwise:
                out = _loop_stepwise(eng, params, obs, w_obs, distance_weights, min_planarity,
                                     min_change, max_iterations, debug_dirpath, X_fix, X_mov, idx)
            else:
                out = _loop_fused(eng, params)
        except _capi.SicpError as e:
            raise _wrap_error(e, max_overlap_distance) from None
        x, sigma, H, residuals, records, iterations, converged, loop_ms = out

        rbp = _make_rbp(obs, rbp_observation_weights, records, iterations, x, sigma)

        _log_run(records, iterations, converged, H, rbp)

        X_t = eng.transform(H, out=transform_out)
        if debug_dirpath:
            _capi.write_xyz(Path(debug_dirpath).joinpath(f"iteration{iterations - 1:03d}_postoptim_pcmov.xyz"),
                            _host_xyz(X_t))
        r = _Result()
        r.H, r.X_mov_transformed, r.rbp, r.residuals = H, X_t, rbp, residuals
        r.idx_selected, r.normals, r.records = idx, nrm, records
        r.iterations, r.converged, r.loop_ms = iterations, converged, loop_ms
        r.timings = eng.timings()
        return r
    except _capi.SicpError as e:
        if e.code == _capi.SICP_ERR_CUDA and engine is None:
            eng.close()  # do not keep a context whose device state is unknown
        raise


def _records(log):
    return [
        dict(n_kept=int(r.n_kept), median=r.median, mad=r.mad, mean_dist=r.mean_dist,
             std_dist=r.std_dist, x=np.array(r.x), mean_res=r.mean_res, std_res=r.std_res,
             distance_weight=r.distance_weight, lm_iterations=int(r.lm_iterations),
             n_bruteforce=int(r.n_bruteforce))
        for r in log
    ]


def _loop_fused(eng: _capi.Engine, params):
    out, log, residuals = eng.run(params)
    H = np.array(out.H).reshape(4, 4)
    return (np.array(out.x), np.array(out.sigma), H, residuals, _records(log), int(out.iterations),
            bool(out.converged), float(out.loop_ms))


def _make_rbp(obs, rbp_observation_weights, records, iterations, x, sigma):
    rbp = optimization.RigidBodyParameters()
    rbp.set_parameter_attributes_from_list(
        "initial_value", list(obs) if iterations <= 1 else list(records[iterations - 2]["x"])
    )
    rbp.set_parameter_attributes_from_list("observed_value", list(obs))
    rbp.set_parameter_attributes_from_list("observation_weight", list(rbp_observation_weights))
    rbp.set_parameter_attributes_from_list("estimated_value", [float(v) for v in x])
    rbp.set_parameter_attributes_from_list("estimated_uncertainty", [float(v) for v in sigma])
    return rbp


def _register_fused(eng, X_fix, X_mov, correspondences, neighbors, min_planarity, max_overlap_distance,
                    min_change, max_iterations, distance_weights, obs, w_obs, rbp_observation_weights,
                    transform_out, mov_neighbors=None, max_angle_between_normals=None) -> _Result:
    for msg in ("Consider partial overlap of point clouds ..." if np.isfinite(max_overlap_distance) else None,
                "Select points for correspondences in fixed point cloud ...",
                "Estimate normals of selected points ...", "Start iterations ..."):
        if msg:
            _log.info(msg)
    lsq = eng.lsq_params(obs, obs, w_obs, distance_weights)
    params = eng.run_params(min_planarity, min_change, max_iterations, lsq)
    try:
        out, log, residuals, X_t = eng.register_fused(
            X_fix, X_mov, correspondences, neighbors,
            max_overlap_distance if np.isfinite(max_overlap_distance) else -1.0, params, transform_out,
            0 if mov_neighbors is None else int(mov_neighbors),
            -1.0 if max_angle_between_normals is None else float(np.deg2rad(max_angle_between_normals)))
    except _capi.SicpError as e:
        raise _wrap_error(e, max_overlap_distance) from None
    records, iterations = _records(log), int(out.iterations)
    H = np.array(out.H).reshape(4, 4)
    rbp = _make_rbp(obs, rbp_observation_weights, records, iterations, np.array(out.x), np.array(out.sigma))
    _log_run(records, iterations, bool(out.converged), H, rbp)
    r = _Result()
    r.H, r.X_mov_transformed, r.rbp, r.residuals = H, X_t, rbp, residuals
    if np.isfinite(max_overlap_distance):
        r.idx_selected = eng.select_n_points(eng.K)  # no-op on the selection, downloads it
    else:
        n_fix, K = eng.n_fix, eng.K
        r.idx_selected = lambda: (pointcloud.subsample_indices(n_fix, K).astype(np.int64) if K < n_fix
                                  else np.arange(n_fix, dtype=np.int64))
    r.normals, r.records = None, records
    r.iterations, r.converged, r.loop_ms = iterations, bool(out.converged), float(out.loop_ms)
    r.timings = eng.timings()
    return r


def _loop_stepwise(eng, params, obs, w_obs, distance_weights, min_planarity, min_change,
                   max_iterations, debug_dirpath, X_fix, X_mov, idx):
    """The same loop driven stage by stage through sicp_match / sicp_reject / sicp_solve; used
    for debug dumps (reference: simpleicp.py:141-143, 189-200, 216-221) and by the tests to check
    the fused loop against its parts."""
    x = np.array(obs, dtype=float)
    H = mathutils.create_homogeneous_transformation_matrix(
        mathutils.euler_angles_to_rotation_matrix(x[0], x[1], x[2]), x[3:]
    )
    records, residuals, prev = [], None, None
    w = distance_weights
    converged = False
    t0 = time.perf_counter()
    it = -1
    dbg = _DebugWriter(debug_dirpath, X_fix, X_mov, idx) if debug_dirpath else None
    for it in range(max_iterations):
        if dbg:
            dbg.preoptim_clouds(eng, it, H)
        pc2_idx, d = eng.match(H)
        keep, n_kept, st = eng.reject(min_planarity)
        if dbg and n_kept >= 6:  # the reference raises before writing (simpleicp.py:209-221)
            dbg.correspondences(it, pc2_idx, d, keep)
        x, H, residuals, rs, w_used = eng.solve(x, obs, w_obs, w, n_kept)
        if w is None:
            w = w_used  # frozen after iteration 0 (simpleicp.py:229-234)
        records.append(dict(n_kept=n_kept, median=st[0], mad=st[1], mean_dist=st[2], std_dist=st[3],
                            x=x.copy(), mean_res=rs[0], std_res=rs[1], distance_weight=w_used,
                            lm_iterations=-1, n_bruteforce=-1))
        if prev is not None:
            if _change(rs[0], prev[0]) < min_change and _change(rs[1], prev[1]) < min_change:
                converged = True
                break
        prev = rs
    sigma = eng.uncertainties()
    return x, sigma, H, residuals, records, it + 1, converged, (time.perf_counter() - t0) * 1e3


class _DebugWriter:
    """The reference's per-iteration debug files (simpleicp.py:189-221, corrpts.py:213-237,
    pointcloud.py:219-226).  The movable cloud is transformed ONCE per iteration (the file
    contains all of it); the correspondence dump takes its movable coordinates from the
    caller's UNTRANSFORMED cloud — the reference writes it after pc2.transform_by_H(inv(H))."""

    def __init__(self, dirpath, X_fix, X_mov, idx):
        self.dir = Path(dirpath)
        self.X_fix = _host_xyz(X_fix)
        self.X_mov = _host_xyz(X_mov)
        self.idx = idx

    def preoptim_clouds(self, eng, it, H):
        if it == 0:
            _capi.write_xyz(self.dir.joinpath(f"iteration{it:03d}_preoptim_pcfix.xyz"), self.X_fix)
        _capi.write_xyz(self.dir.joinpath(f"iteration{it:03d}_preoptim_pcmov.xyz"),
                        np.asarray(eng.transform(H)))

    def correspondences(self, it, pc2_idx, dist, keep):
        P1 = self.X_fix[self.idx[keep]]
        P2 = self.X_mov[pc2_idx[keep]]
        np.savetxt(self.dir.joinpath(f"iteration{it:03d}_preoptim_correspondences.xyz"),
                   np.column_stack((P1, P2, dist[keep])), delimiter=" ",
                   header="X1 Y1 Z1 X2 Y2 Z2 point_to_plane_distance", comments="//")


def _log_run(records, iterations, converged, H, rbp) -> None:
    """The reference's log lines (simpleicp.py:263-313).  On convergence the reference breaks
    before printing the converged iteration's row."""
    n_rows = iterations - 1 if converged else iterations
    for it in range(n_rows):
        r = records[it]
        if it == 0:
            _log.info(f"{'Iteration':>9s} | {'correspondences':>15s} | {'mean(residuals)':>15s} | "
                      f"{'std(residuals)':>15s}")
            _log.info(f"{'orig:0':>9s} | {r['n_kept']:15d} | {r['mean_dist']:15.4f} | "
                      f"{r['std_dist']:15.4f}")
        _log.info(f"{it + 1:9d} | {r['n_kept']:15d} | {r['mean_res']:15.4f} | {r['std_res']:15.4f}")
    if converged:
        _log.info("Convergence criteria fulfilled -> stop iteration!")
    _log.info("Estimated transformation matrix H:")
    for i in range(4):
        _log.info(f"[{H[i, 0]:12.6f} {H[i, 1]:12.6f} {H[i, 2]:12.6f} {H[i, 3]:12.6f}]")
    _log.info("... which corresponds to the following rigid-body transformation parameters:")
    _log.info(f"{'parameter':>9s} | {'est.value':>15s} | {'est.uncertainty':>15s} | "
              f"{'obs.value':>15s} | {'obs.weight':>15s}")
    for parameter in fields(rbp):
        p = getattr(rbp, parameter.name)
        _log.info(f"{parameter.name:>9s} | {p.estimated_value_scaled:15.6f} | "
                  f"{p.estimated_uncertainty_scaled:15.6f} | {p.observed_value_scaled:15.6f} | "
                  f"{p.observation_weight:15.3e}")
    _log.info("(Unit of est.value, est.uncertainty, and obs.value for alpha1/2/3 is degree)")


class SimpleICP:
    """Set up and run simpleICP (same surface as the reference class, simpleicp.py:41-324)."""

    def __init__(self, verbose: bool = True) -> None:
        self.pc1 = None
        self.pc2 = None
        if verbose:
            _enable_verbose_logging()

    def add_point_clouds(self, pc_fix: pointcloud.PointCloud, pc_mov: pointcloud.PointCloud) -> None:
        """pc_fix stays, pc_mov is moved (transformed in place by run)."""
        self.pc1 = pc_fix
        self.pc2 = pc_mov

    def run(
        self,
        correspondences: int = 1000,
        neighbors: int = 10,
        min_planarity: float = 0.3,
        max_overlap_distance: float = np.inf,
        min_change: float = 1.0,
        max_iterations: int = 100,
        distance_weights: Optional[float] = 1,
        rbp_observed_values: Tuple[float] = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
        rbp_observation_weights: Tuple[float] = (0.0, 0.0, 0.0, 0.0, 0.0, 0.0),
        debug_dirpath: str = "",
        max_angle_between_normals: Optional[float] = None,
    ) -> Tuple[np.ndarray, np.ndarray, optimization.RigidBodyParameters, np.ndarray]:
        """Run the registration.  Arguments, units (degrees for the observed angles), return
        tuple ``(H, X_mov_transformed, rbp, distance_residuals)`` and side effects (pc_mov
        transformed in place; pc_fix gains nx, ny, nz, planarity and a thinned ``selected``
        column) are those of the reference's ``SimpleICP.run``.

        If ``pc_mov`` carries normal columns (``pc_mov.estimate_normals(k)`` was called before),
        correspondences are also rejected by the planarity of the movable point, as in the
        reference (corrpts.py:157-162).  ``max_angle_between_normals`` (degrees; one keyword more
        than the reference, default off) enables the rejection step the reference only declares
        (``CorrPts.reject_wrt_to_angle_between_normals``)."""
        start_time = time.time()
        pc1, pc2 = self.pc1, self.pc2
        sel = pc1["selected"].to_numpy(dtype=bool)
        idx0 = None if sel.all() else np.flatnonzero(sel)
        have = set(_NORMAL_COLUMNS).issubset(pc1.columns)
        normals = tuple(np.asarray(pc1[c].to_numpy(), dtype=np.float32) for c in _NORMAL_COLUMNS) if have else None

        def store_normals(idx, nrm):
            if not have:
                pc1.set_normals(idx, *nrm)

        # the reference matches against the SELECTED movable points only (corrpts.py:131-135);
        # the final transform moves all of them (simpleicp.py:316)
        X2 = pc2.X
        sel2 = pc2["selected"].to_numpy(dtype=bool)
        X2_search = X2 if sel2.all() else np.ascontiguousarray(X2[sel2])
        mov_normals = None
        if "planarity" in pc2.columns:
            cols = [c if c in pc2.columns else None for c in _NORMAL_COLUMNS]
            mov_normals = tuple(
                (np.asarray(pc2[c].to_numpy(), dtype=np.float32) if c is not None
                 else np.full(len(sel2), np.nan, dtype=np.float32))[sel2] for c in cols)

        res = register(
            pc1.X, X2_search, correspondences=correspondences, neighbors=neighbors,
            min_planarity=min_planarity, max_overlap_distance=max_overlap_distance,
            min_change=min_change, max_iterations=max_iterations, distance_weights=distance_weights,
            rbp_observed_values=rbp_observed_values, rbp_observation_weights=rbp_observation_weights,
            debug_dirpath=debug_dirpath, idx_selected=idx0, normals=normals, on_normals=store_normals,
            mov_normals=mov_normals, max_angle_between_normals=max_angle_between_normals,
        )
        pc1.idx_selected = res.idx_selected
        X_t = np.asarray(res.X_mov_transformed) if sel2.all() else X2 @ res.H[:3, :3].T + res.H[:3, 3]
        pc2._set_xyz(X_t)  # copies the three columns into the frame
        _log.info(f"Finished in {time.time() - start_time:.3f} seconds!")
        # the reference returns pc2.X (simpleicp.py:324): the same values as X_t, which is handed
        # out directly instead of being re-assembled from the frame's columns (5 ms at 1M points)
        return res.H, X_t, res.rbp, res.residuals


def simpleicp(X_fix, X_mov, **kwargs):
    """Functional front end: ``H, X_mov_transformed, rbp, distance_residuals =
    simpleicp(X_fix, X_mov, correspondences=..., ...)``.

    X_fix / X_mov: (n, 3) float64 NumPy arrays or CUDA torch tensors.  Keyword arguments are
    those of ``SimpleICP.run``.  Inputs are not modified.
    """
    kwargs.setdefault("want_normals", False)
    res = register(X_fix, X_mov, **kwargs)
    return res.H, res.X_mov_transformed, res.rbp, res.residuals
