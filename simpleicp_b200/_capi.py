"""ctypes binding of libsicp_b200.so (the C ABI declared in include/sicp_b200.h).

There is no CPU fallback: if the library is missing it is built with nvcc; if that is impossible
an ImportError is raised, and creating an Engine without a CUDA device raises SicpError.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path
from typing import Optional, Sequence

import numpy as np

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libsicp_b200.so"

SICP_OK, SICP_ERR_BAD_ARG, SICP_ERR_NO_OVERLAP, SICP_ERR_TOO_FEW_CORR = 0, 1, 2, 3
SICP_ERR_CUDA, SICP_ERR_SINGULAR, SICP_ERR_STATE = 4, 5, 6
ABI_VERSION = 5  # include/sicp_b200.h: SICP_ABI_VERSION
NN_AUTO, NN_GRID, NN_BRUTE = 0, 1, 2
SIGN_DGEEV, SIGN_CANONICAL = 0, 1

# selection diagnostics of Engine.phase_times() (csrc/reject_solve.cuh: SelectPath, SelectOutcome)
SLOT_SEL_PATH, SLOT_SEL_FUSED = 29, 30
SEL_PATH_RADIX, SEL_PATH_BINSTORE = 0, 2
SEL_OK, SEL_NO_PREDICTION, SEL_MEDIAN_OUTSIDE = 0, 1, 3
SEL_MEDIAN_GAP, SEL_MEDIAN_CANDIDATES, SEL_MAD_BRACKET, SEL_MAD_WINDOW = 5, 6, 7, 8
SEL_MAD_CANDIDATES, SEL_BIN_CAP = 9, 10
SEL_OUTCOMES = {
    "SEL_OK": SEL_OK, "SEL_NO_PREDICTION": SEL_NO_PREDICTION, "SEL_MEDIAN_OUTSIDE": SEL_MEDIAN_OUTSIDE,
    "SEL_MEDIAN_GAP": SEL_MEDIAN_GAP, "SEL_MEDIAN_CANDIDATES": SEL_MEDIAN_CANDIDATES,
    "SEL_MAD_BRACKET": SEL_MAD_BRACKET, "SEL_MAD_WINDOW": SEL_MAD_WINDOW,
    "SEL_MAD_CANDIDATES": SEL_MAD_CANDIDATES, "SEL_BIN_CAP": SEL_BIN_CAP,
}

# every symbol include/sicp_b200.h declares (tests check the library exports all of them)
SYMBOLS = (
    "sicp_abi_version", "sicp_create", "sicp_destroy", "sicp_last_error", "sicp_set_option",
    "sicp_set_clouds", "sicp_set_selected", "sicp_select_in_range", "sicp_estimate_normals",
    "sicp_set_normals", "sicp_set_mov_normals", "sicp_get_knn", "sicp_match", "sicp_reject", "sicp_solve",
    "sicp_uncertainties", "sicp_run", "sicp_get_transform", "sicp_get_residuals", "sicp_iterate", "sicp_transform",
    "sicp_select_n_points", "sicp_register",
    "sicp_register_batch", "sicp_set_map", "sicp_register_to_map", "sicp_register_pairs", "sicp_register_joint", "sicp_get_batch_outputs",
    "sicp_register_joint_priors", "sicp_register_joint_relative", "sicp_get_joint_covariances",
    "sicp_get_joint_selected_covariances",
    "sicp_map_insert", "sicp_get_map", "sicp_map_crop", "sicp_map_thin", "sicp_map_carve", "sicp_map_distances", "sicp_overlap_graph", "sicp_get_timings", "sicp_time_stages", "sicp_get_phase_times", "sicp_get_match_phase_times",
    "sicp_debug_seed_predictor", "sicp_debug_match_counts", "sicp_debug_grid_params",
    "sicp_xyz_load", "sicp_xyz_free", "sicp_xyz_save", "sicp_io_last_error",
)


class LsqParams(C.Structure):
    _fields_ = [("x0", C.c_double * 6), ("observed", C.c_double * 6),
                ("obs_weight", C.c_double * 6), ("distance_weight", C.c_double)]


class RunParams(C.Structure):
    _fields_ = [("min_planarity", C.c_double), ("min_change", C.c_double),
                ("max_iterations", C.c_int32), ("reserved", C.c_int32), ("lsq", LsqParams)]


class RegisterParams(C.Structure):
    _fields_ = [("correspondences", C.c_int64), ("neighbors", C.c_int32), ("mov_neighbors", C.c_int32),
                ("max_overlap_distance", C.c_double), ("run", RunParams), ("max_angle_rad", C.c_double)]


class IterRecord(C.Structure):
    _fields_ = [("n_kept", C.c_int64), ("median", C.c_double), ("mad", C.c_double),
                ("mean_dist", C.c_double), ("std_dist", C.c_double), ("x", C.c_double * 6),
                ("mean_res", C.c_double), ("std_res", C.c_double), ("distance_weight", C.c_double),
                ("lm_iterations", C.c_int32), ("n_bruteforce", C.c_int32)]


class RunResult(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("converged", C.c_int32), ("x", C.c_double * 6),
                ("H", C.c_double * 16), ("sigma", C.c_double * 6), ("n_residuals", C.c_int64),
                ("loop_ms", C.c_double)]


class Timings(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("upload_ms", "grid_mov_ms", "grid_fix_ms", "overlap_ms",
                                          "normals_ms", "match_ms", "reject_solve_ms",
                                          "transform_ms")] + [("kernel_launches", C.c_int64),
                                                            ("fused_iterations", C.c_int64),
                                                            ("rerun_iterations", C.c_int64),
                                                            ("mov_normals_ms", C.c_double),
                                                            ("overlap_candidates", C.c_int64)]


class PairResult(C.Structure):
    _fields_ = [("status", C.c_int32), ("iterations", C.c_int32), ("converged", C.c_int32),
                ("reserved", C.c_int32), ("n_kept", C.c_int64), ("H", C.c_double * 16),
                ("x", C.c_double * 6), ("sigma", C.c_double * 6), ("mean_res", C.c_double),
                ("std_res", C.c_double)]


class SicpError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"libsicp_b200 error {code}: {message}")
        self.code = code
        self.message = message


_lib = None


def load_library(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if needed) the CUDA library.  Never falls back to a CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    override = os.environ.get("SICP_B200_LIB")  # diagnostics: an experimental build of the same ABI
    if override:
        lib_path = Path(override)
        if not lib_path.exists():
            raise ImportError(f"SICP_B200_LIB={override} does not exist")
    else:
        lib_path = LIB_PATH
    if not override:
        if build_if_missing:
            # digest-checked and cheap when up to date: a library left over from older sources is
            # rebuilt instead of being loaded against newer ctypes struct layouts.  Where nvcc is
            # absent (a box that only received the built .so) the existing library is used and the
            # ABI version check below is the guard.
            from . import _build

            try:
                _build.build()
            except RuntimeError:
                if not LIB_PATH.exists():
                    raise ImportError(f"{LIB_PATH} is missing and cannot be built (nvcc not found)")
        elif not LIB_PATH.exists():
            raise ImportError(f"{LIB_PATH} is missing; run `python -m simpleicp_b200._build`")
    lib = C.CDLL(str(lib_path))
    vp, i32, i64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    lib.sicp_abi_version.restype = i32
    if lib.sicp_abi_version() != ABI_VERSION:
        raise ImportError(f"{lib_path} has ABI version {lib.sicp_abi_version()}, this binding needs "
                          f"{ABI_VERSION}: rebuild with `python -m simpleicp_b200._build --force`")
    lib.sicp_last_error.restype = C.c_char_p
    lib.sicp_last_error.argtypes = [vp]
    sigs = {
        "sicp_create": [i32, vp, C.POINTER(vp)],
        "sicp_destroy": [vp],
        "sicp_set_option": [vp, C.c_char_p, dbl],
        "sicp_set_clouds": [vp, vp, i64, vp, i64],
        "sicp_set_selected": [vp, vp, i64],
        "sicp_select_in_range": [vp, C.POINTER(dbl), dbl, vp, C.POINTER(i64)],
        "sicp_estimate_normals": [vp, i32, vp, vp, vp, vp],
        "sicp_set_normals": [vp, vp, vp, vp, vp],
        "sicp_set_mov_normals": [vp, vp, vp, vp, vp, C.c_double],
        "sicp_get_knn": [vp, vp, vp],
        "sicp_match": [vp, C.POINTER(dbl), vp, vp],
        "sicp_reject": [vp, dbl, vp, C.POINTER(i64), C.POINTER(dbl)],
        "sicp_solve": [vp, C.POINTER(LsqParams), C.POINTER(dbl), C.POINTER(dbl), vp,
                       C.POINTER(dbl), C.POINTER(dbl)],
        "sicp_uncertainties": [vp, C.POINTER(dbl)],
        "sicp_run": [vp, C.POINTER(RunParams), C.POINTER(RunResult), C.POINTER(IterRecord)],
        "sicp_get_transform": [vp, C.POINTER(C.c_double)],
        "sicp_get_residuals": [vp, vp, i64, C.POINTER(i64)],
        "sicp_iterate": [vp, C.POINTER(RunParams), C.POINTER(dbl), C.POINTER(IterRecord)],
        "sicp_transform": [vp, C.POINTER(dbl), vp],
        "sicp_select_n_points": [vp, i64, vp],
        "sicp_register": [vp, vp, i64, vp, i64, C.POINTER(RegisterParams), C.POINTER(RunResult),
                          C.POINTER(IterRecord), vp, C.POINTER(i64)],
        "sicp_register_batch": [vp, i32, C.POINTER(vp), C.POINTER(i64), C.POINTER(vp), C.POINTER(i64),
                                C.POINTER(RegisterParams), vp, C.POINTER(PairResult), vp],
        "sicp_set_map": [vp, vp, i64],
        "sicp_register_to_map": [vp, i32, C.POINTER(vp), C.POINTER(i64), C.POINTER(RegisterParams), vp,
                                 C.POINTER(PairResult), vp],
        "sicp_register_pairs": [vp, i32, C.POINTER(vp), C.POINTER(i64), i32, C.POINTER(i32), C.POINTER(i32),
                                C.POINTER(RegisterParams), vp, C.POINTER(PairResult), vp],
        "sicp_register_joint": [vp, i32, C.POINTER(vp), C.POINTER(i64), i32, C.POINTER(i32), C.POINTER(i32),
                                C.POINTER(i32), vp, C.POINTER(RegisterParams), vp, C.POINTER(PairResult), vp],
        "sicp_register_joint_priors": [vp, i32, C.POINTER(vp), C.POINTER(i64), i32, C.POINTER(i32), C.POINTER(i32),
                                       C.POINTER(i32), vp, vp, vp, C.POINTER(RegisterParams), vp,
                                       C.POINTER(PairResult), vp],
        "sicp_register_joint_relative": [vp, i32, C.POINTER(vp), C.POINTER(i64), i32, C.POINTER(i32),
                                         C.POINTER(i32), C.POINTER(i32), vp, vp, vp, i32, C.POINTER(i32),
                                         C.POINTER(i32), vp, vp, C.POINTER(RegisterParams), vp,
                                         C.POINTER(PairResult), vp],
        "sicp_get_batch_outputs": [vp, i32, C.POINTER(vp), C.POINTER(vp), C.POINTER(IterRecord), C.POINTER(dbl)],
        "sicp_get_joint_covariances": [vp, i32, vp, i32, vp, C.POINTER(dbl)],
        "sicp_get_joint_selected_covariances": [vp, i32, vp, i32, vp, C.POINTER(dbl)],
        "sicp_map_insert": [vp, i32, C.POINTER(vp), C.POINTER(i64), vp, dbl, vp],
        "sicp_get_map": [vp, vp, i64, C.POINTER(i64)],
        "sicp_map_crop": [vp, i32, vp, dbl, C.POINTER(i64)],
        "sicp_map_thin": [vp, dbl, C.POINTER(i64)],
        "sicp_map_carve": [vp, i32, C.POINTER(vp), C.POINTER(i64), vp, vp, dbl, dbl, i32, vp, C.POINTER(i64)],
        "sicp_map_distances": [vp, i32, C.POINTER(vp), C.POINTER(i64), vp, dbl, i32, C.POINTER(vp), C.POINTER(vp),
                               C.POINTER(vp), C.POINTER(vp), vp],
        "sicp_overlap_graph": [vp, i32, C.POINTER(vp), C.POINTER(i64), vp, dbl, i64, vp, vp, vp, vp, i64,
                               C.POINTER(i64)],
        "sicp_get_timings": [vp, C.POINTER(Timings)],
        "sicp_time_stages": [vp, C.POINTER(RunParams), i32, i32, C.POINTER(dbl)],
        "sicp_get_phase_times": [vp, C.POINTER(dbl)],
        "sicp_get_match_phase_times": [vp, C.POINTER(dbl)],
        "sicp_debug_seed_predictor": [vp, dbl, dbl, dbl],
        "sicp_debug_match_counts": [vp, C.POINTER(i64)],
        "sicp_debug_grid_params": [vp, i32, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(i32)],
    }
    for name, args in sigs.items():
        # entry points added without a layout change keep the version: a library that predates
        # one of them is refused by name
        fn = getattr(lib, name, None)
        if fn is None:
            raise ImportError(f"{lib_path} does not export {name}: rebuild with "
                              f"`python -m simpleicp_b200._build --force`")
        fn.argtypes = args
        fn.restype = i32
    lib.sicp_xyz_load.argtypes = [C.c_char_p, C.POINTER(C.POINTER(dbl)), C.POINTER(i64)]
    lib.sicp_xyz_load.restype = i32
    lib.sicp_xyz_free.argtypes = [C.POINTER(dbl)]
    lib.sicp_xyz_free.restype = None
    lib.sicp_xyz_save.argtypes = [C.c_char_p, vp, i64, i32, i32]
    lib.sicp_xyz_save.restype = i32
    lib.sicp_io_last_error.restype = C.c_char_p
    _lib = lib
    return lib


def read_xyz(path) -> np.ndarray:
    """Fast multi-threaded .xyz reader (x y z per line, '/'/'#' comment lines skipped); the
    doubles equal what np.genfromtxt parses from the same text."""
    lib = load_library()
    p = C.POINTER(C.c_double)()
    n = C.c_int64(0)
    rc = lib.sicp_xyz_load(str(path).encode(), C.byref(p), C.byref(n))
    if rc != SICP_OK:
        raise OSError(lib.sicp_io_last_error().decode())
    try:
        return np.ctypeslib.as_array(p, shape=(int(n.value), 3)).copy()
    finally:
        lib.sicp_xyz_free(p)


def write_xyz(path, X, decimals: int = 3, header: bool = True) -> None:
    """CloudCompare-style text file like the reference's PointCloud.write_xyz."""
    lib = load_library()
    X = np.ascontiguousarray(X, dtype=np.float64)
    if X.ndim != 2 or X.shape[1] != 3:
        raise ValueError("X must have 3 columns!")
    rc = lib.sicp_xyz_save(str(path).encode(), X.ctypes.data, X.shape[0], int(decimals), int(header))
    if rc != SICP_OK:
        raise OSError(lib.sicp_io_last_error().decode())


def _ptr(a) -> Optional[int]:
    """Raw address of a NumPy array or a torch tensor (host or CUDA); None passes NULL."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(f"unsupported buffer type {type(a)}")


def _xyz_out_ptr(out, n: int) -> int:
    """Address of a caller's output for n transformed points: a NumPy array or a torch tensor
    (host, or CUDA on any device) of shape (n, 3), float64 and C-contiguous, into which the
    library writes 24 n bytes.  Anything else raises ValueError before the library is called."""
    if isinstance(out, np.ndarray):
        f64, contiguous, addr = out.dtype == np.float64, out.flags.c_contiguous, out.ctypes.data
    elif hasattr(out, "data_ptr") and hasattr(out, "is_contiguous"):
        import torch

        f64, contiguous, addr = out.dtype == torch.float64, out.is_contiguous(), out.data_ptr()
    else:
        raise ValueError(f"the output must be a NumPy array or a torch tensor, not {type(out).__name__}")
    if not (f64 and contiguous and tuple(out.shape) == (n, 3)):
        raise ValueError(f"the output must be a C-contiguous float64 array of shape ({n}, 3); got "
                         f"{out.dtype} of shape {tuple(out.shape)}{'' if contiguous else ', not contiguous'}")
    return addr


def _as_f64_xyz(X):
    """(n,3) float64 C-contiguous view/copy of a NumPy array or torch tensor."""
    if isinstance(X, np.ndarray) or not hasattr(X, "data_ptr"):
        X = np.ascontiguousarray(X, dtype=np.float64)
        if X.ndim != 2 or X.shape[1] != 3:
            raise ValueError("X must have 3 columns!")
        return X
    import torch

    if X.dim() != 2 or X.shape[1] != 3:
        raise ValueError("X must have 3 columns!")
    return X.to(torch.float64).contiguous()


def _clouds_arg(clouds, allow_none: bool = False):
    """A cloud sequence as the C calls take it: (keep, ptrs, counts) -- every cloud through
    _as_f64_xyz, their addresses and their point counts; with `allow_none` a None entry passes
    NULL and 0.  The library reads the arrays in `keep`, which may be copies made here: the caller
    holds `keep` until the call has returned."""
    keep = [None if X is None and allow_none else _as_f64_xyz(X) for X in clouds]
    ptrs = (C.c_void_p * len(keep))(*[_ptr(X) for X in keep])
    counts = (C.c_int64 * len(keep))(*[0 if X is None else int(X.shape[0]) for X in keep])
    return keep, ptrs, counts


def _shaped_arg(a, name: str, shape: tuple):
    """None, or `a` as a C-contiguous float64 array of `shape` (else ValueError)."""
    if a is None:
        return None
    a = np.ascontiguousarray(a, dtype=np.float64)
    if a.shape != shape:
        raise ValueError(f"{name} must have shape {shape}, got {a.shape}")
    return a


def _ids_arg(ids, name: str):
    """(n, 2) integer cloud ids, n >= 1, as their two columns in contiguous int32 arrays (else
    ValueError); `name` is "pairs" or "edges".  The library checks them against [0, n_clouds)."""
    ids = np.asarray(ids)
    if ids.ndim != 2 or ids.shape[1] != 2 or ids.shape[0] < 1 or not np.issubdtype(ids.dtype, np.integer):
        raise ValueError(f"{name} must be integers of shape (n_{name}, 2) with n_{name} >= 1, got {ids.dtype} "
                         f"of shape {ids.shape}")
    if ids.min() < -(1 << 31) or ids.max() >= (1 << 31):
        raise ValueError("cloud ids must fit in int32")
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    return np.ascontiguousarray(ids[:, 0]), np.ascontiguousarray(ids[:, 1])


def _d6(v: Sequence[float]):
    return (C.c_double * 6)(*[float(x) for x in v])


def _d16(H) -> "C.Array":
    H = np.asarray(H, dtype=np.float64).reshape(16)
    return (C.c_double * 16)(*H.tolist())


def current_stream_ptr(device: int) -> int:
    """torch's current CUDA stream on `device` (PyTorch owns streams and user-visible buffers);
    the legacy default stream when torch is not importable."""
    try:
        import torch

        if torch.cuda.is_available():
            return int(torch.cuda.current_stream(device).cuda_stream)
    except ImportError:
        pass
    return 0


def current_device() -> int:
    try:
        import torch

        if torch.cuda.is_available():
            return int(torch.cuda.current_device())
    except ImportError:
        pass
    return 0


def pinned_empty(shape, dtype) -> np.ndarray:
    """Host output buffer in pinned memory (through torch) so D2H copies run at link speed."""
    try:
        import torch

        if torch.cuda.is_available():
            tdt = {np.float64: torch.float64, np.float32: torch.float32, np.int64: torch.int64,
                   np.uint8: torch.uint8}[np.dtype(dtype).type]
            return torch.empty(shape, dtype=tdt, pin_memory=True).numpy()
    except (ImportError, RuntimeError):
        pass
    return np.empty(shape, dtype=dtype)


class Engine:
    """Thin object wrapper over one sicp_ctx."""

    def __init__(self, device: int = 0, stream: Optional[int] = None):
        self._lib = load_library()
        self._h = C.c_void_p()
        self.device = device
        st = current_stream_ptr(device) if stream is None else stream
        rc = self._lib.sicp_create(device, C.c_void_p(st), C.byref(self._h))
        if rc != SICP_OK:
            msg = self._lib.sicp_last_error(None).decode()
            self._h = C.c_void_p()
            raise SicpError(rc, msg)
        self.n_fix = self.n_mov = self.K = self.n_map = 0

    # -- plumbing
    def _check(self, rc: int):
        if rc != SICP_OK:
            raise SicpError(rc, self._lib.sicp_last_error(self._h).decode())

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.sicp_destroy(self._h)
            self._h = C.c_void_p()

    @property
    def alive(self) -> bool:
        return bool(getattr(self, "_h", None))

    def reset_options(self):
        """Back to the library defaults (used when a cached engine is handed out again)."""
        self._check(self._lib.sicp_set_option(self._h, b"defaults", 0.0))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def set_option(self, key: str, value: float):
        self._check(self._lib.sicp_set_option(self._h, key.encode(), float(value)))

    # -- stages
    def set_clouds(self, X_fix, X_mov):
        Xf, Xm = _as_f64_xyz(X_fix), _as_f64_xyz(X_mov)
        self.n_fix, self.n_mov = int(Xf.shape[0]), int(Xm.shape[0])
        self._check(self._lib.sicp_set_clouds(self._h, _ptr(Xf), self.n_fix, _ptr(Xm), self.n_mov))
        self.K = 0

    def set_selected(self, idx=None):
        if idx is None:
            self._check(self._lib.sicp_set_selected(self._h, None, self.n_fix))
            self.K = self.n_fix
        else:
            idx = np.ascontiguousarray(idx, dtype=np.int64)
            self._check(self._lib.sicp_set_selected(self._h, _ptr(idx), idx.size))
            self.K = int(idx.size)

    def select_in_range(self, H0, max_range: float) -> np.ndarray:
        keep = np.empty(self.K, dtype=np.uint8)
        n = C.c_int64(0)
        self._check(self._lib.sicp_select_in_range(self._h, _d16(H0), float(max_range), _ptr(keep),
                                                   C.byref(n)))
        return keep.astype(bool)

    def estimate_normals(self, neighbors: int, download: bool = True):
        if not download:
            self._check(self._lib.sicp_estimate_normals(self._h, int(neighbors), None, None, None, None))
            return None
        out = np.empty((4, self.K), dtype=np.float32)
        self._check(self._lib.sicp_estimate_normals(
            self._h, int(neighbors), out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data,
            out[3].ctypes.data))
        return out[0], out[1], out[2], out[3]

    def set_normals(self, nx, ny, nz, planarity):
        a = [np.ascontiguousarray(v, dtype=np.float32) for v in (nx, ny, nz, planarity)]
        for v in a:
            if v.size != self.K:
                raise ValueError("normal arrays must have one entry per selected point")
        self._check(self._lib.sicp_set_normals(self._h, *[_ptr(v) for v in a]))

    def set_mov_normals(self, nx, ny, nz, planarity, max_angle_deg=None):
        """Movable-side attributes (sicp_set_mov_normals): n_mov floats each, NaN = not estimated;
        ``set_mov_normals(None, None, None, None)`` clears them.  ``max_angle_deg`` switches the
        rejection by the angle between the normals on (degrees, like the facade's other angles)."""
        if nx is None and ny is None and nz is None and planarity is None:
            self._check(self._lib.sicp_set_mov_normals(self._h, None, None, None, None, -1.0))
            return
        a = [np.ascontiguousarray(v, dtype=np.float32) for v in (nx, ny, nz, planarity)]
        for v in a:
            if v.size != self.n_mov:
                raise ValueError("movable normal arrays must have one entry per movable point")
        ang = -1.0 if max_angle_deg is None else float(np.deg2rad(max_angle_deg))
        self._check(self._lib.sicp_set_mov_normals(self._h, *[_ptr(v) for v in a], ang))

    def get_knn(self, k: int):
        """Neighbour lists of the last estimate_normals (needs set_option("keep_knn", 1) before it)."""
        idx = np.empty((self.K, k), dtype=np.int64)
        d2 = np.empty((self.K, k), dtype=np.float64)
        self._check(self._lib.sicp_get_knn(self._h, _ptr(idx), _ptr(d2)))
        return idx, d2

    def match(self, H):
        idx = np.empty(self.K, dtype=np.int64)
        d = np.empty(self.K, dtype=np.float64)
        self._check(self._lib.sicp_match(self._h, _d16(H), _ptr(idx), _ptr(d)))
        return idx, d

    def reject(self, min_planarity: float):
        keep = np.empty(self.K, dtype=np.uint8)
        n = C.c_int64(0)
        stats = (C.c_double * 4)()
        self._check(self._lib.sicp_reject(self._h, float(min_planarity), _ptr(keep), C.byref(n), stats))
        return keep.astype(bool), int(n.value), list(stats)

    @staticmethod
    def lsq_params(x0, observed, obs_weight, distance_weight) -> LsqParams:
        p = LsqParams()
        p.x0 = _d6(x0)
        p.observed = _d6(observed)
        p.obs_weight = _d6(obs_weight)
        p.distance_weight = float("nan") if distance_weight is None else float(distance_weight)
        return p

    def solve(self, x0, observed, obs_weight, distance_weight, n_kept: int):
        p = self.lsq_params(x0, observed, obs_weight, distance_weight)
        x = (C.c_double * 6)()
        H = (C.c_double * 16)()
        stats = (C.c_double * 2)()
        w = C.c_double(0)
        res = np.empty(n_kept, dtype=np.float64)
        self._check(self._lib.sicp_solve(self._h, C.byref(p), x, H, _ptr(res), stats, C.byref(w)))
        return np.array(x), np.array(H).reshape(4, 4), res, list(stats), float(w.value)

    def uncertainties(self) -> np.ndarray:
        s = (C.c_double * 6)()
        self._check(self._lib.sicp_uncertainties(self._h, s))
        return np.array(s)

    @staticmethod
    def run_params(min_planarity, min_change, max_iterations, lsq: LsqParams) -> RunParams:
        p = RunParams()
        p.min_planarity = float(min_planarity)
        p.min_change = float(min_change)
        p.max_iterations = int(max_iterations)
        p.lsq = lsq
        return p

    def run(self, params: RunParams):
        out = RunResult()
        log = (IterRecord * int(params.max_iterations))()
        self._check(self._lib.sicp_run(self._h, C.byref(params), C.byref(out), log))
        n = C.c_int64(0)
        res = np.empty(int(out.n_residuals), dtype=np.float64)
        self._check(self._lib.sicp_get_residuals(self._h, _ptr(res), res.size, C.byref(n)))
        return out, [log[i] for i in range(out.iterations)], res

    def select_n_points(self, n: int, want_idx: bool = True):
        """PointCloud.select_n_points on the device; returns the resulting selection (int64)."""
        k = min(int(n), self.K if self.K else self.n_fix)
        idx = np.empty(k, dtype=np.int64) if want_idx else None
        self._check(self._lib.sicp_select_n_points(self._h, int(n), None if idx is None else _ptr(idx)))
        self.K = k
        return idx

    def register_fused(self, X_fix, X_mov, correspondences, neighbors, max_overlap_distance,
                       params: RunParams, transform_out=None, mov_neighbors: int = 0,
                       max_angle_rad: float = -1.0):
        """SimpleICP.run as one library call (sicp_register): uploads, selection, normals, the
        loop and the final transform, with the movable upload overlapped with the fixed-side work.
        ``mov_neighbors`` = k > 0 estimates the movable cloud's normals from k neighbours on the
        device first (pc_mov.estimate_normals(k)); ``max_angle_rad`` (negative: off) then rejects
        by the angle between the normals."""
        Xf, Xm = _as_f64_xyz(X_fix), _as_f64_xyz(X_mov)
        self.n_fix, self.n_mov = int(Xf.shape[0]), int(Xm.shape[0])
        rp = self._register_params(correspondences, neighbors, params, max_overlap_distance, mov_neighbors,
                                   max_angle_rad)
        out = RunResult()
        log = (IterRecord * int(params.max_iterations))()
        if transform_out is None:
            transform_out = pinned_empty((self.n_mov, 3), np.float64)
        nsel = C.c_int64(0)
        self._check(self._lib.sicp_register(self._h, _ptr(Xf), self.n_fix, _ptr(Xm), self.n_mov, C.byref(rp),
                                            C.byref(out), log, _xyz_out_ptr(transform_out, self.n_mov),
                                            C.byref(nsel)))
        self.K = int(nsel.value)
        n = C.c_int64(0)
        res = np.empty(int(out.n_residuals), dtype=np.float64)
        self._check(self._lib.sicp_get_residuals(self._h, _ptr(res), res.size, C.byref(n)))
        return out, [log[i] for i in range(out.iterations)], res, transform_out

    def register_batch(self, pairs, correspondences, neighbors, params: RunParams,
                       max_overlap_distance: float = -1.0, observed=None, mov_neighbors: int = 0,
                       max_angle_rad: float = -1.0):
        """sicp_register_batch: SimpleICP.run for every (X_fix, X_mov) of `pairs` with one set of
        kernel launches per stage for the whole batch.  Clouds are NumPy arrays (pinned ones
        upload at link speed) or CUDA tensors; nothing is copied on the host.

        `max_overlap_distance` finite and > 0 runs the overlap filter per pair; `observed`, an
        (n_pairs, 6) array in radians, gives each pair its own x0 = observed values (None: those
        of `params`).  `mov_neighbors` / `max_angle_rad` as in register_fused, for every pair's
        movable cloud.  Returns the ctypes array of PairResult (status per pair); its attribute
        `n_selected` holds the selected fixed points of each pair (int64)."""
        keep_f, fp, nf = _clouds_arg([a for a, _ in pairs])
        keep_m, mp, nm = _clouds_arg([b for _, b in pairs])
        n = len(nm)
        observed = _shaped_arg(observed, "observed", (n, 6))
        rp = self._register_params(correspondences, neighbors, params, max_overlap_distance, mov_neighbors,
                                   max_angle_rad)
        return self._batched(self._lib.sicp_register_batch, params, nm, None, n, fp, nf, mp, nm, C.byref(rp),
                             _ptr(observed))

    def set_map(self, X_map):
        """sicp_set_map: upload a fixed cloud and build its grid once; it stays on this engine
        (``None`` releases it) and is the fixed cloud of every register_to_map call."""
        if X_map is None:
            self._check(self._lib.sicp_set_map(self._h, None, 0))
            self.n_map = 0
            return
        X = _as_f64_xyz(X_map)
        self._check(self._lib.sicp_set_map(self._h, _ptr(X), int(X.shape[0])))
        self.n_map = int(X.shape[0])

    def register_to_map(self, scans, correspondences, neighbors, params: RunParams,
                        max_overlap_distance: float = -1.0, observed=None, mov_neighbors: int = 0,
                        max_angle_rad: float = -1.0):
        """sicp_register_to_map: register_batch with the resident map (set_map) as the fixed cloud
        of every scan, which is neither uploaded nor gridded again, and with an overlap filter
        that only searches the map points near each scan.  Same arguments and result as
        register_batch, with the movable clouds `scans` in place of the pairs."""
        keep, mp, nm = _clouds_arg(scans)
        n = len(nm)
        observed = _shaped_arg(observed, "observed", (n, 6))
        rp = self._register_params(correspondences, neighbors, params, max_overlap_distance, mov_neighbors,
                                   max_angle_rad)
        return self._batched(self._lib.sicp_register_to_map, params, nm, None, n, mp, nm, C.byref(rp), _ptr(observed))

    def register_pairs(self, clouds, pairs, correspondences, neighbors, params: RunParams,
                       max_overlap_distance: float = -1.0, observed=None, mov_neighbors: int = 0,
                       max_angle_rad: float = -1.0):
        """sicp_register_pairs: register_batch for pairs drawn from one set of clouds.  `clouds` is a
        sequence of (n_i, 3) NumPy arrays or CUDA tensors, None for a cloud no pair uses; `pairs`
        is (n_pairs, 2) of (fixed, movable) indices into `clouds`.  Each referenced cloud is
        uploaded and gridded once (and with `mov_neighbors` given its normals once), and pair i's
        result equals, bit for bit, register_batch's for (clouds[pairs[i, 0]], clouds[pairs[i, 1]]).
        Same other arguments and result as register_batch (`n_mov` is the size of each pair's
        movable cloud), so batch_outputs works on it."""
        fix, mov = _ids_arg(pairs, "pairs")
        keep, ptrs, counts = _clouds_arg(clouds, allow_none=True)
        n = len(fix)
        observed = _shaped_arg(observed, "observed", (n, 6))
        rp = self._register_params(correspondences, neighbors, params, max_overlap_distance, mov_neighbors,
                                   max_angle_rad)
        i32p = C.POINTER(C.c_int32)
        return self._batched(self._lib.sicp_register_pairs, params, counts, mov, len(counts), ptrs, counts, n,
                             fix.ctypes.data_as(i32p), mov.ctypes.data_as(i32p), C.byref(rp), _ptr(observed))

    def register_joint(self, clouds, edges, fixed, H0, correspondences, neighbors, params: RunParams,
                       max_overlap_distance: float = -1.0, prior_H=None, prior_w=None, rel_pairs=None,
                       rel_H=None, rel_w=None):
        """sicp_register_joint_relative: one pose per cloud from the edges (n_edges, 2) of (fixed
        side, movable side) indices into `clouds` (NumPy arrays or CUDA tensors, None for a cloud no
        edge uses), `fixed` a boolean mask of the clouds whose pose is held, `H0` (n_clouds, 4, 4)
        or None (identity) the start poses, world <- cloud, the pose priors `prior_H`
        (n_clouds, 4, 4) and `prior_w` (n_clouds, 6) or None (DESIGN.md §6.12; both None is
        sicp_register_joint), and the relative observations `rel_pairs` (n_rel, 2) of clouds (a,
        b), `rel_H` (n_rel, 4, 4) and `rel_w` (n_rel, 6) or None (DESIGN.md §6.13; None is
        sicp_register_joint_priors).  Always the linearised rules; the lsq part of `params` is not
        read beyond its checks.  Returns (H, out): the final poses (n_clouds, 4, 4) and the
        PairResult array per edge (H = final T_a^-1 T_b), which batch_outputs reads."""
        fix, mov = _ids_arg(edges, "edges")
        keep, ptrs, counts = _clouds_arg(clouds, allow_none=True)
        n, m = len(fix), len(counts)
        is_fixed = np.ascontiguousarray(np.asarray(fixed, dtype=bool).reshape(m), dtype=np.int32)
        H0 = _shaped_arg(H0, "H0", (m, 4, 4))
        prior_H = _shaped_arg(prior_H, "prior_H", (m, 4, 4))
        prior_w = _shaped_arg(prior_w, "prior_w", (m, 6))
        ra = rb = np.zeros(0, dtype=np.int32)
        if rel_pairs is not None:
            ra, rb = _ids_arg(rel_pairs, "rel_pairs")
        k = len(ra)
        rel_H = _shaped_arg(rel_H, "rel_H", (k, 4, 4))
        rel_w = _shaped_arg(rel_w, "rel_w", (k, 6))
        rp = self._register_params(correspondences, neighbors, params, max_overlap_distance, 0, -1.0)
        H = np.zeros((m, 4, 4))
        i32p = C.POINTER(C.c_int32)
        out = self._batched(self._lib.sicp_register_joint_relative, params, counts, mov, m, ptrs, counts, n,
                            fix.ctypes.data_as(i32p), mov.ctypes.data_as(i32p), is_fixed.ctypes.data_as(i32p),
                            _ptr(H0), _ptr(prior_H), _ptr(prior_w), k, ra.ctypes.data_as(i32p),
                            rb.ctypes.data_as(i32p), _ptr(rel_H), _ptr(rel_w), C.byref(rp), _ptr(H))
        return H, out

    def joint_covariances(self, n_clouds: int, n_edges: int):
        """sicp_get_joint_covariances for the last register_joint: (cov, edge_cov, s0) with cov
        (n_clouds, 6, 6) the covariance of each cloud's (omega, d origin), edge_cov (n_edges, 6, 6)
        that of each edge's (alpha, d q) in frame a, and s0 (DESIGN.md §6.9)."""
        return self._joint_cov(self._lib.sicp_get_joint_covariances, n_clouds, n_edges)

    def joint_selected_covariances(self, n_clouds: int, n_edges: int):
        """sicp_get_joint_selected_covariances: joint_covariances' outputs after a register_joint
        under either joint_solver; after a sparse call by selected inversion of its factor
        (DESIGN.md §6.14)."""
        return self._joint_cov(self._lib.sicp_get_joint_selected_covariances, n_clouds, n_edges)

    def _joint_cov(self, fn, n_clouds: int, n_edges: int):
        cov = np.empty((int(n_clouds), 6, 6))
        edge_cov = np.empty((int(n_edges), 6, 6))
        s0 = C.c_double(0.0)
        self._check(fn(self._h, int(n_clouds), _ptr(cov), int(n_edges), _ptr(edge_cov), C.byref(s0)))
        return cov, edge_cov, s0.value

    def _batched(self, fn, params: RunParams, counts, mov, *args):
        """The end of the batched register_* calls: fn(ctx, *args, out, n_selected) with `out` one
        PairResult per pair, returned with its attributes `n_selected`, `n_mov` (the movable point
        counts, which batch_outputs sizes its clouds by) and `max_iterations`.  Pair i's movable
        cloud has counts[i] points, or counts[mov[i]] given the movable cloud ids `mov`, which are
        read only after the library has accepted them."""
        n = len(counts) if mov is None else len(mov)
        out = (PairResult * n)()
        n_selected = np.zeros(n, dtype=np.int64)
        self._check(fn(self._h, *args, out, _ptr(n_selected)))
        n_mov = np.array(counts, dtype=np.int64)
        out.n_selected = n_selected
        out.n_mov = n_mov if mov is None else n_mov[mov]
        out.max_iterations = int(params.max_iterations)
        return out

    def map_insert(self, clouds, H=None, *, voxel_size: float) -> np.ndarray:
        """sicp_map_insert: append to the resident map, per voxel of `voxel_size` it does not
        occupy, the first finite point of `clouds` (in order) falling into it, cloud i moved by
        H[i] first when `H` (n_clouds x 4 x 4) is given.  Returns the points each cloud added
        (int64)."""
        keep, ptrs, counts = _clouds_arg(clouds)
        n = len(counts)
        H = _shaped_arg(H, "H", (n, 4, 4))
        added = np.zeros(n, dtype=np.int64)
        self._check(self._lib.sicp_map_insert(self._h, n, ptrs, counts, _ptr(H), float(voxel_size), _ptr(added)))
        self.n_map += int(added.sum())
        return added

    def map_distances(self, clouds, H=None, *, max_distance: float, neighbors: int = 0):
        """sicp_map_distances: the nearest map point of every point of `clouds` (cloud i moved by
        H[i] first when `H` (n_clouds x 4 x 4) is given) whose squared distance is below
        max_distance^2.  Returns (idx, dist2, plane_dist, planarity, n_within): per cloud the map
        index (int64, -1 where none) and the squared distance (float64, +inf beyond the bound, NaN
        for a non-finite point); with `neighbors` = k > 0 per cloud the signed distance along the
        matched map point's normal (float64) and its planarity (float32), both NaN where idx is -1,
        else None; and the within points of each cloud (int64)."""
        keep, ptrs, counts = _clouds_arg(clouds)
        n = len(counts)
        H = _shaped_arg(H, "H", (n, 4, 4))
        k = int(neighbors)
        sizes = [int(c) for c in counts]
        idx = [np.empty(m, dtype=np.int64) for m in sizes]
        d2 = [np.empty(m, dtype=np.float64) for m in sizes]
        pd = [np.empty(m, dtype=np.float64) for m in sizes] if k > 0 else None
        pl = [np.empty(m, dtype=np.float32) for m in sizes] if k > 0 else None
        n_within = np.zeros(n, dtype=np.int64)

        def arr(a):
            return None if a is None else (C.c_void_p * n)(*[_ptr(x) for x in a])

        self._check(self._lib.sicp_map_distances(self._h, n, ptrs, counts, _ptr(H), float(max_distance), k, arr(idx),
                                                 arr(d2), arr(pd), arr(pl), _ptr(n_within)))
        return idx, d2, pd, pl, n_within

    def overlap_graph(self, clouds, H=None, *, max_distance: float, stride: int = 1, cap: int = 0):
        """sicp_overlap_graph: the overlapping pairs of `clouds` under the poses `H` ((n_clouds, 4,
        4) world <- cloud, or None: one frame).  Returns (total, pairs, counts): the number of
        pairs the rule reports, and the first min(total, cap) of them, pairs (m, 2) int64 (a < b,
        ascending) and counts (m, 2) int64 [count_ab, count_ba]."""
        keep, ptrs, counts = _clouds_arg(clouds)
        n = len(counts)
        H = _shaped_arg(H, "H", (n, 4, 4))
        cap = max(int(cap), 0)
        a, b = np.empty(cap, dtype=np.int32), np.empty(cap, dtype=np.int32)
        cab, cba = np.empty(cap, dtype=np.int64), np.empty(cap, dtype=np.int64)
        total = C.c_int64(0)
        self._check(self._lib.sicp_overlap_graph(self._h, n, ptrs, counts, _ptr(H), float(max_distance), int(stride),
                                                 _ptr(a), _ptr(b), _ptr(cab), _ptr(cba), cap, C.byref(total)))
        m = min(int(total.value), cap)
        return (int(total.value), np.column_stack((a[:m], b[:m])).astype(np.int64),
                np.column_stack((cab[:m], cba[:m])))

    def get_map(self) -> np.ndarray:
        """sicp_get_map: the resident map, (n_map, 3) float64 in map order."""
        n = C.c_int64(0)
        self._check(self._lib.sicp_get_map(self._h, None, 0, C.byref(n)))
        X = np.empty((int(n.value), 3), dtype=np.float64)
        self._check(self._lib.sicp_get_map(self._h, _ptr(X), X.shape[0], C.byref(n)))
        return X

    def map_crop(self, centers, radius: float) -> int:
        """sicp_map_crop: keep the map points whose squared distance to at least one of `centers`
        ((n, 3) float64) is below radius^2, in map order.  Returns the points removed."""
        c = np.ascontiguousarray(np.asarray(centers, dtype=np.float64).reshape(-1, 3))
        removed = C.c_int64(0)
        self._check(self._lib.sicp_map_crop(self._h, c.shape[0], _ptr(c), float(radius), C.byref(removed)))
        self.n_map -= int(removed.value)
        return int(removed.value)

    def map_thin(self, voxel_size: float) -> int:
        """sicp_map_thin: keep the first map point of every voxel key floor(p / voxel_size), in map
        order.  Returns the points removed."""
        removed = C.c_int64(0)
        self._check(self._lib.sicp_map_thin(self._h, float(voxel_size), C.byref(removed)))
        self.n_map -= int(removed.value)
        return int(removed.value)

    def map_carve(self, clouds, H=None, *, origins=None, radius: float, margin: float, min_passes: int = 1,
                  passes=None) -> int:
        """sicp_map_carve: remove the map points that at least `min_passes` rays pass, a ray running
        from cloud i's origin (origins[i], or with origins None H[i]'s translation column) to each
        finite point of cloud i (moved by H[i] first when `H` (n_clouds x 4 x 4) is given).
        `passes` is None or a uint32 array / tensor (host or CUDA) of the map's size before the
        call, which receives every map point's pass count.  Returns the points removed."""
        keep, ptrs, counts = _clouds_arg(clouds)
        n = len(counts)
        H = _shaped_arg(H, "H", (n, 4, 4))
        origins = _shaped_arg(origins, "origins", (n, 3))
        removed = C.c_int64(0)
        self._check(self._lib.sicp_map_carve(self._h, n, ptrs, counts, _ptr(H), _ptr(origins), float(radius),
                                             float(margin), int(min_passes), _ptr(passes), C.byref(removed)))
        self.n_map -= int(removed.value)
        return int(removed.value)

    def batch_outputs(self, result):
        """sicp_get_batch_outputs for `result`, the PairResult array the last register_batch /
        register_to_map / register_pairs on this engine returned: per pair (X_mov_transformed, residuals, log, T)
        -- the transformed movable cloud (pinned NumPy), the final residuals in kept order, the
        IterRecord of every iteration run and the applied 4 x 4 transform -- or None for a pair
        whose status is not SICP_OK."""
        n, it = len(result), int(result.max_iterations)
        ok = [result[i].status == SICP_OK for i in range(n)]
        X = [pinned_empty((int(result.n_mov[i]), 3), np.float64) if ok[i] else None for i in range(n)]
        R = [np.empty(int(result[i].n_kept), dtype=np.float64) if ok[i] else None for i in range(n)]
        log = (IterRecord * (n * it))()
        T = np.zeros((n, 16))
        self._check(self._lib.sicp_get_batch_outputs(
            self._h, n, (C.c_void_p * n)(*[_ptr(x) for x in X]), (C.c_void_p * n)(*[_ptr(r) for r in R]), log,
            T.ctypes.data_as(C.POINTER(C.c_double))))
        return [(X[i], R[i], [log[i * it + j] for j in range(result[i].iterations)], T[i].reshape(4, 4))
                if ok[i] else None for i in range(n)]

    @staticmethod
    def _register_params(correspondences, neighbors, params: RunParams, max_overlap_distance, mov_neighbors,
                         max_angle_rad) -> RegisterParams:
        rp = RegisterParams()
        rp.correspondences = int(correspondences)
        rp.neighbors = int(neighbors)
        rp.max_overlap_distance = float(max_overlap_distance)
        rp.run = params
        rp.mov_neighbors = int(mov_neighbors)
        rp.max_angle_rad = float(max_angle_rad)
        return rp

    def get_transform(self) -> np.ndarray:
        """The 4 x 4 transform the last run/solve applied to the movable cloud."""
        T = (C.c_double * 16)()
        self._check(self._lib.sicp_get_transform(self._h, T))
        return np.array(T).reshape(4, 4)

    def iterate(self, params: RunParams, x_in=None, want_record: bool = False):
        rec = IterRecord() if want_record else None
        self._check(self._lib.sicp_iterate(
            self._h, C.byref(params), None if x_in is None else _d6(x_in),
            C.byref(rec) if rec is not None else None))
        return rec

    def transform(self, H, out=None):
        """X_mov transformed by H.  `out` (None: a new pinned array) is an (n_mov, 3) float64
        C-contiguous NumPy array or torch tensor, host or CUDA on any device."""
        if out is None:
            out = pinned_empty((self.n_mov, 3), np.float64)
        self._check(self._lib.sicp_transform(self._h, _d16(H), _xyz_out_ptr(out, self.n_mov)))
        return out

    def time_stages(self, params: RunParams, reps: int, flush_l2: bool, outer_only: bool = False) -> dict:
        """Average device milliseconds per iteration of each kernel group (CUDA events).
        outer_only: only the events around the whole iteration (no bubbles from the inner ones)."""
        ms = (C.c_double * 4)()
        self._check(self._lib.sicp_time_stages(self._h, C.byref(params), int(reps),
                                               (1 if flush_l2 else 0) | (2 if outer_only else 0), ms))
        return {"match_grid": ms[0], "bruteforce_pass": ms[1], "reject_solve": ms[2], "iteration": ms[3]}

    def phase_times(self) -> list:
        """Diagnostics: block-0 phase stamps (us) of the last reject+solve kernel."""
        us = (C.c_double * 32)()
        self._check(self._lib.sicp_get_phase_times(self._h, us))
        return list(us)

    def match_phase_times(self) -> list:
        """Diagnostics: first- and last-block phase stamps (us) of the last one-pair grid match run
        with the option match_stamps (sicp_get_match_phase_times)."""
        us = (C.c_double * 16)()
        self._check(self._lib.sicp_get_match_phase_times(self._h, us))
        return list(us)

    def selection(self) -> dict:
        """Selection diagnostics of the last reject/solve launches (phase_times slots 29 and 30):
        which path produced the last record's median/MAD, and the outcome code of the last
        predictor attempt of the barrier-free kernel."""
        us = self.phase_times()
        return {"path": int(us[SLOT_SEL_PATH]), "fused": int(us[SLOT_SEL_FUSED]),
                "cnt_med": int(us[26]), "cnt_edge": int(us[27])}

    def seed_predictor(self, med: float, mad: float, min_planarity: float):
        """Test-only (sicp_debug_seed_predictor): the predictor the next match bins with."""
        self._check(self._lib.sicp_debug_seed_predictor(self._h, float(med), float(mad), float(min_planarity)))

    def match_counts(self) -> int:
        """Test-only (sicp_debug_match_counts): queries the last match answered from a certificate."""
        n = C.c_int64(0)
        self._check(self._lib.sicp_debug_match_counts(self._h, C.byref(n)))
        return int(n.value)

    def grid_params(self, side: str = "mov"):
        """Test-only (sicp_debug_grid_params): (origin, cell size, dims) of the movable ("mov") or
        the fixed ("fix") cloud's grid."""
        o = (C.c_double * 3)()
        h = C.c_double(0)
        dims = (C.c_int32 * 3)()
        self._check(self._lib.sicp_debug_grid_params(self._h, {"fix": 0, "mov": 1}[side], o, C.byref(h), dims))
        return np.array(o), float(h.value), tuple(int(d) for d in dims)

    def timings(self) -> dict:
        t = Timings()
        self._check(self._lib.sicp_get_timings(self._h, C.byref(t)))
        return {n: getattr(t, n) for n, _ in Timings._fields_}
