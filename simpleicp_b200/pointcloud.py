"""PointCloud container of the facade.

API mirror of the reference's ``PointCloud(pd.DataFrame)`` (python/simpleicp/pointcloud.py:15-226):
same constructor contract (columns x, y, z required, boolean ``selected`` added), same properties
and selection helpers, same exceptions.  The compute methods of the reference
(select_in_range :149-171, estimate_normals :173-203, transform_by_H :205-217) are served by the
CUDA library; they are kept as methods here so user code calling them directly keeps working.
"""
from __future__ import annotations

from pathlib import Path
from typing import List, Optional

import numpy as np
import pandas as pd

from . import _capi

_XYZ = ["x", "y", "z"]
_NORMAL_COLUMNS = ("nx", "ny", "nz", "planarity")


class PointCloudException(Exception):
    """Raised when the PointCloud class is misused (reference: pointcloud.py:229)."""


class PointCloud(pd.DataFrame):
    """DataFrame of points with a boolean ``selected`` column."""

    def __init__(self, *args, remapping: Optional[str] = None, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        missing = [c for c in _XYZ if c not in self]
        if missing:
            raise PointCloudException(f'Column "{missing[0]}" is missing in DataFrame.')
        self._num_points = len(self)
        if "selected" not in self:
            self["selected"] = np.ones(self._num_points, dtype=bool)

    # ---- coordinates
    @property
    def x(self) -> np.ndarray:
        return self["x"].to_numpy()

    @property
    def y(self) -> np.ndarray:
        return self["y"].to_numpy()

    @property
    def z(self) -> np.ndarray:
        return self["z"].to_numpy()

    @property
    def X(self) -> np.ndarray:
        """(n, 3) array of all points."""
        return self[_XYZ].to_numpy()

    def _sel(self) -> np.ndarray:
        return self["selected"].to_numpy(dtype=bool)

    @property
    def x_selected(self) -> np.ndarray:
        return self.x[self._sel()]

    @property
    def y_selected(self) -> np.ndarray:
        return self.y[self._sel()]

    @property
    def z_selected(self) -> np.ndarray:
        return self.z[self._sel()]

    @property
    def X_selected(self) -> np.ndarray:
        return self.X[self._sel()]

    # ---- selection
    @property
    def idx_selected(self) -> np.ndarray:
        return np.flatnonzero(self._sel())

    @idx_selected.setter
    def idx_selected(self, idx_selected: List[int]) -> None:
        mask = np.zeros(self._num_points, dtype=bool)
        mask[np.asarray(idx_selected, dtype=np.int64)] = True
        self["selected"] = mask

    @property
    def num_points(self) -> int:
        return self._num_points

    @property
    def num_selected_points(self) -> int:
        return int(self._sel().sum())

    def select_all_points(self) -> None:
        self["selected"] = np.ones(self._num_points, dtype=bool)

    def unselect_all_points(self) -> None:
        self["selected"] = np.zeros(self._num_points, dtype=bool)

    def select_by_indices(self, indices: List[int]) -> None:
        """Keep only currently selected points whose index is in ``indices``."""
        self.idx_selected = np.intersect1d(self.idx_selected, indices)

    def select_n_points(self, n: int) -> None:
        """Thin the selection to n points, equidistant in index (reference :132-147:
        round-half-even of linspace over the selected indices)."""
        idx = self.idx_selected
        if idx.size > n:
            self.idx_selected = idx[subsample_indices(idx.size, n)]

    # ---- compute methods (GPU)
    def select_in_range(self, X: np.ndarray, max_range: float) -> None:
        """Keep selected points whose nearest neighbour in X is strictly closer than max_range."""
        if np.shape(X)[1] != 3:
            raise PointCloudException("X must have 3 columns!")
        idx = self.idx_selected
        with _capi.Engine() as eng:
            eng.set_clouds(self.X, X)
            eng.set_selected(idx)
            try:
                keep = eng.select_in_range(np.eye(4), max_range)
            except _capi.SicpError as e:
                if e.code != _capi.SICP_ERR_NO_OVERLAP:
                    raise
                keep = np.zeros(idx.size, dtype=bool)
        self.idx_selected = idx[keep]

    def estimate_normals(self, neighbors: int) -> None:
        """Normals and planarity of the selected points from their k nearest neighbours."""
        idx = self.idx_selected
        self.set_normals(idx, *estimate_normals_of(self.X, idx, neighbors))

    def set_normals(self, idx, nx, ny, nz, planarity) -> None:
        """Store float32 attribute columns (NaN where not estimated), as the reference does
        (pointcloud.py:200-203: ``pd.arrays.SparseArray`` of a dense NaN-filled column).  The sparse
        column is assembled directly from (index, value) pairs when the indices are strictly
        increasing -- the same array, dtype and sparse index, without scanning n points four
        times (15 -> 1.5 ms at one million points)."""
        idx = np.asarray(idx, dtype=np.int64)
        for name, vals in zip(_NORMAL_COLUMNS, (nx, ny, nz, planarity)):
            self[name] = _sparse_f32_column(self._num_points, idx, np.asarray(vals, dtype=np.float32))

    def transform_by_H(self, H: np.ndarray) -> None:
        """Apply a 4 x 4 homogeneous transformation to all points, in place."""
        H = np.asarray(H, dtype=float)
        if abs(H[3, 3] - 1.0) > 0 or np.any(H[3, :3] != 0):  # projective: not the GPU's case
            Xh = np.hstack((self.X, np.ones((self._num_points, 1)))) @ H.T
            Xe = Xh[:, :3] / Xh[:, 3:4]
        else:
            with _capi.Engine() as eng:
                eng.set_clouds(self.X[:1], self.X)
                Xe = eng.transform(H)
        self._set_xyz(Xe)

    def _set_xyz(self, Xe: np.ndarray) -> None:
        self["x"] = Xe[:, 0]
        self["y"] = Xe[:, 1]
        self["z"] = Xe[:, 2]

    def write_xyz(self, file: Path):
        """CloudCompare-style xyz text file (reference: pointcloud.py:219-226)."""
        self[_XYZ].to_csv(file, sep=" ", header=["//X", "Y", "Z"], index=False, float_format="%.3f")


def estimate_normals_of(X, idx, neighbors: int):
    """(nx, ny, nz, planarity) float32 of the points X[idx] (idx None: all of them) from their k
    nearest neighbours in X, itself included: what PointCloud.estimate_normals stores."""
    with _capi.Engine() as eng:
        eng.set_clouds(X, X[:1])
        eng.set_selected(idx)
        return eng.estimate_normals(neighbors)


def _sparse_f32_column(n: int, idx: np.ndarray, vals: np.ndarray):
    """``pd.arrays.SparseArray(col)`` for ``col = full(n, nan, float32); col[idx] = vals``."""
    if idx.size and n < 2**31 and (idx.size == 1 or bool(np.all(idx[1:] > idx[:-1]))) and idx[0] >= 0 and idx[-1] < n:
        try:
            from pandas._libs.sparse import IntIndex

            stored = ~np.isnan(vals)  # the dense route does not store NaN values either
            return pd.arrays.SparseArray(vals[stored], sparse_index=IntIndex(n, idx[stored].astype(np.int32)),
                                         fill_value=np.nan, dtype=pd.SparseDtype(np.float32, np.nan))
        except Exception:  # private pandas module moved: the dense route below is always valid
            pass
    col = np.full(n, np.nan, dtype=np.float32)
    col[idx] = vals
    return pd.arrays.SparseArray(col)


def subsample_indices(m: int, n: int) -> np.ndarray:
    """Positions of n equidistant picks among m items: rint(linspace(0, m - 1, n)) — NumPy's
    linspace and round-half-even are kept on the host so the picks are bit-identical to the
    reference's (pointcloud.py:142-144)."""
    return np.round(np.linspace(0, m - 1, n)).astype(int)
