"""NumPy statement of sicp_overlap_graph's rule (include/sicp_b200.h, DESIGN.md §6.10): for every
ordered pair (a, b), count_ab = the points p of X_a[::s] whose query q = T_ab^-1 p has a point of
X_b at squared distance below r^2 (cKDTree's strict distance_upper_bound), T_ab = H_a^-1 H_b."""
import numpy as np
from scipy.spatial import cKDTree


def relative(H, a, b):
    """T_ab = H_a^-1 H_b with H_a's inverse formed from its transposed rotation (the library's)."""
    if H is None:
        return np.eye(4)
    Ra, ta = H[a][:3, :3], H[a][:3, 3]
    inv = np.eye(4)
    inv[:3, :3] = Ra.T
    inv[:3, 3] = -(Ra.T @ ta)
    return inv @ H[b]


def queries(Xa, T, s):
    """The queries of X_a[::s] in b's frame: q = R^T p - R^T t for T = (R, t)."""
    R, t = T[:3, :3], T[:3, 3]
    return Xa[::s] @ R - R.T @ t


def count(Xa, Xb, T, r, s):
    """count_ab through a k-d tree of X_b."""
    if len(Xa) == 0 or len(Xb) == 0:
        return 0
    d, _ = cKDTree(Xb).query(queries(Xa, T, s), distance_upper_bound=r)
    return int(np.count_nonzero(d < r))


def overlap_graph(clouds, H, r, s):
    """(pairs, counts) of the rule: one row per a < b with count_ab + count_ba > 0, ascending."""
    pairs, counts = [], []
    for a in range(len(clouds)):
        for b in range(a + 1, len(clouds)):
            cab = count(clouds[a], clouds[b], relative(H, a, b), r, s)
            cba = count(clouds[b], clouds[a], relative(H, b, a), r, s)
            if cab + cba > 0:
                pairs.append((a, b))
                counts.append((cab, cba))
    return np.array(pairs, dtype=np.int64).reshape(-1, 2), np.array(counts, dtype=np.int64).reshape(-1, 2)
