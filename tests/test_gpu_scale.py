"""The grid builder, the shared exclusive scan (grid.cu: scan_u32) and the map and batch engines at
the sizes they are built for, against references that are exact by construction.

Code that only runs at scale:
  * scan_u32's second level, k_scan_blocksums, walks the block sums 1024 at a time and carries a
    running total between chunks: the carry only runs past 1024 x 4096 = 4 194 304 elements.  Every
    grid build (cells), the batch overlap filter (fixed points), the map filter (mask words), the
    map's insert, crop, thin and distances (points), and sicp_register's overlap selection and
    final residuals (uint8 keep flags) scan through it;
  * the kernels with one thread per pair or cloud (k_compact_bounds: the boundaries of the batch
    filter and of the map's insert and distances; k_gather_flags, k_bbox_init) use more than one
    block only past 256, 128 or 42;
  * the batch match takes 4 lanes once Kmax x n_pairs passes 65 536;
  * the map filter's mask rows, popcount scan and survivor offsets are uint32 up to
    n_scans x n_map < 2^32.

Geometry.  The sheet lattice in units U = 2^-10 m: point (i, j) = O + (8i, 8j, (7i + 3j) mod 5) U,
numbered i * SJ + j.  A query that is a lattice point plus an offset in {-1, 0, 1}^3 units has that
point as its unique nearest neighbour (every other one is at least 7 units away in x or y, against
sqrt(3)), at an exact integer squared distance, so indices and distances come from the
construction.  test_gpu_nn_exact explains why the coordinates and their differences are exact at
both origins."""
import numpy as np
import pytest
import torch

from oracle import simpleicp_oracle as O
from test_gpu_batch_overlap import _lsq, _same_as_register, _same_bits
from test_gpu_map_distances import _plane
from test_gpu_nn_exact import ORIGINS, U, inverse, perm_H, rigid_apply, to_xyz
from test_grid_plan import plan
from test_map_crop_host import crop_keep, thin_oracle
from test_map_insert_host import insert_oracle, voxel_keys

import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from simpleicp_b200.simpleicp import _observed_in_radians

CHUNK = 1024 * 4096  # elements scanned before k_scan_blocksums carries into its next chunk


# ------------------------------------------------------------------------------ sheet lattice
def sheet_k(idx, SJ):
    """Lattice units of sheet points idx (point i * SJ + j is (8i, 8j, (7i + 3j) mod 5))."""
    i, j = np.divmod(np.asarray(idx, dtype=np.int64), SJ)
    return np.column_stack((8 * i, 8 * j, (7 * i + 3 * j) % 5))


def sheet_crop_keep(n, SJ, ck, R):
    """crop_keep of the first n sheet points for centres ck (lattice units) and radius R U, in
    integers: the differences, squares and sums are exact, so d2 < fl(r r) is |dk|^2 < R^2.  Only
    the lattice box around each centre is visited."""
    keep = np.zeros(n, dtype=bool)
    SI = (n + SJ - 1) // SJ
    for cx, cy, cz in np.asarray(ck, dtype=np.int64):
        i0, i1 = max(0, -((R - cx) // 8)), min(SI - 1, (cx + R) // 8)
        j0, j1 = max(0, -((R - cy) // 8)), min(SJ - 1, (cy + R) // 8)
        if i0 > i1 or j0 > j1:
            continue
        idx = (np.arange(i0, i1 + 1)[:, None] * SJ + np.arange(j0, j1 + 1)[None, :]).ravel()
        idx = idx[idx < n]
        k = sheet_k(idx, SJ)
        d2 = ((k[:, 0] - cx) ** 2 + (k[:, 1] - cy) ** 2) + (k[:, 2] - cz) ** 2
        keep[idx[d2 < R * R]] = True
    return keep


def _one_key(K):
    """Integer-valued voxel keys (rows) as one int64 each, order-free but one-to-one."""
    assert np.isfinite(K).all() and np.abs(K).max() < 2.0 ** 53
    K = K.astype(np.int64)
    K -= K.min(axis=0)
    span = K.max(axis=0) + 1
    assert float(span[0]) * float(span[1]) * float(span[2]) < 2.0 ** 62
    return (K[:, 0] * span[1] + K[:, 1]) * span[2] + K[:, 2]


def thin_fast(M, v):
    """thin_oracle with the keys as one int64 (np.unique over rows is too slow at 9 M points)."""
    _, first = np.unique(_one_key(voxel_keys(M, v)), return_index=True)
    return M[np.sort(first)]


def insert_fast(M, clouds, v):
    """insert_oracle with the keys as one int64."""
    C = np.concatenate([np.asarray(X, dtype=np.float64).reshape(-1, 3) for X in clouds])
    owner = np.repeat(np.arange(len(clouds)), [len(X) for X in clouds])
    fin = np.flatnonzero(np.isfinite(C).all(axis=1))
    _, first = np.unique(_one_key(np.concatenate([voxel_keys(M, v), voxel_keys(C[fin], v)])), return_index=True)
    add = fin[np.sort(first[first >= len(M)]) - len(M)]
    return np.concatenate([M, C[add]]), np.bincount(owner[add], minlength=len(clouds)).astype(np.int64)


def _near(rng, n_src, n, SJ, origin):
    """n queries: sheet points (random sources) moved by offsets in {-1, 0, 1}^3; (xyz, src, |o|^2)."""
    src = rng.integers(0, n_src, n)
    off = rng.integers(-1, 2, (n, 3))
    return to_xyz(sheet_k(src, SJ) + off, origin), src, (off * off).sum(axis=1)


@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_lattice_rules_equal_the_plain_rules(where):
    """The integer crop rule and the one-key thin and insert rules against crop_oracle,
    thin_oracle and insert_oracle on a 100 000-point sheet (a partial last row)."""
    n, SJ = 100_003, 317
    o = ORIGINS[where]
    M = to_xyz(sheet_k(np.arange(n), SJ), o)
    rng = np.random.default_rng(1)
    ck = np.concatenate([sheet_k(rng.integers(0, n, 40), SJ) + rng.integers(-9, 10, (40, 3)),
                         rng.integers(-400, 3000, (20, 3)) * [1, 1, 0]])
    for R in (5, 8, 64, 200):
        assert np.array_equal(sheet_crop_keep(n, SJ, ck, R), crop_keep(M, to_xyz(ck, o), R * U)), R
    clouds = [_near(rng, n, 30_000, SJ, o)[0], to_xyz(sheet_k(rng.integers(0, n, 20_000), SJ) + [0, 0, 40], o),
              np.full((5, 3), np.nan), np.zeros((0, 3))]
    for v in (16 * U, 5 * U):
        assert np.array_equal(thin_fast(M, v), thin_oracle(M, v)), v
        a, b = insert_fast(M, clouds, v), insert_oracle(M, clouds, v)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), v


# ------------------------------------------------------------------------------ 1. one-pair grid
@pytest.mark.gpu
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_one_pair_grid_past_the_scan_chunk(gpu, where):
    """A 9 M-point movable sheet at grid_target_occupancy 1: its grid has more than two scan
    chunks of cells.  match(I), match(H) for a signed axis permutation H, and select_in_range
    between the offsets' squared distances 2 and 3 give the construction's answer."""
    o = ORIGINS[where]
    n_mov, SJ = 9_000_001, 3001
    Mk = sheet_k(np.arange(n_mov), SJ)
    M = to_xyz(Mk, o)
    rng = np.random.default_rng(2)
    Qk_src = rng.integers(0, n_mov, 1_000_000)
    off = rng.integers(-1, 2, (len(Qk_src), 3))
    Qk = Mk[Qk_src] + off
    R = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]])
    s = np.array([5, -3, 2])
    with _capi.Engine() as e:
        e.set_option("grid_target_occupancy", 1.0)
        for H, Pk in ((np.eye(4), Qk), (perm_H(R, s, o), Qk @ R.T + s)):
            P = to_xyz(Pk, o)
            assert np.array_equal(rigid_apply(inverse(H), P), to_xyz(Qk, o)), "the transform is not exact"
            e.set_clouds(P, M)
            _, _, dims = e.grid_params("mov")
            assert dims[0] * dims[1] * dims[2] > 2 * CHUNK, dims
            e.set_selected(None)
            z = np.zeros(e.K, dtype=np.float32)
            e.set_normals(z, z, np.ones(e.K, dtype=np.float32), np.full(e.K, 0.9, dtype=np.float32))
            idx, d = e.match(H)
            assert np.array_equal(idx, Qk_src)
            # the point-to-plane distance through the normal (0, 0, 1): one coordinate difference
            assert np.array_equal(d, rigid_apply(H, M[Qk_src])[:, 2] - P[:, 2])
            keep = e.select_in_range(H, 1.5 * U)  # r^2 = 2.25 U^2, exact
            assert np.array_equal(keep, (off * off).sum(axis=1) <= 2)


def _offset_sheet(where, seed):
    """The 9 M-point sheet (movable) and its points moved by offsets in {-1, 0, 1}^3 units (fixed):
    fixed point i has movable point i as its nearest, at squared distance |off_i|^2 U^2."""
    n, SJ = 9_000_001, 3001
    Mk = sheet_k(np.arange(n), SJ)
    off = np.random.default_rng(seed).integers(-1, 2, (n, 3))
    return to_xyz(Mk + off, ORIGINS[where]), to_xyz(Mk, ORIGINS[where]), off


@pytest.mark.gpu
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_register_overlap_selection_past_the_scan_chunk(gpu, where):
    """sicp_register with max_overlap_distance on a 9 M-point fixed cloud: the keep flags of all
    its points are compacted into the selection on the device, over more than two scan chunks.
    With correspondences >= the survivors the selection is the survivors, which the construction
    gives (|off|^2 <= 2 for r = 1.5 U), and the one call equals the stage-by-stage path
    (select_in_range, the compaction in NumPy) bit for bit.  The sheet is nearly a plane: the
    in-plane parameters are fixed, so the solve stays regular."""
    X_fix, X_mov, off = _offset_sheet(where, 5)
    want = np.flatnonzero((off * off).sum(axis=1) <= 2)
    assert want[-1] > 2 * CHUNK
    kw = dict(correspondences=len(X_fix), max_overlap_distance=1.5 * U, min_planarity=0.0, max_iterations=3,
              rbp_observation_weights=(0.0, 0.0, np.inf, np.inf, np.inf, 0.0))
    with _capi.Engine() as e:
        a = sb.register(X_fix, X_mov, engine=e, want_normals=False, **kw)  # one call
        b = sb.register(X_fix, X_mov, engine=e, want_normals=True, **kw)   # stage by stage
    assert np.array_equal(a.idx_selected, want) and np.array_equal(b.idx_selected, want)
    assert np.array_equal(a.H, b.H) and a.iterations == b.iterations and a.converged == b.converged
    assert len(a.residuals) > CHUNK and np.array_equal(a.residuals, b.residuals)
    assert np.array_equal(np.asarray(a.X_mov_transformed), np.asarray(b.X_mov_transformed))
    for ra, rb in zip(a.records, b.records):
        assert ra["n_kept"] == rb["n_kept"] and ra["mean_res"] == rb["mean_res"] and ra["std_res"] == rb["std_res"]


@pytest.mark.gpu
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_residuals_past_the_scan_chunk(gpu, where):
    """The ordered compaction of the residuals by 9 M keep flags (more than two scan chunks), more
    than one chunk of them kept: the offset-sheet queries matched at the identity, normals
    (0, 0, 1), every seventh planarity below min_planarity, and a solve with all six parameters
    fixed, whose transform is the identity.  Each residual is then exactly the kept query's match
    distance, the construction's -off_z U."""
    X_fix, X_mov, off = _offset_sheet(where, 6)
    n = len(X_fix)
    flat = np.arange(n) % 7 != 3
    with _capi.Engine() as e:
        e.set_clouds(X_fix, X_mov)
        e.set_selected(None)
        z = np.zeros(n, dtype=np.float32)
        e.set_normals(z, z, np.ones(n, dtype=np.float32), np.where(flat, 0.9, 0.1).astype(np.float32))
        idx, d = e.match(np.eye(4))
        assert np.array_equal(idx, np.arange(n)) and np.array_equal(d, -off[:, 2] * U)
        keep, n_kept, _ = e.reject(0.3)  # |d - median| <= U: only the planarity rejects
        assert np.array_equal(keep, flat) and n_kept > CHUNK
        x, _, res, _, _ = e.solve(np.zeros(6), np.zeros(6), np.full(6, np.inf), 1.0, n_kept)
    assert np.array_equal(x, np.zeros(6))
    assert np.array_equal(res, d[flat]) and np.array_equal(res, -off[flat, 2] * U)


# ------------------------------------------------------------------------------ 2. the map at 9 M points
N_MAP, SJ_MAP = 3001 * 2999, 2999  # 8 999 999 points: not a multiple of 4096, three scan chunks
OCC = {"default": None, "occ1": 1.0}
_BIG = {}


def _sheet_map(where):
    if where not in _BIG:
        _BIG[where] = to_xyz(sheet_k(np.arange(N_MAP), SJ_MAP), ORIGINS[where])
    return _BIG[where]


def _map_engine(X, occ):
    e = _capi.Engine()
    if OCC[occ] is not None:
        e.set_option("grid_target_occupancy", OCC[occ])
    e.set_map(X)
    return e


def _scans(where, rng):
    """Four 50 x 50 tiles of the sheet with offsets, moved by a few units."""
    out = []
    for c in (1_000_000, 3_500_000, 5_200_000, 8_100_000):
        i, j = divmod(c, SJ_MAP)
        idx = ((i + np.arange(-25, 25))[:, None] * SJ_MAP + (j + np.arange(-25, 25))[None, :]).ravel()
        out.append(to_xyz(sheet_k(idx, SJ_MAP) + rng.integers(-1, 2, (len(idx), 3)) + [3, -2, 1], ORIGINS[where]))
    return out


def _registers_as_fresh(e, occ, where):
    """register_to_map on e's map (with and without the overlap filter) gives the bits of a fresh
    map of the same points."""
    scans = _scans(where, np.random.default_rng(3))
    X = e.get_map()
    params = e.run_params(0.0, 1.0, 100, _lsq(e))  # the sheet is rough at its own spacing: keep every planarity
    got = [e.register_to_map(scans, 1000, 10, params, **kw) for kw in (dict(max_overlap_distance=40 * U), dict())]
    with _map_engine(X, occ) as f:
        want = [f.register_to_map(scans, 1000, 10, params, **kw) for kw in (dict(max_overlap_distance=40 * U), dict())]
    for a, b in zip(got, want):
        assert np.array_equal(a.n_selected, b.n_selected)
        assert all(_same_bits(a[i], b[i]) for i in range(len(scans)))
    assert any(got[0][i].status == 0 for i in range(len(scans)))


@pytest.mark.gpu
@pytest.mark.parametrize("occ", sorted(OCC))
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_map_crop_past_the_scan_chunk(gpu, where, occ):
    X = _sheet_map(where)
    assert N_MAP > 2 * CHUNK and N_MAP % 4096
    rng = np.random.default_rng(4)
    # 300 centres: 260 spread over the sheet (among them the scans' tiles), 40 beside it
    ck = np.concatenate([sheet_k(np.linspace(0, N_MAP - 1, 256).astype(np.int64), SJ_MAP),
                         sheet_k([1_000_000, 3_500_000, 5_200_000, 8_100_000], SJ_MAP),
                         rng.integers(-3000, -500, (40, 3))])
    R = 400
    keep = sheet_crop_keep(N_MAP, SJ_MAP, ck, R)
    with _map_engine(X, occ) as e:
        removed = e.map_crop(to_xyz(ck, ORIGINS[where]), R * U)
        got = e.get_map()
        assert np.array_equal(got, X[keep]) and removed == N_MAP - keep.sum()
        assert np.flatnonzero(keep)[-1] > 2 * CHUNK  # kept points after the second chunk
        _registers_as_fresh(e, occ, where)


@pytest.mark.gpu
@pytest.mark.parametrize("occ", sorted(OCC))
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_map_thin_past_the_scan_chunk(gpu, where, occ):
    X = _sheet_map(where)
    v = 16 * U
    want = thin_fast(X, v)
    with _map_engine(X, occ) as e:
        removed = e.map_thin(v)
        assert np.array_equal(e.get_map(), want) and removed == N_MAP - len(want)
        _registers_as_fresh(e, occ, where)


def _insert_clouds(where, rng):
    """4.5 M points in 300 clouds (k_compact_bounds runs two blocks): near the sheet (taken voxels,
    and new ones beyond its edges), far outside with NaN rows, an empty cloud, and 297 pieces lifted
    by 40 units (new voxels, many points per voxel)."""
    o = ORIGINS[where]
    near = _near(rng, N_MAP, 2_000_000, SJ_MAP, o)[0]
    lifted = to_xyz(sheet_k(rng.integers(0, N_MAP, 2_000_000), SJ_MAP) + [0, 0, 40], o)
    far = to_xyz(rng.integers(-60_000, -20_000, (499_000, 3)), o)
    bad = near[:1000].copy()
    bad[::2, 1] = np.nan
    bad[1::2, 2] = np.inf
    mixed = np.concatenate([far, bad])[rng.permutation(500_000)]
    return [near, mixed, np.zeros((0, 3))] + np.array_split(lifted, 297)


@pytest.mark.gpu
@pytest.mark.parametrize("occ", sorted(OCC))
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_map_insert_past_the_scan_chunk(gpu, where, occ):
    X = _sheet_map(where)
    clouds = _insert_clouds(where, np.random.default_rng(5))
    assert sum(len(c) for c in clouds) > CHUNK and len(clouds) > 256
    v = 16 * U
    want, counts = insert_fast(X, clouds, v)
    assert counts[0] > 0 and counts[1] > 0 and (counts[3:] > 0).all()
    with _map_engine(X, occ) as e:
        added = e.map_insert(clouds, voxel_size=v)
        assert np.array_equal(added, counts) and e.n_map == len(want)
        assert np.array_equal(e.get_map(), want)
        _registers_as_fresh(e, occ, where)


@pytest.mark.gpu
@pytest.mark.parametrize("occ", sorted(OCC))
@pytest.mark.parametrize("where", sorted(ORIGINS))
def test_map_distances_past_the_scan_chunk(gpu, where, occ):
    """4.5 M query points over four clouds, and the first one again in 300 pieces: index, squared
    distance and n_within from the construction; with neighbors = 10 the plane distances of a sample equal estimate_normals on
    the same map points."""
    X = _sheet_map(where)
    o = ORIGINS[where]
    rng = np.random.default_rng(6)
    parts = [_near(rng, N_MAP, m, SJ_MAP, o) for m in (2_300_000, 1_900_000, 0, 300_000)]
    clouds = [p[0] for p in parts]
    far = to_xyz(rng.integers(-9000, -100, (300, 3)), o)
    clouds[3] = np.concatenate([clouds[3], far, np.full((7, 3), np.nan)])
    assert sum(len(c) for c in clouds) > CHUNK
    r = 2 * U  # r^2 = 4 U^2: every offset (|o|^2 <= 3) is within, every far point is not
    with _map_engine(X, occ) as e:
        idx, d2, _, _, n_within = e.map_distances(clouds, max_distance=r)
        for i, (P, src, o2) in enumerate(parts):
            m = len(P)
            assert np.array_equal(idx[i][:m], src), i
            assert np.array_equal(d2[i][:m], o2 * (U * U)), i
            assert n_within[i] == m, i
        assert (idx[3][-307:] == -1).all() and np.isinf(d2[3][-307:-7]).all() and np.isnan(d2[3][-7:]).all()
        # the first cloud in 300 pieces: the per-cloud counts come from two blocks of k_compact_bounds
        pieces = np.array_split(clouds[0], 300)
        idx_p, d2_p, _, _, n_p = e.map_distances(pieces, max_distance=r)
        assert np.array_equal(np.concatenate(idx_p), idx[0]) and np.array_equal(np.concatenate(d2_p), d2[0])
        assert np.array_equal(n_p, [len(P) for P in pieces])
        k = 10
        idx_n, d2_n, pd, pl, n_n = e.map_distances(clouds[:1], max_distance=r, neighbors=k)
        assert np.array_equal(idx_n[0], idx[0]) and np.array_equal(d2_n[0], d2[0]) and n_n[0] == n_within[0]
    sample = rng.choice(len(clouds[0]), 20_000, replace=False)
    uniq = np.unique(idx[0][sample])
    with _capi.Engine() as f:
        f.set_clouds(X, X[:1000])
        f.set_selected(uniq)
        nx, ny, nz, plan = f.estimate_normals(k)
    at = np.searchsorted(uniq, idx[0][sample])
    assert pl[0][sample].tobytes() == plan[at].tobytes()
    assert pd[0][sample].tobytes() == _plane(clouds[0][sample], X[idx[0][sample]], nx[at], ny[at], nz[at]).tobytes()


# ------------------------------------------------------------------------------ 3. thousands of pairs
N_PAIRS, SPLIT = 4096, 8
FAR = set(range(511, N_PAIRS, 512))  # movable clouds 1 km away: no overlap under the filter
_PAIRS = {}


def _many_pairs():
    """4096 ragged pairs (2 000 - 4 000 points per side) over 64 geometries, one prior per pair
    (degrees, the true transform plus noise)."""
    if "p" not in _PAIRS:
        rng = np.random.default_rng(7)
        geo = []
        for g in range(64):
            true = np.concatenate((rng.uniform(-1, 1, 3), rng.uniform(-0.2, 0.2, 3)))
            Xf = O.surface(4000, 90_000 + 2 * g, extent=30.0)
            Xm = O.transform_by_H(O.surface(4000, 90_001 + 2 * g, extent=30.0),
                                  np.linalg.inv(O.rbp_to_H(_observed_in_radians(true))))
            geo.append((Xf, Xm, true))
        pairs, rows = [], []
        for p in range(N_PAIRS):
            Xf, Xm, true = geo[p % 64]
            nf, nm = rng.integers(2000, 4001, 2)
            Xm = Xm[:nm] + ([1000.0, 0.0, 0.0] if p in FAR else 0.0)
            pairs.append((np.ascontiguousarray(Xf[:nf]), np.ascontiguousarray(Xm)))
            rows.append(true + np.concatenate((rng.normal(0, 0.05, 3), rng.normal(0, 0.03, 3))))
        _PAIRS["p"] = pairs, np.array(rows)
    return _PAIRS["p"]


def _outputs_bytes(out):
    X, R, log, T = out
    return np.asarray(X).tobytes(), R.tobytes(), b"".join(bytes(r) for r in log), T.tobytes()


ANGLE_DEG = 20.0
BATCH_CONFIGS = {"plain": {}, "overlap": dict(max_overlap_distance=1.0),
                 "mov_attr": dict(mov_neighbors=10, max_angle_rad=np.deg2rad(ANGLE_DEG))}


def _movable_cells():
    """Cells of the movable grids of the 4096 pairs at grid_target_occupancy 1, by test_grid_plan's
    statement of the batch policy (checked there against grid_plan.h)."""
    if "cells" not in _PAIRS:
        _PAIRS["cells"] = sum(int(np.prod(plan(Xm, "batch", target=1.0)["dims"])) for _, Xm in _many_pairs()[0])
    return _PAIRS["cells"]


@pytest.mark.gpu
@pytest.mark.parametrize("config", sorted(BATCH_CONFIGS))
def test_4096_pairs_in_one_call_equal_the_call_split(gpu, config):
    """4096 pairs in one register_batch call at grid_target_occupancy 1 against the same pairs 8
    per call: every field bit for bit, and for every 64th pair that registers its outputs and its
    result against sicp_register.  The movable grids' concatenated cell table and the 12 M overlap flags each span
    more than two scan chunks, and Kmax x n_pairs puts the match at 4 lanes.

    The pairs are registered once as built, then again ordered by their iteration counts, fastest
    first, and each pair must give the same bits in both calls.  In the second call every pair in
    k_gather_flags' first block has stopped while later pairs still run, so the loop's end depends
    on the stop flags gathered past that block."""
    pairs0, rows0 = _many_pairs()
    kw = BATCH_CONFIGS[config]
    obs0 = np.array([_observed_in_radians(r) for r in rows0])
    assert sum(len(Xf) for Xf, _ in pairs0) > 2 * CHUNK and _movable_cells() > 2 * CHUNK
    assert min(1000, min(len(Xf) for Xf, _ in pairs0)) * N_PAIRS > 65_536  # Kmax x n_pairs: the 4-lane match
    with _capi.Engine() as e:
        e.set_option("grid_target_occupancy", 1.0)
        params = e.run_params(0.3, 1.0, 100, _lsq(e))
        first = e.register_batch(pairs0, 1000, 10, params, observed=obs0, **kw)
        order = np.argsort([first[p].iterations for p in range(N_PAIRS)], kind="stable")
        pairs, obs, rows = [pairs0[i] for i in order], obs0[order], rows0[order]
        far = np.isin(order, sorted(FAR))
        big = e.register_batch(pairs, 1000, 10, params, observed=obs, **kw)
        assert np.array_equal(big.n_selected, first.n_selected[order])
        for k in range(N_PAIRS):
            assert _same_bits(big[k], first[order[k]]), f"{config}: pair {order[k]} at position {k}"
        iterations = np.array([big[k].iterations for k in range(N_PAIRS)])
        assert iterations[128:].max() > iterations[:128].max(), iterations
        sample = [int(k) for k in np.flatnonzero(~far)[::64]]  # a pair that failed has no outputs
        outs = e.batch_outputs(big)
        big_out = {k: _outputs_bytes(outs[k]) for k in sample}
        del outs
        for c0 in range(0, N_PAIRS, SPLIT):
            part = e.register_batch(pairs[c0:c0 + SPLIT], 1000, 10, params, observed=obs[c0:c0 + SPLIT], **kw)
            assert np.array_equal(part.n_selected, big.n_selected[c0:c0 + SPLIT]), c0
            for i in range(SPLIT):
                assert _same_bits(part[i], big[c0 + i]), f"{config}: pair {order[c0 + i]} at position {c0 + i}"
            mine = [k for k in sample if c0 <= k < c0 + SPLIT]
            if mine:
                part_out = e.batch_outputs(part)
                for k in mine:
                    assert _outputs_bytes(part_out[k - c0]) == big_out[k], f"{config}: outputs at position {k}"
        status = np.array([big[k].status for k in range(N_PAIRS)])
        if "max_overlap_distance" in kw:
            assert (status[far] == _capi.SICP_ERR_NO_OVERLAP).all()
        assert (status[~far] == 0).all(), order[~far][status[~far] != 0]
        reg_kw = dict(max_overlap_distance=kw.get("max_overlap_distance", np.inf))
        if "mov_neighbors" in kw:
            reg_kw.update(mov_neighbors=kw["mov_neighbors"], max_angle_between_normals=ANGLE_DEG)
        for k in sample:
            Xf, Xm = pairs[k]
            r = sb.register(Xf, Xm, engine=e, want_normals=False, rbp_observed_values=rows[k], **reg_kw)
            _same_as_register(big[k], int(big.n_selected[k]), r, f"{config}: pair {order[k]}")


# ------------------------------------------------------------------------------ 4. the 32-bit map limit
N_LIM, SJ_LIM = 2 ** 27 + 4097, 11_586
N_SCANS_LIM = ((1 << 32) - 1) // N_LIM  # 31: n_scans x n_map just below 2^32
# device bytes the test needs free: the engine held 23.8 GiB after the registrations (map, grid,
# masks and the 3.9 G-entry survivor list) on an H100 80GB HBM3 at a 700 W power limit; the crop
# adds its flags, scan and the kept points
PEAK_LIM = 28 << 30


def _sheet_inplace(n, SJ, origin, rows=1024):
    """to_xyz(sheet_k(arange(n), SJ), origin) written row block by row block into one array (the
    same operations, so the same bits, without whole-size temporaries)."""
    X = np.empty((n, 3))
    o = np.asarray(origin, dtype=np.float64)
    for s in range(0, n, rows * SJ):
        k = sheet_k(np.arange(s, min(n, s + rows * SJ)), SJ)
        X[s:s + len(k)] = o[None, :] + k * U
    return X


@pytest.mark.gpu
def test_map_filter_at_the_32_bit_limit(gpu):
    """A sheet map of 2^27 + 4097 points and 31 scans whose overlap filter keeps most of the map
    for each of them: the mask rows, their popcount scan and the survivor offsets reach 31 x 2^27
    (about 4.2e9 of the uint32 range).  The 31-scan call equals the scans one per call bit for bit,
    batch outputs included; 32 scans are refused before any device work; a crop scans the map's
    2^27 + 4097 keep flags.  Peak device memory: 23.8 GiB held by the engine after the
    registrations (see PEAK_LIM); the test skips, saying so, when less than PEAK_LIM is free."""
    free = torch.cuda.mem_get_info()[0]
    if free < PEAK_LIM:
        pytest.skip(f"needs {PEAK_LIM / 2 ** 30:.0f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    o = ORIGINS["utm"]
    X = _sheet_inplace(N_LIM, SJ_LIM, o)
    assert np.array_equal(X[-5:], to_xyz(sheet_k(np.arange(N_LIM - 5, N_LIM), SJ_LIM), o))
    rng = np.random.default_rng(8)
    # 31 scans of 20 000 points spread over the whole sheet: 0.6 m reaches most map points
    scans = [_near(rng, N_LIM, 20_000, SJ_LIM, o)[0] + [2 * U, -U, 0.0] for _ in range(N_SCANS_LIM + 1)]
    assert N_SCANS_LIM == 31 and N_SCANS_LIM * N_LIM < 2 ** 32 <= (N_SCANS_LIM + 1) * N_LIM
    with _capi.Engine() as e:
        free0 = torch.cuda.mem_get_info()[0]
        e.set_map(X)
        params = e.run_params(0.3, 1.0, 20, _lsq(e))
        kw = dict(max_overlap_distance=0.6)
        big = e.register_to_map(scans[:N_SCANS_LIM], 1000, 10, params, **kw)
        big_out = [_outputs_bytes(x) for x in e.batch_outputs(big)]
        n_sel = big.n_selected.copy()
        assert (n_sel == 1000).all()
        for i, S in enumerate(scans[:N_SCANS_LIM]):
            one = e.register_to_map([S], 1000, 10, params, **kw)
            assert one.n_selected[0] == n_sel[i] and _same_bits(one[0], big[i]), f"scan {i}"
            assert _outputs_bytes(e.batch_outputs(one)[0]) == big_out[i], f"outputs of scan {i}"
        with pytest.raises(_capi.SicpError) as ei:
            e.register_to_map(scans, 1000, 10, params, **kw)
        assert ei.value.code == _capi.SICP_ERR_BAD_ARG
        assert e.n_map == N_LIM and np.array_equal(e.get_map(), X)
        ck = np.concatenate([sheet_k(np.linspace(0, N_LIM - 1, 300).astype(np.int64), SJ_LIM),
                             rng.integers(-3000, -500, (20, 3))])
        R = 200
        keep = sheet_crop_keep(N_LIM, SJ_LIM, ck, R)
        removed = e.map_crop(to_xyz(ck, o), R * U)
        assert removed == N_LIM - keep.sum() and np.flatnonzero(keep)[-1] > 2 ** 27
        assert np.array_equal(e.get_map(), X[keep])
        print(f"32-bit map: device memory held by the engine {(free0 - torch.cuda.mem_get_info()[0]) / 2 ** 30:.1f} GiB")
