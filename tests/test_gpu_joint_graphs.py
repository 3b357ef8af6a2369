"""The sparse joint solve (joint_solver 1, DESIGN.md §6.11) and the dense one on the edge graphs of
real surveys, beyond the band graphs of tests/test_gpu_joint_sparse.py: a 2-D block of tiles with
8-neighbour edges, the same block with anchors inside it, a star around one wide hub scan, the
complete graph of repeated scans of one site, several such pieces in one call, and the block with
reversed and duplicated edges.  Each runs through both solves, which must agree (iterations,
convergence and kept counts exact, poses and statistics within 1e-9); the star also in lock-step
with the oracle.  Past the dense solve's cap, the first iteration's solve is checked by its
backward error against the system assembled exactly from the oracle's per-edge sums."""
import time

import numpy as np
import pytest

from oracle import joint_oracle as J
from simpleicp_b200 import _capi

from test_gpu_joint import _lockstep, strip
from test_gpu_joint_sparse import _assert_agree, _joint

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    e = _capi.Engine(0)
    yield e
    e.close()


def _surface(x, y):
    return 0.05 * x + 0.03 * y + 2 * np.sin(2 * np.pi * x / 25) * np.cos(2 * np.pi * y / 40)


def _scan(rng, x0, y0, size, n_points, start=True):
    """One scan of the C3 surface of strip() over [x0, x0 + size) x [y0, y0 + size), in its own
    frame as strip() makes it (centred on its patch, turned by up to 1 degree, moved by up to
    0.3 m); its true pose and its start pose (perturbed by 0.3 degrees and 5 cm when `start`)."""
    x = rng.uniform(x0, x0 + size, n_points)
    y = rng.uniform(y0, y0 + size, n_points)
    P = np.column_stack((x, y, _surface(x, y) + rng.normal(0, 0.01, n_points)))
    T = J.rigid_from_x(np.concatenate((np.deg2rad(rng.uniform(-1, 1, 3)), rng.uniform(-0.3, 0.3, 3))))
    T[:3, 3] += (x0 + size / 2, y0 + size / 2, 0.0)
    Ti = np.linalg.inv(T)
    dH = J.rigid_from_x(np.concatenate((np.deg2rad(rng.normal(0, 0.3, 3)), rng.normal(0, 0.05, 3))))
    return np.ascontiguousarray(P @ Ti[:3, :3].T + Ti[:3, 3]), T, (T @ dH if start else T)


def tiles(nx, ny, n_points, seed=21, fixed=(0,)):
    """nx x ny tiles of one surface, tile k = i ny + j over x in [10 i, 10 i + 26), y in
    [10 j, 10 j + 26), each scan in its own frame; the fixed tiles start at their true pose.
    Returns scans, truth, start poses."""
    rng = np.random.default_rng(seed)
    fx = set(fixed)
    out = [_scan(rng, 10.0 * (k // ny), 10.0 * (k % ny), 26.0, n_points, k not in fx) for k in range(nx * ny)]
    return [o[0] for o in out], np.array([o[1] for o in out]), np.array([o[2] for o in out])


def block_edges(nx, ny):
    """The 8-neighbour pairs of an nx x ny block of tiles: parallel lines, cross lines and both
    diagonals, each pair once, the smaller tile first."""
    E = []
    for i in range(nx):
        for j in range(ny):
            k = i * ny + j
            for di, dj in ((1, 0), (0, 1), (1, 1), (1, -1)):
                if 0 <= i + di < nx and 0 <= j + dj < ny:
                    E.append((k, (i + di) * ny + j + dj))
    return np.array(E)


def star(n_sat=99, hub_points=60_000, sat_points=3_000, seed=23):
    """One hub scan over [0, 116)^2 (cloud 0) and n_sat satellite tiles of a 10 x 10 layout (clouds
    1 ..), edges hub-satellite only, the first half written (hub, sat) and the rest (sat, hub)."""
    rng = np.random.default_rng(seed)
    hub = _scan(rng, 0.0, 0.0, 116.0, hub_points)
    sats = [_scan(rng, 10.0 * (k // 10), 10.0 * (k % 10), 26.0, sat_points) for k in range(n_sat)]
    scans = [hub[0]] + [s[0] for s in sats]
    truth = np.array([hub[1]] + [s[1] for s in sats])
    H0 = np.array([hub[2]] + [s[2] for s in sats])
    edges = np.array([(0, s) if s <= n_sat // 2 else (s, 0) for s in range(1, n_sat + 1)])
    return scans, truth, H0, edges


def complete(n, n_points=2_000, seed=25):
    """n scans of the one patch [0, 26)^2 and all n (n - 1) / 2 pairs between them."""
    rng = np.random.default_rng(seed)
    out = [_scan(rng, 0.0, 0.0, 26.0, n_points) for _ in range(n)]
    edges = np.array([(i, j) for i in range(n) for j in range(i + 1, n)])
    return [o[0] for o in out], np.array([o[1] for o in out]), np.array([o[2] for o in out]), edges


def _both(eng, scans, edges, fixed, H0, **kw):
    """The problem through the dense and the sparse solve; both must succeed and agree."""
    dense = _joint(eng, 0, scans, edges, fixed, H0, **kw)
    sparse = _joint(eng, 1, scans, edges, fixed, H0, **kw)
    assert all(o.status == 0 for o in dense[1])
    _assert_agree(dense, sparse)
    return dense, sparse


# ------------------------------------------------------------------------------- the graphs
def test_block_15x17_8_neighbours_one_fixed_corner(eng):
    """254 free clouds: top separators of 15 to 20 clouds (about 100 columns) over structs of
    dozens of clouds, many children per separator, structs scattered over the panel's rows."""
    scans, truth, H0 = tiles(15, 17, 3_000)
    _both(eng, scans, block_edges(15, 17), (0,), H0)


def test_block_with_a_fixed_column_and_every_fifth_tile_fixed(eng):
    """Anchors inside the graph: the fixed column i = 7 splits one call into independent subtrees,
    and every edge to a fixed tile reaches only a diagonal block (the bit 2 e + 1)."""
    fixed = sorted({7 * 17 + j for j in range(17)} | set(range(0, 255, 5)))
    scans, truth, H0 = tiles(15, 17, 3_000, seed=22, fixed=fixed)
    _both(eng, scans, block_edges(15, 17), tuple(fixed), H0)


def test_star_of_99_satellites_around_one_hub(eng):
    """One free hub, 98 free satellites and one fixed: one separator (the hub) with 98 children,
    the update loop over 98 descendants, both edge orientations on and off the diagonal."""
    scans, truth, H0, edges = star()
    H0[5] = truth[5]
    _both(eng, scans, edges, (5,), H0)


def test_complete_graph_of_64_scans_of_one_site(eng):
    """2 016 pairs, one fixed: one supernode, a 379 x 378 panel, whose column and row loops wrap
    the 256 threads of the block."""
    scans, truth, H0, edges = complete(64)
    H0[0] = truth[0]
    _both(eng, scans, edges, (0,), H0)


def _pieces():
    """A block, a star and a complete graph in one call.  Every piece starts with the same two
    clouds (tiles (0, 0), fixed, and (1, 0)) and the same first edge between them, so the common
    centre c_w of a piece's own call is the joint call's.  The block adds two free clouds whose
    only edges go to fixed clouds (supernodes with an empty struct)."""
    rng = np.random.default_rng(31)
    base = [_scan(rng, 0.0, 0.0, 26.0, 3_000, False), _scan(rng, 10.0, 0.0, 26.0, 3_000)]
    parts = []
    # the block: the 4 x 4 tiles, tile (3, 3) fixed too, and two lonely free clouds
    sc, tr, h0 = tiles(4, 4, 3_000, seed=32, fixed=(0, 15))
    for k, (i, j) in enumerate(((0, 0), (1, 0))):
        sc[4 * i + j], tr[4 * i + j], h0[4 * i + j] = base[k]
    lone = [_scan(rng, 2.0, 2.0, 26.0, 3_000), _scan(rng, 28.0, 28.0, 26.0, 3_000)]
    E = [(0, 4)] + [tuple(e) for e in block_edges(4, 4) if tuple(e) != (0, 4)] + [(0, 16), (17, 15)]
    parts.append((sc + [lone[0][0], lone[1][0]], np.concatenate((tr, [lone[0][1], lone[1][1]])),
                  np.concatenate((h0, [lone[0][2], lone[1][2]])), np.array(E), (0, 15)))
    # the star: a hub over [0, 56)^2 and the 4 x 4 tiles as satellites
    hub = _scan(rng, 0.0, 0.0, 56.0, 30_000)
    sats = [_scan(rng, 10.0 * (k // 4), 10.0 * (k % 4), 26.0, 3_000) for k in range(16)]
    sats[0], sats[4] = base   # tiles (0, 0) and (1, 0)
    order = [0, 4] + [k for k in range(16) if k not in (0, 4)]
    sc = [sats[k][0] for k in order] + [hub[0]]
    tr = np.array([sats[k][1] for k in order] + [hub[1]])
    h0 = np.array([sats[k][2] for k in order] + [hub[2]])
    E = [(0, 1)] + [(16, s) if s % 2 else (s, 16) for s in range(16)]
    parts.append((sc, tr, h0, np.array(E), (0,)))
    # the complete graph: the two base tiles and 14 scans of the patch of tile (0, 0)
    c = complete(14, 3_000, seed=33)
    sc = [base[0][0], base[1][0]] + c[0]
    tr = np.concatenate(([base[0][1], base[1][1]], c[1]))
    h0 = np.concatenate(([base[0][2], base[1][2]], c[2]))
    E = [(i, j) for i in range(16) for j in range(i + 1, 16)]
    parts.append((sc, tr, h0, np.array(E), (0,)))
    return parts


def test_pieces_in_one_call_equal_each_piece_alone(eng):
    """Several roots, one of them per piece, and supernodes with nt = 0; one unused (None) cloud.
    Fixed iterations (min_change = 0 never stops), so that the pieces' counts cannot part."""
    parts = _pieces()
    scans, H0, edges, fixed, at = [], [], [], [], 0
    for sc, tr, h0, E, fx in parts:
        scans += list(sc)
        H0.append(h0)
        edges.append(E + at)
        fixed += [f + at for f in fx]
        at += len(sc)
    scans.append(None)
    H0 = np.concatenate(H0 + [2.0 * np.eye(4)[None]])
    edges = np.concatenate(edges)
    kw = dict(max_iterations=4, min_change=0.0)
    H, out, outputs = _joint(eng, 1, scans, edges, tuple(fixed), H0, **kw)
    assert all(o.status == 0 and o.iterations == 4 for o in out)
    assert np.array_equal(H[-1], H0[-1])
    at, ea = 0, 0
    for sc, tr, h0, E, fx in parts:
        Hs, outs, os_ = _joint(eng, 0, sc, E, fx, h0, **kw)
        assert np.abs(H[at:at + len(sc)] - Hs).max() < 1e-9
        for o, p, (_, _, la, _), (_, _, lb, _) in zip(out[ea:ea + len(E)], outs, outputs[ea:ea + len(E)], os_):
            assert p.status == 0 and o.iterations == p.iterations
            assert [r.n_kept for r in la[:4]] == [r.n_kept for r in lb[:4]]
        at, ea = at + len(sc), ea + len(E)


def test_block_with_reversed_and_duplicated_edges(eng):
    """The 15 x 17 block with every third edge written (b, a) and every seventh given twice: the
    block lists of joint_sparse_ids with two edges and both orientations."""
    scans, truth, H0 = tiles(15, 17, 3_000)
    E = []
    for e, (a, b) in enumerate(block_edges(15, 17)):
        E.append((b, a) if e % 3 == 1 else (a, b))
        if e % 7 == 3:
            E.append(E[-1])
    _both(eng, scans, np.array(E), (0,), H0)


def test_relabelled_block_gives_the_same_poses(eng):
    """The 15 x 17 block with its clouds and its edges after the first permuted (the first fixes
    the common centre c_w): another ordering of the same system, so only rounding may differ."""
    scans, truth, H0 = tiles(15, 17, 3_000)
    edges = block_edges(15, 17)
    rng = np.random.default_rng(8)
    new = rng.permutation(len(scans))
    old = np.argsort(new)
    order = np.concatenate(([0], 1 + rng.permutation(len(edges) - 1)))
    H, out, _ = _joint(eng, 1, scans, edges, (0,), H0)
    Hp, outp, _ = _joint(eng, 1, [scans[i] for i in old], new[edges[order]], (int(new[0]),), H0[old])
    assert np.abs(Hp[new] - H).max() < 1e-9
    assert [o.n_kept for o in outp] == [out[e].n_kept for e in order]


def test_star_two_calls_give_the_same_bits(eng):
    scans, truth, H0, edges = star()
    H, out, o = _joint(eng, 1, scans, edges, (5,), H0)
    H2, out2, o2 = _joint(eng, 1, scans, edges, (5,), H0)
    assert np.array_equal(H, H2)
    assert all(bytes(a) == bytes(b) for a, b in zip(out, out2))
    for (X, r, lg, T), (X2, r2, lg2, T2) in zip(o, o2):
        assert np.array_equal(X, X2) and np.array_equal(r, r2) and np.array_equal(T, T2)
        assert all(bytes(a) == bytes(b) for a, b in zip(lg, lg2))


def test_star_lockstep_with_the_oracle(eng):
    """Three iterations of the star in lock-step with the oracle (the device's normals handed
    over): every kept count exact, the poses within 1e-10 (measured 3.8e-13, H100)."""
    scans, truth, H0, edges = star()
    eng.set_option("joint_solver", 1)
    try:
        H, out, logs, ref = _lockstep(eng, scans, H0, edges, (5,), max_iterations=3)
    finally:
        eng.set_option("joint_solver", 0)
    assert all(o.status == 0 and o.iterations == len(ref.log) for o in out)
    for it, row in enumerate(ref.log):
        assert [lg[it].n_kept for lg in logs] == [r.n_kept for r in row], it
    gap = np.abs(H - ref.H).max()
    print(f"star lock-step: |H - H_oracle| = {gap:.2e}")
    assert gap < 1e-10


# ------------------------------------------------------------------------------- backward error
def _increments(H0, H1, free):
    """Each free cloud's first increment in the kernel's variables: (omega, u) about the origin
    o_c of its start pose, from H1 H0^-1 = dH(omega, t) (the oracle's rigid_from_x inverted) and
    t = u - omega x o_c."""
    R0, p0 = H0[free, :3, :3], H0[free, :3, 3]
    R1, p1 = H1[free, :3, :3], H1[free, :3, 3]
    R = R1 @ np.transpose(R0, (0, 2, 1))
    t = p1 - np.einsum("cij,cj->ci", R, p0)
    w = np.column_stack((np.arctan2(-R[:, 1, 2], R[:, 2, 2]), np.arcsin(np.clip(R[:, 0, 2], -1, 1)),
                         np.arctan2(-R[:, 0, 1], R[:, 0, 0])))
    return np.column_stack((w, t + np.cross(w, p0)))


def _skew(v):
    Z = np.zeros(v.shape[:-1] + (3, 3), dtype=v.dtype)
    Z[..., 0, 1], Z[..., 0, 2], Z[..., 1, 2] = -v[..., 2], v[..., 1], -v[..., 0]
    Z[..., 1, 0], Z[..., 2, 0], Z[..., 2, 1] = v[..., 2], -v[..., 1], v[..., 0]
    return Z


def _backward_error(sums, edges, H0, y):
    """eta = |b - M y|_inf / (|M|_inf |y|_inf + |b|_inf) for the first iteration's joint system M y
    = b in the kernel's variables, assembled from the oracle's per-edge sums: edge e = (a, b)
    with T_a = (R, p) gives xi_e = G_b y_b - G_a y_a, G_c = [[R^T, 0], [-R^T [p - o_c]x, R^T]] with
    metre levers p - o_c, and M = sum_e J_e^T N_e J_e, b = sum_e J_e^T g_e over the edges with at
    least 6 kept rows.  M y is summed edge by edge in np.longdouble; |M|_inf from M assembled in
    float64."""
    from scipy import sparse

    slot = {c: k for k, c in enumerate(sums.free)}
    F = len(sums.free)
    use = sums.n_kept >= 6
    E = np.asarray(edges)[use]
    N, g, Ta = sums.N[use], sums.g[use], sums.T_a[use]
    ld = np.longdouble
    R, p = Ta[:, :3, :3], Ta[:, :3, 3]
    Y = np.vstack((np.asarray(y, dtype=ld).reshape(F, 6), np.zeros((1, 6), dtype=ld)))  # row F: fixed
    ia = np.array([slot.get(int(a), F) for a in E[:, 0]])
    ib = np.array([slot.get(int(b), F) for b in E[:, 1]])
    G = []
    for ic, c in ((ia, E[:, 0]), (ib, E[:, 1])):
        Gc = np.zeros((len(E), 6, 6))
        Rt = np.transpose(R, (0, 2, 1))
        Gc[:, :3, :3] = Rt
        Gc[:, 3:, 3:] = Rt
        Gc[:, 3:, :3] = -Rt @ _skew(p - H0[c, :3, 3])
        G.append(Gc)
    Ga, Gb = G
    xi = np.einsum("eij,ej->ei", Gb.astype(ld), Y[ib]) - np.einsum("eij,ej->ei", Ga.astype(ld), Y[ia])
    z = np.einsum("eij,ej->ei", N.astype(ld), xi) - g.astype(ld)
    res = np.zeros((F + 1, 6), dtype=ld)
    np.add.at(res, ib, np.einsum("eji,ej->ei", Gb.astype(ld), z))
    np.add.at(res, ia, -np.einsum("eji,ej->ei", Ga.astype(ld), z))
    bvec = np.zeros((F + 1, 6))
    np.add.at(bvec, ib, np.einsum("eji,ej->ei", Gb, g))
    np.add.at(bvec, ia, -np.einsum("eji,ej->ei", Ga, g))
    rows, cols, vals = [], [], []
    r6, c6 = np.repeat(np.arange(6), 6), np.tile(np.arange(6), 6)
    for (i1, G1, s1) in ((ia, Ga, -1.0), (ib, Gb, 1.0)):
        for (i2, G2, s2) in ((ia, Ga, -1.0), (ib, Gb, 1.0)):
            ok = (i1 < F) & (i2 < F)
            B = s1 * s2 * np.transpose(G1, (0, 2, 1)) @ N @ G2
            rows.append((6 * i1[ok, None] + r6).ravel())
            cols.append((6 * i2[ok, None] + c6).ravel())
            vals.append(B[ok].reshape(-1, 36).ravel())
    M = sparse.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(6 * F, 6 * F))
    norm_M = float(np.abs(M).sum(axis=1).max())
    yv = np.asarray(y).ravel()
    return float(np.abs(res[:F]).max() / (norm_M * np.abs(yv).max() + np.abs(bvec[:F]).max()))


def _block(n):
    scans, truth, H0 = tiles(n, n, 1_000, seed=40 + n)
    return scans, truth, H0, block_edges(n, n)


BACKWARD = {"block_32x32": lambda: _block(32), "block_64x64": lambda: _block(64),
            "strip_2048": lambda: strip(2048, 2_000, 6_400), "strip_4096": lambda: strip(4096, 2_000, 12_800)}


def _oracle_sums(eng, scans, edges, H0):
    """The oracle's first-iteration sums with the device's float32 normals of every edge's
    selection (as _device_normals hands them over), per edge in the order of `edges`.  The oracle
    runs over the edges sorted by fixed cloud, so that each cloud is uploaded and gridded for the
    normal search once rather than once per edge (12 800 edges on the 4096-cloud strip)."""
    order = np.argsort(edges[:, 0], kind="stable")
    cur = [-1]

    def normals(k, idx):
        if idx.size == 0:  # an edge without overlap
            return np.zeros((0, 3)), np.zeros(0)
        a = int(edges[order[k], 0])
        if cur[0] != a:
            eng.set_clouds(scans[a], scans[a][:10])
            cur[0] = a
        eng.set_selected(idx)
        nx, ny, nz, pl = eng.estimate_normals(10)
        return np.column_stack((nx, ny, nz)), pl.copy()

    s = J.first_iteration_sums(scans, edges[order], fixed=(0,), H0=H0, max_overlap_distance=1.0, normals=normals)
    back = np.argsort(order)
    return J.EdgeSums(N=s.N[back], g=s.g[back], n_kept=s.n_kept[back], T_a=s.T_a[back], free=s.free)


@pytest.mark.parametrize("problem", list(BACKWARD))
def test_first_iteration_backward_error(eng, problem):
    """One iteration past the dense cap: 32 x 32 and 64 x 64 blocks of 1 000 points per tile
    (F = 1023 and 4095; the 64 x 64 block's three top separators hold 90, 63 and 43 clouds, panels
    of 540, 378 and 258 columns that take 119, 77 and 49 descendant updates) and the 2048- and
    4096-cloud strips of DESIGN.md §6.11 with 2 000 points per cloud.  The kept counts equal the
    oracle's (given the device's normals), and the increment recovered from the device's poses
    solves the system assembled exactly from the oracle's per-edge sums to a backward error eta at
    the floor of that recovery, eps_rec = 2^-52 max_c |p_c| / |y|_inf (the poses' translations run
    to kilometres on the strips).  Being a backward error, eta does not grow with the conditioning
    of the strip, so it separates the solve from §6.9's rule.  Measured (H100 80GB HBM3):

    problem       eta      eps_rec  first step |y|_inf  max |p_c|
    block_32x32   1.6e-15  1.4e-13  0.73                457 m
    block_64x64   3.3e-15  2.5e-13  0.80                910 m
    strip_2048    8.6e-17  2.0e-14  45 m                4.1 km
    strip_4096    2.9e-18  1.1e-15  1.6e3 m             8.2 km

    The bound max(1e-12, 10 eps_rec) is at least 300 times each."""
    scans, truth, H0, edges = BACKWARD[problem]()
    t0 = time.perf_counter()
    H, out, outputs = _joint(eng, 1, scans, edges, (0,), H0, max_iterations=1)
    status = np.array([o.status for o in out])
    parked = (status == _capi.SICP_ERR_NO_OVERLAP) | (status == _capi.SICP_ERR_TOO_FEW_CORR)
    assert np.all((status == 0) | parked), np.unique(status, return_counts=True)
    sums = _oracle_sums(eng, scans, edges, H0)
    # an edge without overlap or with too few correspondences is parked by the device and takes
    # no part in the oracle's system either
    ok = status == 0
    assert np.all(sums.n_kept[~ok] < 6), (status[~ok], sums.n_kept[~ok])
    assert [o[2][0].n_kept for o, k in zip(outputs, ok) if k] == list(sums.n_kept[ok])
    y = _increments(H0, H, np.array(sums.free))
    eta = _backward_error(sums, edges, H0, y)
    pmax = max(np.linalg.norm(H0[:, :3, 3], axis=1).max(), np.linalg.norm(H[:, :3, 3], axis=1).max())
    eps_rec = 2.0 ** -52 * pmax / np.abs(y).max()
    print(f"{problem}: eta {eta:.2e}, eps_rec {eps_rec:.2e}, |y|_inf {np.abs(y).max():.3g}, "
          f"max |p| {pmax:.0f} m, {int(status.size - ok.sum())} parked, {time.perf_counter() - t0:.0f} s")
    assert eta <= max(1e-12, 10.0 * eps_rec)
