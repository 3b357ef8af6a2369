"""Run under compute-sanitizer (GPU): one small registration through every engine path —
fused register, stage-by-stage, linearised variant, brute-force engine, K > 4096 (cooperative
first iteration, barrier-free kernel with several blocks afterwards), the three k-NN kernels,
2 / 4 / 16 lanes per query, movable-side attributes, the batched engine — so memcheck sees all
kernels.  python tools/sanitize_probe.py"""
import sys
from pathlib import Path
import numpy as np
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from bench import make_pair

X_fix, X_mov, H_true = make_pair(60_000, 0)
with _capi.Engine() as e:
    a = sb.register(X_fix, X_mov, correspondences=2000, engine=e, want_normals=False)       # fused, single block
    b = sb.register(X_fix, X_mov, correspondences=2000, engine=e, want_normals=True)        # staged
    assert np.array_equal(a.H, b.H)
    c = sb.register(X_fix, X_mov, correspondences=6000, engine=e, want_normals=False)       # cooperative path
    d = sb.register(X_fix, X_mov, correspondences=2000, engine=e, max_overlap_distance=2.0, want_normals=False)
    e.set_option("nn_engine", _capi.NN_BRUTE)
    f = sb.register(X_fix, X_mov, correspondences=500, engine=e, want_normals=True)
    e.set_option("nn_engine", _capi.NN_AUTO)
    e.set_option("grid_max_rings", 1)                                                       # forces the TMA fallback
    g = sb.register(X_fix, X_mov, correspondences=2000, engine=e, want_normals=True)
    e.set_option("grid_max_rings", 8)
    assert np.linalg.norm(g.H - b.H) < 1e-9
    l = sb.simpleicp_linearized(X_fix, X_mov, correspondences=6000, engine=e)
    # round 2: k-NN kernel variants, lanes per query, cooperative-only loop, movable attributes
    for mode in (0, 1, 2):
        e.set_option("knn_coop", mode)
        h = sb.register(X_fix, X_mov, correspondences=3000, engine=e, want_normals=True)
        assert np.linalg.norm(h.H - H_true) < 5e-2
    e.set_option("knn_coop", -1)
    for mg in (2, 4, 16):
        e.set_option("match_group", mg)
        h = sb.register(X_fix, X_mov, correspondences=6000, engine=e, want_normals=False)
        assert np.linalg.norm(h.H - c.H) < 1e-9
    e.set_option("match_group", 0)
    e.set_option("fused", 0)
    h = sb.register(X_fix, X_mov, correspondences=6000, engine=e, want_normals=False)
    assert np.linalg.norm(h.H - c.H) < 1e-9
    e.set_option("fused", 1)
    pc = sb.PointCloud(X_mov[:20000], columns=["x", "y", "z"])
    pc.estimate_normals(10)
    mov = tuple(pc[col].to_numpy().astype(np.float32) for col in ("nx", "ny", "nz", "planarity"))
    m = sb.register(X_fix, X_mov[:20000], correspondences=6000, engine=e, mov_normals=mov, max_angle_between_normals=20.0)
    assert np.linalg.norm(m.H - H_true) < 5e-2
pairs = [sb.synthetic.c5_pair(i, 20_000) for i in range(4)]
tab = sb.simpleicp_batch([(p[0], p[1]) for p in pairs], engine="batched", correspondences=500)
assert np.isfinite(tab).all()
# overlap filter + a prior per pair in the batch, one pair without any overlap
ov = [(p[0][p[0][:, 0] < 20], p[1][p[1][:, 0] > 10]) for p in pairs] + [(pairs[0][0], pairs[0][1] + 1e4)]
tab_o = sb.simpleicp_batch(ov, engine="batched", correspondences=500, max_overlap_distance=0.5,
                           rbp_observed_values=np.zeros((len(ov), 6)), on_error="nan")
assert np.isfinite(tab_o[:-1]).all() and tab_o[-1, 16] == -_capi.SICP_ERR_NO_OVERLAP
# pairs drawn from shared clouds: a self pair, a cloud in both roles, an unreferenced NULL cloud,
# with the overlap filter and movable normals on (every shared-write hazard of the batch reached)
with _capi.Engine() as e:
    prm = e.run_params(0.3, 1.0, 20, e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0))
    sh = [pairs[0][0], None, pairs[0][1], pairs[1][1]]
    rs = e.register_pairs(sh, [[0, 0], [0, 2], [2, 3], [3, 0], [2, 0]], 500, 10, prm, max_overlap_distance=0.5,
                          mov_neighbors=10)
    outs = e.batch_outputs(rs)
    assert rs[1].status == 0 and outs[1] is not None
# map insert: with H (a NaN point, an empty cloud, a cloud at an odd point offset), without H, and
# one that adds nothing
with sb.Map(X_fix[:30_000]) as mp:
    ins = [X_mov[:1001].copy(), np.zeros((0, 3)), X_mov[1001:3000]]
    ins[0][5, 1] = np.nan
    k1 = mp.insert(ins, np.stack([H_true, np.eye(4), H_true]), voxel_size=0.05)
    k2 = mp.insert([X_mov[3000:9000] + 0.01], voxel_size=0.2)
    k3 = mp.insert([mp.points()[:500]], voxel_size=0.05)
    assert k1.sum() > 0 and k2.sum() > 0 and k3.sum() == 0 and mp.n_points == 30_000 + k1.sum() + k2.sum()
    # map distances: with H and normals (the same odd-offset, NaN and empty clouds), without either,
    # and a cloud entirely beyond the bound
    d1 = mp.distances(ins, np.stack([H_true, np.eye(4), H_true]), max_distance=0.5, neighbors=10)
    d2 = mp.distances([X_mov[3000:9000]], max_distance=0.2)
    d3 = mp.distances([X_mov[:100] + 1e4], max_distance=0.5, neighbors=30)
    assert d1[0].n_within > 0 and d1[1].n_within == 0 and d2[0].n_within > 0 and d3[0].n_within == 0
    # map crop and thin: several centres (more than one shared-memory chunk), one that removes
    # nothing, one that would remove everything (refused, the map unchanged), and a thin
    n0 = mp.n_points
    cen = np.concatenate([mp.points()[::97][:300], np.full((3, 3), 1e4)])
    c1 = mp.crop(cen, radius=0.3)
    c2 = mp.crop(cen[:5], radius=1e4)
    try:
        mp.crop(np.full(3, 1e5), radius=1.0)
        raise AssertionError("a crop that keeps nothing must be refused")
    except _capi.SicpError as err:
        assert err.code == _capi.SICP_ERR_NO_OVERLAP
    t1 = mp.thin(voxel_size=0.1)
    assert c1 > 0 and c2 == 0 and t1 > 0 and mp.n_points == n0 - c1 - t1
    # map carve: with H and default origins (the NaN point, the empty and odd-offset clouds), and with
    # explicit origins that remove nothing
    n1 = mp.n_points
    org = np.array([[2.0, 2.0, 5.0], [0.0, 0.0, 0.0], [40.0, 60.0, 3.0]])
    v1 = mp.carve(ins, np.stack([H_true, np.eye(4), H_true]), radius=0.1, margin=0.2)
    v2, p2 = mp.carve(ins, origins=org, radius=0.3, margin=0.0, min_passes=1000, return_passes=True)
    assert v2 == 0 and p2.sum() > 0 and mp.n_points == n1 - v1
print("ok", a.iterations, m.iterations, int(tab[:, 16].sum()), c.iterations, d.iterations, f.iterations, g.iterations, l.iterations,
      float(np.linalg.norm(c.H - H_true)), float(np.linalg.norm(l.T - H_true)))
