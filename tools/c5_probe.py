"""Diagnostics (GPU): BASELINE configs[4] on one GPU — pairs/s of the batched engine against the
per-pair engine pool, on the C5 batch and on an overlap workload (the same surfaces cropped to
about 50 % overlap, a prior per pair drawn like C5's H_i, max_overlap_distance 0.5).  Not part of
the product.

    python tools/c5_probe.py [--dump FILE]    (--dump: np.save of the C5 batched table)"""
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import simpleicp_b200 as sb
from simpleicp_b200 import _capi, synthetic
from bench import make_c5_pairs


def overlap_pairs(n_pairs, n_pts):
    """C5's surfaces cropped to x < 20 (fixed) and x > 10 (movable, before its transform): half of
    each cloud overlaps the other.  Priors: an independent draw of C5's distribution (the true
    H_i are C5's), in degrees for the front end."""
    x_true = synthetic.c5_transforms(max(512, n_pairs))
    pairs = []
    for i in range(n_pairs):
        Xf = synthetic.surface(n_pts, 10_000 + 2 * i, extent=30.0)
        Xm = synthetic.surface(n_pts, 10_001 + 2 * i, extent=30.0)
        Xf, Xm = Xf[Xf[:, 0] < 20.0], Xm[Xm[:, 0] > 10.0]
        Xm = synthetic.apply_H(Xm, np.linalg.inv(synthetic.H_from_rbp(x_true[i])))
        pairs.append(tuple(torch.from_numpy(np.ascontiguousarray(X)).pin_memory().numpy() for X in (Xf, Xm)))
    rng = np.random.default_rng(7)
    prior = np.column_stack((rng.uniform(-1.0, 1.0, (n_pairs, 3)), rng.uniform(-0.2, 0.2, (n_pairs, 3))))
    return pairs, prior


def timed(pairs, reps=3, **kw):
    sb.simpleicp_batch(pairs, on_error="nan", **kw)
    torch.cuda.synchronize()
    best, tab = np.inf, None
    for _ in range(reps):
        t0 = time.perf_counter()
        tab = sb.simpleicp_batch(pairs, on_error="nan", **kw)
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best, tab


def report(label, n_pairs, dt, tab):
    print(f"{label:22s}: {n_pairs / dt:8.0f} pairs/s ({dt * 1e3:.1f} ms for {n_pairs} pairs), mean iterations "
          f"{tab[tab[:, 16] > 0, 16].mean():.1f}, failed {(tab[:, 16] < 0).sum()}", flush=True)


def main(n_pairs=64, n_pts=100_000, dump=None):
    print(torch.cuda.get_device_name(0), flush=True)
    pairs = make_c5_pairs(range(n_pairs), n_pts, pinned=True)
    for label, kw in (("batched", dict(engine="batched", batch_size=n_pairs)),
                      ("batched/32", dict(engine="batched", batch_size=32)),
                      ("pool x8", dict(engine="pool", concurrency=8))):
        dt, tab = timed(pairs, **kw)
        report(label, n_pairs, dt, tab)
        if dump and label == "batched":
            np.save(dump, tab)
    eng = sb.batch._BATCH_ENGINES[0]
    print({k: round(v, 3) for k, v in eng.timings().items()})

    opairs, prior = overlap_pairs(n_pairs, n_pts)
    kw = dict(max_overlap_distance=0.5, rbp_observed_values=prior)
    dt_b, tab_b = timed(opairs, engine="batched", batch_size=n_pairs, **kw)
    report("overlap batched", n_pairs, dt_b, tab_b)
    t = eng.timings()
    print(f"overlap filter stage: {t['overlap_ms']:.3f} ms for {n_pairs} pairs "
          f"({sum(len(a) for a, _ in opairs)} fixed points); grid_mov {t['grid_mov_ms']:.3f} ms, "
          f"normals {t['normals_ms']:.3f} ms, loop {t['reject_solve_ms']:.3f} ms", flush=True)
    dt_p, tab_p = timed(opairs, engine="pool", concurrency=8, **kw)
    report("overlap pool x8", n_pairs, dt_p, tab_p)
    ok = (tab_b[:, 16] > 0) & (tab_p[:, 16] > 0)
    print(f"batched vs pool: max |dH| {np.abs(tab_b[ok, :16] - tab_p[ok, :16]).max():.2e}, "
          f"equal counts {np.array_equal(tab_b[:, 16:18], tab_p[:, 16:18])}")


if __name__ == "__main__":
    main(dump=sys.argv[sys.argv.index("--dump") + 1] if "--dump" in sys.argv else None)
