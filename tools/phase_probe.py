"""Diagnostics (GPU): phase timeline of the reject/solve kernel and per-iteration cost of the
first iterations of a registration for a few ring limits.  Not part of the product."""
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from bench import make_pair

LABELS = {1: "median", 2: "mad", 3: "accum", 4: "sync", 5: "solve", 6: "sync", 7: "resid", 8: "sync", 9: "exit"}


def probe(n, K, rings=(4, 8, 12, 16)):
    X_fix, X_mov, _ = make_pair(n, 0)
    with _capi.Engine() as e:
        e.set_clouds(X_fix, X_mov)
        idx = sb.pointcloud.subsample_indices(n, K).astype(np.int64)
        e.set_selected(idx)
        e.estimate_normals(10)
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        p = e.run_params(0.3, 1.0, 100, lsq)
        print(f"== n={n} K={K}")
        for r in rings:
            e.set_option("grid_max_rings", r)
            e.iterate(p, x_in=np.zeros(6))  # warm
            rows = []
            import torch
            for it in range(6):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rec = e.iterate(p, x_in=np.zeros(6) if it == 0 else None, want_record=True)
                dt = (time.perf_counter() - t0) * 1e6
                rows.append((dt, rec.n_bruteforce, rec.n_kept, rec.lm_iterations))
            print(f"rings={r:3d}: " + " | ".join(f"{dt:7.0f}us bf={b} kept={k} lm={l}" for dt, b, k, l in rows))
        # steady-state phase timeline
        for rep in range(3):
            rec_lm = e.iterate(p, want_record=True).lm_iterations
            t = e.phase_times()
            seq = " ".join(f"{LABELS[i]}={t[i]:.1f}" for i in range(1, 10))
            sel = (f"med[lv={t[24]:.0f} cand={t[26]:.0f}: levels={t[10]:.1f} gather={t[11]:.1f} sort={t[12]:.1f}] "
                   f"mad[lv={t[25]:.0f} cand={t[27]:.0f}: levels={t[14]:.1f} gather={t[15]:.1f} sort={t[16]:.1f}]")
            print("  phases(us): " + seq + f" | D: reduce={t[17]:.1f} assemble={t[18]:.1f} eval0={t[21]:.1f} chol0={t[22]:.1f} lm={t[19]:.1f} lm_it={rec_lm} fastsel={t[28]:.0f} cand={t[26]:.0f}/{t[27]:.0f}")
            print("  " + sel)
        for mg in (1, 4, 8, 16):
            e.set_option("match_group", mg)
            sw = e.time_stages(p, 10, False)
            sc = e.time_stages(p, 10, True)
            print(f"  match_group={mg:2d}: match warm {sw['match_grid']*1e3:6.1f} us  cold {sc['match_grid']*1e3:6.1f} us")
        e.set_option("match_group", 0)
    for occ in (1.5, 2.0, 4.0, 6.0):
        with _capi.Engine() as e:
            e.set_option("grid_target_occupancy", occ)
            e.set_clouds(X_fix, X_mov)
            e.set_selected(idx)
            e.estimate_normals(10)
            lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
            p = e.run_params(0.3, 1.0, 100, lsq)
            e.iterate(p, x_in=np.zeros(6), want_record=True)
            for _ in range(4):
                e.iterate(p, want_record=True)
            sw = e.time_stages(p, 10, False)
            tm = e.timings()
            print(f"  occupancy target {occ}: match warm {sw['match_grid']*1e3:6.1f} us, grid build {tm['grid_mov_ms']:.3f} ms, normals {tm['normals_ms']:.3f} ms")


if __name__ == "__main__":
    probe(1_000_000, 100_000)
    probe(100_000, 1000, rings=(4, 12))
