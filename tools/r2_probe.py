"""Diagnostics (GPU), round 2: cooperative vs barrier-free reject/solve kernel on C3 and on the
small configurations; phase stamps of the barrier-free kernel; end-to-end registrations with the
number of iterations each path served.  Not part of the product."""
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tests"))
import simpleicp_b200 as sb
from simpleicp_b200 import _capi
from bench import make_pair


def stages(e, p, reps=20):
    out = {}
    for fused, warm in ((0, 0), (1, 1), (1, 2)):
        e.set_option("fused", fused)
        e.set_option("warm_start", 1 if warm else 0)
        e.set_option("sphere_scan", 1 if warm == 2 else 0)
        e.iterate(p, x_in=np.zeros(6), want_record=True)
        for _ in range(12):
            e.iterate(p, want_record=True)
        sc = e.time_stages(p, reps, True)
        sw = e.time_stages(p, reps, False)
        out[(fused, warm)] = (sc, sw, e.phase_times())
    return out


def show(tag, res):
    for fused, (sc, sw, t) in res.items():
        print(f"{tag} fused/warm={fused}: cold match {sc['match_grid']*1e3:6.1f} rs {sc['reject_solve']*1e3:6.1f} it {sc['iteration']*1e3:6.1f} us | "
              f"warm match {sw['match_grid']*1e3:6.1f} rs {sw['reject_solve']*1e3:6.1f} it {sw['iteration']*1e3:6.1f} us | path {t[28]:.0f}")
        if t[28] == 2:
            print(f"    fused phases (us since stamp 0): kernel entry {t[23]:.1f} plan {t[10]:.1f} scan {t[11]:.1f} median {t[12]:.1f} select {t[2]:.1f} accumulate {t[3]:.1f} tail start {t[4]:.1f} "
                  f"partials {t[17]:.1f} assemble {t[18]:.1f} eval0 {t[21]:.1f} chol0 {t[22]:.1f} solve {t[19]:.1f} exit {t[9]:.1f} cand {t[26]:.0f}/{t[27]:.0f}")
            # k_rs_solve: entry, end of the rehearsal, wait released
            print(f"    solve kernel (us since stamp 0): entry {t[1]:.1f} rehearsal end {t[5]:.1f} wait released {t[6]:.1f} "
                  f"| rehearsal {t[5]-t[1]:.1f} us, real tail {t[9]-t[4]:.1f} us")


def c3():
    n, K = 1_000_000, 100_000
    X_fix, X_mov, _ = make_pair(n, 0)
    with _capi.Engine() as e:
        e.set_clouds(X_fix, X_mov)
        e.set_selected(sb.pointcloud.subsample_indices(n, K).astype(np.int64))
        e.estimate_normals(10)
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        p = e.run_params(0.3, 1.0, 100, lsq)
        show("C3", stages(e, p))
        e.set_option("fused", 1); e.set_option("warm_start", 1); e.set_option("sphere_scan", 1)
        for mg in (2, 4, 8):
            e.set_option("match_group", mg)
            e.iterate(p, x_in=np.zeros(6), want_record=True)
            for _ in range(12):
                e.iterate(p, want_record=True)
            sc, sw = e.time_stages(p, 20, True), e.time_stages(p, 20, False)
            print(f"C3 match_group={mg}: match cold {sc['match_grid']*1e3:.1f} warm {sw['match_grid']*1e3:.1f} us")
        e.set_option("match_group", 0)
        import torch

        for fused in (0, 1):
            e.set_option("fused", fused)
            e.set_option("warm_start", fused)
            e.set_option("sphere_scan", fused)
            sb.register(X_fix, X_mov, correspondences=K, engine=e, want_normals=False)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = sb.register(X_fix, X_mov, correspondences=K, engine=e, want_normals=False)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            tm = e.timings()
            print(f"C3 register fused={fused}: {dt*1e3:.2f} ms, {r.iterations} iterations, loop {r.loop_ms:.3f} ms, "
                  f"fused {tm['fused_iterations']} re-run {tm['rerun_iterations']}, normals {tm['normals_ms']:.3f} ms, "
                  f"grids {tm['grid_fix_ms']:.3f}+{tm['grid_mov_ms']:.3f} ms")
        # first iteration (far queries) with and without the sphere scan
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        p = e.run_params(0.3, 1.0, 100, lsq)
        for sph in (0, 1):
            e.set_option("sphere_scan", sph)
            ts = []
            for _ in range(3):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rec = e.iterate(p, x_in=np.zeros(6), want_record=True)
                ts.append((time.perf_counter() - t0) * 1e6)
            print(f"C3 first iteration (host wall, incl. sync) sphere_scan={sph}: {min(ts):.0f} us, brute-force queries {rec.n_bruteforce}")


def small(name, kw):
    from conftest import load_pair

    X_fix, X_mov = load_pair(name)
    with _capi.Engine() as e:
        for fused in (0, 1):
            e.set_option("fused", fused)
            e.set_option("warm_start", fused)
            e.set_option("sphere_scan", fused)
            sb.register(X_fix, X_mov, engine=e, want_normals=False, **kw)
            t0 = time.perf_counter()
            for _ in range(5):
                r = sb.register(X_fix, X_mov, engine=e, want_normals=False, **kw)
            dt = (time.perf_counter() - t0) / 5
            tm = e.timings()
            print(f"{name} fused={fused}: {dt*1e3:.2f} ms per call, {r.iterations} iterations, loop {r.loop_ms:.3f} ms "
                  f"({r.loop_ms/r.iterations*1e3:.1f} us/it), fused {tm['fused_iterations']} re-run {tm['rerun_iterations']}")


def normals_probe():
    from conftest import load_pair

    for name, n, K in (("C3", 1_000_000, 100_000), ("dragon", 0, 1000)):
        if name == "C3":
            X_fix, X_mov, _ = make_pair(n, 0)
        else:
            X_fix, X_mov = load_pair(name)
        with _capi.Engine() as e:
            e.set_clouds(X_fix, X_mov)
            e.set_selected(sb.pointcloud.subsample_indices(X_fix.shape[0], K).astype(np.int64))
            for mode in (1, 0, 2, -1):
                e.set_option("knn_coop", mode)
                e.estimate_normals(10, download=False)
                e.estimate_normals(10, download=False)
                print(f"normals {name} K={K} knn_coop={mode}: {e.timings()['normals_ms'] * 1e3:.1f} us")


if __name__ == "__main__":
    normals_probe()
    if len(sys.argv) > 1 and sys.argv[1] == "normals":
        sys.exit(0)
    c3()
    small("dragon", {})
    small("bunny", {"max_overlap_distance": 1.0})
    small("airborne", {})
    small("terrestrial", {})
