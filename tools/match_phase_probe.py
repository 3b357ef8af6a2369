"""Diagnostics (GPU): where the steady-state one-pair match spends its time on the C3 pair
(1M <-> 1M, K = 100 000).  After the bench's 12 warm-up iterations it times 7 x 20 cold-L2 steps
(inner events, as bench.py's per-kernel split) for each lane count, and prints the %globaltimer
phase stamps of the first and the last block of the last step of every round (option
match_stamps), the queries answered from a certificate (sicp_debug_match_counts), the grid size
and the waves it takes at the kernel's register count.  Not part of the product.

    python tools/match_phase_probe.py [--lanes 0,2,4] [--out DIR]
"""
import argparse
import json
import re
import sys
from pathlib import Path

import numpy as np

REPO = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(REPO))
import simpleicp_b200 as sb  # noqa: E402
from simpleicp_b200 import _build, _capi  # noqa: E402
from bench import make_pair  # noqa: E402

PHASES = ("entry", "wait released", "state+cert loaded", "certified decision", "normal loaded",
          "histogram atomic returned", "exit")


def blocks_per_sm(lanes: int) -> tuple:
    """(registers, resident 128-thread blocks per SM) of k_match_grid_coop<lanes>, from the build's
    ptxas report (65536 registers per SM, allocated per warp in units of 256, at most 16 blocks)."""
    txt = (_build.OBJ / "nn.ptxas.txt").read_text()
    m = re.search(rf"k_match_grid_coopILi{lanes}E\S*\n.*\n.*Used (\d+) registers", txt)
    regs = int(m.group(1))
    per_warp = -(-regs * 32 // 256) * 256
    return regs, min(16, 65536 // (per_warp * 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", default="0,2,4", help="match_group values to time (0 = the library's choice)")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None, help="write the results as JSON here")
    args = ap.parse_args()
    import torch

    n, K = 1_000_000, 100_000
    X_fix, X_mov, _ = make_pair(n, 0)
    props = torch.cuda.get_device_properties(0)
    n_sm = props.multi_processor_count
    results = {"device": props.name, "sms": n_sm, "runs": []}
    with _capi.Engine() as e:
        e.set_clouds(X_fix, X_mov)
        e.set_selected(sb.pointcloud.subsample_indices(n, K).astype(np.int64))
        e.estimate_normals(10)
        lsq = e.lsq_params(np.zeros(6), np.zeros(6), np.zeros(6), 1.0)
        p = e.run_params(0.3, 1.0, 100, lsq)
        stamps = hasattr(e, "match_phase_times")
        for lanes in [int(v) for v in args.lanes.split(",")]:
            e.set_option("match_group", lanes)
            if stamps:
                e.set_option("match_stamps", 1)
            e.iterate(p, x_in=np.zeros(6), want_record=True)
            for _ in range(11):
                e.iterate(p, want_record=True)
            match_ms, it_ms, rounds = [], [], []
            for _ in range(args.rounds):
                st = e.time_stages(p, args.steps, True)
                match_ms.append(st["match_grid"] * 1e3)
                it_ms.append(st["iteration"] * 1e3)
                rounds.append(e.match_phase_times() if stamps else None)
            n_cert = e.match_counts()
            used = lanes if lanes else None
            run = {"match_group": lanes, "match_us": match_ms, "iteration_inner_us": it_ms, "n_certified": n_cert,
                   "stamps_us": rounds}
            print(f"match_group={lanes}: match {min(match_ms):.1f}-{max(match_ms):.1f} us (median "
                  f"{np.median(match_ms):.1f}), iteration with inner events {np.median(it_ms):.1f} us, "
                  f"certified {n_cert}/{K} ({100.0 * n_cert / K:.2f} %)")
            for mg in ((used,) if used else (2, 4)):
                regs, bps = blocks_per_sm(mg)
                grid = -(-K * mg // 128)
                print(f"    {mg} lanes: {regs} registers, {bps} blocks/SM, grid {grid} blocks = "
                      f"{grid / (bps * n_sm):.2f} waves on {n_sm} SMs")
            if stamps:
                t = np.array(rounds)
                for blk, off in (("first block", 0), ("last block", 8)):
                    cols = [np.median(t[:, off + i]) for i in range(7)]
                    print(f"    {blk} (us from the first block's entry, median of {args.rounds}): "
                          + ", ".join(f"{name} {v:.2f}" for name, v in zip(PHASES, cols)))
            results["runs"].append(run)
            if stamps:
                e.set_option("match_stamps", 0)
        e.set_option("match_group", 0)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "match_phase_probe.json").write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
