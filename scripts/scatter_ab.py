"""A/B of two scatter generations on the train bench: `bench.py --steps N --no-companions --no-cpu-baseline` in a fresh
process per run, the arms alternated (HRF_SCATTER=a, b, a, b, ...) so that drift of the shared host or of the clock under
the power cap falls on both.  Reports, per arm, the scatter phase (`phases_ms.scatter`, CUDA events inside
FusedTrainer.step) and the train rate (`value`) with median, min, max and spread (max - min), and the median SM clock of
each run's `clocks`.  The last line is one JSON object with every run.

Decision rule applied in the summary: arm b wins when its median scatter time is below the LOWEST scatter time of arm a,
and its median train rate exceeds arm a's by more than the larger of the two arms' rate spreads.

usage: python scripts/scatter_ab.py [--arms 5 6] [--runs 5] [--steps 50] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def run_once(gen: str, steps: int) -> dict:
    env = dict(os.environ, HRF_SCATTER=gen)
    cmd = [sys.executable, str(ROOT / "bench.py"), "--gpus", "1", "--steps", str(steps), "--no-companions", "--no-cpu-baseline"]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise RuntimeError(f"bench.py failed (HRF_SCATTER={gen}, rc {r.returncode}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    line = json.loads(lines[-1])
    return {"gen": gen, "value": line["value"], "ms_per_step": line["ms_per_step"], "scatter_ms": line["phases_ms"]["scatter"],
            "phases_ms": line["phases_ms"], "sm_mhz": line["clocks"].get("sm_mhz"), "clock_reasons": line["clocks"].get("reasons"),
            "samples_after_prune": line["config"].get("samples_after_prune_mean")}


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "spread": max(xs) - min(xs)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arms", nargs=2, default=["5", "6"], metavar=("A", "B"), help="HRF_SCATTER of the two arms")
    ap.add_argument("--runs", type=int, default=5, help="runs per arm (at least 5 for the decision rule)")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", help="directory for the per-run JSON and the summary")
    args = ap.parse_args()
    a, b = args.arms
    runs = []
    for i in range(args.runs):
        for gen in (a, b):
            r = run_once(gen, args.steps)
            runs.append(r)
            print(f"run {i} HRF_SCATTER={gen}: scatter {r['scatter_ms']:.3f} ms  step {r['ms_per_step']:.3f} ms  "
                  f"{r['value'] / 1e6:.4f} M rays/s  SM {r['sm_mhz']} MHz {r['clock_reasons']}", flush=True)
    arm = {g: {"scatter_ms": stats([r["scatter_ms"] for r in runs if r["gen"] == g]),
               "value": stats([r["value"] for r in runs if r["gen"] == g]),
               "ms_per_step": stats([r["ms_per_step"] for r in runs if r["gen"] == g]),
               "sm_mhz": stats([r["sm_mhz"] for r in runs if r["gen"] == g and r["sm_mhz"] is not None] or [0.0])}
           for g in (a, b)}
    sa, sb = arm[a], arm[b]
    scatter_win = sb["scatter_ms"]["median"] < sa["scatter_ms"]["min"]
    gain = sb["value"]["median"] - sa["value"]["median"]
    rate_win = gain > max(sa["value"]["spread"], sb["value"]["spread"])
    for g in (a, b):
        s = arm[g]
        print(f"HRF_SCATTER={g}: scatter median {s['scatter_ms']['median']:.3f} ms [{s['scatter_ms']['min']:.3f}, {s['scatter_ms']['max']:.3f}]  "
              f"train {s['value']['median'] / 1e6:.4f} M rays/s [{s['value']['min'] / 1e6:.4f}, {s['value']['max'] / 1e6:.4f}]  "
              f"step {s['ms_per_step']['median']:.3f} ms  SM clock median {s['sm_mhz']['median']:.0f} MHz")
    print(f"arm {b} vs {a}: scatter median below arm {a}'s lowest run: {scatter_win}; train rate gain {gain / 1e6:+.4f} M rays/s "
          f"({100 * gain / sa['value']['median']:+.2f} %) beyond the run-to-run spread: {rate_win}")
    summary = {"arms": [a, b], "runs_per_arm": args.runs, "steps": args.steps, "per_arm": arm, "scatter_win": scatter_win,
               "rate_win": rate_win, "rate_gain_pct": 100 * gain / sa["value"]["median"], "runs": runs}
    if args.out:
        out = Path(args.out)
        out.mkdir(parents=True, exist_ok=True)
        (out / f"scatter_ab_{a}_vs_{b}.json").write_text(json.dumps(summary, indent=1))
    print(json.dumps({k: v for k, v in summary.items() if k != "runs"}))


if __name__ == "__main__":
    main()
