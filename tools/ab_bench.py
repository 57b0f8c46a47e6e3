#!/usr/bin/env python
"""A/B of one environment switch on the bench workloads (one GPU):
    python tools/ab_bench.py GS_PDL=0 [--workloads bonsai,garden,synth16m] [--steps 20]
Runs bench.py without and with the setting, prints frames/s, e2e and the per-kernel times that moved by more than 1 us."""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def run(workload, steps, env):
    out = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--workload", workload, "--steps", str(steps), "--warmup", "3", "--no-cpu-baseline"],
                         capture_output=True, text=True, env={**os.environ, **env}, timeout=900)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    if out.returncode or not lines:
        raise SystemExit(f"bench failed ({env}): {out.stderr[-1500:]}")
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("setting", help="NAME=VALUE applied to the B arm")
    ap.add_argument("--workloads", default="bonsai")
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    name, value = a.setting.split("=", 1)
    for w in a.workloads.split(","):
        base = run(w, a.steps, {})
        test = run(w, a.steps, {name: value})
        moved = {}
        for k in sorted(set(base["kernel_ms"]) | set(test["kernel_ms"])):
            x, y = base["kernel_ms"].get(k, 0.0) * 1e3, test["kernel_ms"].get(k, 0.0) * 1e3
            if abs(x - y) > 1.0:
                moved[k] = [round(x, 1), round(y, 1)]
        print(json.dumps({"workload": w, "setting": a.setting, "fps": [round(base["value"], 1), round(test["value"], 1)],
                          "e2e_fps": [round(base["e2e"]["value"], 1), round(test["e2e"]["value"], 1)], "kernel_us_moved": moved,
                          "tile_instances": [base["tile_instances"], test["tile_instances"]]}), flush=True)


if __name__ == "__main__":
    main()
