"""One GPU call, every measurement knob: runs bench.py under each environment setting and prints the stage
times side by side (run on the GPU box: `python tools/variant_sweep.py [--steps 10]`).  All variants produce
the same results; the bench's parity block (kept on for the first run of each knob) confirms it."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = [
    ("default (a2 on tensor cores)", {}),
    ("exact fp32 a2 (PB_K1_TC=0)", {"PB_K1_TC": "0"}),
    ("exact a2 + code-diff diagnostic", {"PB_K1_TC_DIAG": "1"}),
    ("tensor cores, E=2", {"PB_K1_TC_E": "2"}),
    ("approx grid x4", {"PB_APPROX_GRID": "4"}),
    ("filter off", {"PB_FAST_EXACT": "0"}),
    ("list-scan probe (exact a2)", {"PB_PROBE16": "0", "PB_K1_TC": "0"}),
    ("token-form exact stage (PB_PAIR_EXACT=0)", {"PB_PAIR_EXACT": "0"}),
    ("pass-2 grid 1", {"PB_WS_GRID2": "1"}),
    ("pass-2 grid 4", {"PB_WS_GRID2": "4"}),
    ("pass-2 grid 8", {"PB_WS_GRID2": "8"}),
    ("pass-2 grid 16", {"PB_WS_GRID2": "16"}),
    ("pass-2 grid 32", {"PB_WS_GRID2": "32"}),
    ("ws grid 4", {"PB_WS_GRID": "4"}),
    ("ws grid 16", {"PB_WS_GRID": "16"}),
    ("ws grid 32", {"PB_WS_GRID": "32"}),
    ("lanes 2 (PB_LANES=2)", {"PB_LANES": "2"}),
    ("lanes 3", {"PB_LANES": "3"}),
    ("lanes 4", {"PB_LANES": "4"}),
    ("nq=48 queries", {"__args__": "--nq 48"}),
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--only", default="", help="comma-separated substrings of variant names")
    args = ap.parse_args()
    rows = []
    for name, env in VARIANTS:
        if args.only and not any(s in name for s in args.only.split(",")):
            continue
        env = dict(env)
        extra = env.pop("__args__", "").split()
        e = dict(os.environ, **env)
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--steps", str(args.steps), "--warmup", "3",
               "--recall-queries", "0", "--no-cpu", "--threads", "1"] + extra
        out = subprocess.run(cmd, env=e, capture_output=True, text=True, timeout=600)
        line = [l for l in out.stdout.splitlines() if l.startswith("{")]
        if out.returncode != 0 or not line:
            rows.append((name, None, out.stderr[-300:]))
            continue
        d = json.loads(line[-1])
        rows.append((name, d, ""))
    for name, d, err in rows:
        if d is None:
            print(f"{name:34s} FAILED {err}")
            continue
        st = d["stage_ms_per_step"]
        par = d.get("self_parity") or {}
        print(f"{name:34s} {d['value']:8.0f} q/s  " + "  ".join(f"{k}={st[k]:.3f}" for k in
              ("centroid_scores", "probe", "approx", "exact")) +
              "  " + "  ".join(f"k.{k}={v:.3f}" for k, v in d.get("kernel_ms_per_step", {}).items()) +
              f"  parity {par.get('ids_identical')}/{par.get('queries')} dmax={par.get('max_abs_score_diff')}"
              f"  k1_code_diff={d.get('work_per_step', {}).get('k1_tc_max_code_diff')}"
              f"  tc/redo={d.get('work_per_step', {}).get('n_k1_tc')}/{d.get('work_per_step', {}).get('n_k1_tc_redo')}"
              f"  recheck_docs={d.get('work_per_step', {}).get('n_recheck_docs')}")


if __name__ == "__main__":
    main()
