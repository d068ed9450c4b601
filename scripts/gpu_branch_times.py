"""Per-pass times of the three parts of a GSF pipeline pass that could run beside one another (DESIGN.md §4):

  C     checkSigs: k_cond_mark + k_cond_nodes<0> (k_cond_scan), k_cond_score, k_cond_nodes<1> (k_cond_select)
  D     delivery dispatch: k_dispatch_count, scan A (k_scan_a_partial + k_scan_a_final), k_dispatch_scatter
  TAIL  emission: scan B (k_scan_partial + k_scan_final), k_emit, multisplit (k_ms_count + k_ms_scan + k_ms_scatter);
        k_free, which runs beside the multisplit, is listed apart

on the workload of `bench.py` (GSFSignature, seed 0, the whole run of a fresh network in K steps of runMs(⌈run length / K⌉)).
The times come from the serial profiled pass (CUDA events around each group of kernels), so each is the part's own.
A pass that ran C of the next millisecond beside TAIL would save about min(C, TAIL) − D of what the two-branch pass spends
(C ∥ D, then TAIL).  An unprofiled device-timed run of the same window gives the µs per pass that saving is set against.

    python scripts/gpu_branch_times.py [--nodes 65536] [--steps 22] [--out branch_times.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PARTS = {
    "C": ["k_cond_scan", "k_cond_score", "k_cond_select"],
    "D": ["k_dispatch_count", "k_scan_a_partial", "k_scan_a_final", "k_dispatch_scatter"],
    "TAIL": ["k_scan_partial", "k_scan_final", "k_emit", "k_ms_count", "k_ms_scan", "k_ms_scatter"],
    "k_free": ["k_free"],
}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=22)
    ap.add_argument("--out", default="")
    args = ap.parse_args()

    import __graft_entry__ as g

    g.build()
    import bench

    n, K = args.nodes, args.steps
    p, _ = bench.make_gsf(n, 0)  # run length, as bench.py's warm-up measures it
    t_done = 0
    while p.continue_if() and t_done < 60000:
        p.network().run_ms(50)
        t_done += 50
    del p
    S = max(10, -(-t_done // K))

    p, _ = bench.make_gsf(n, 0)
    net = p.network()
    net.timer_start()
    for _ in range(K):
        net.run_ms(S)
    dev_ms = net.timer_stop_ms()
    passes = net.time
    del p, net

    p, _ = bench.make_gsf(n, 0)
    net = p.network()
    net.profile_enable(True, split_scans=True)
    for _ in range(K):
        net.run_ms(S)
    prof = net.profile_read()
    net.profile_enable(False)
    del p, net

    ticks = prof["k_begin"][1]
    us = {k: 1000.0 * v[0] / ticks for k, v in prof.items() if v[1]}
    parts = {name: round(sum(us.get(k, 0.0) for k in ks), 2) for name, ks in PARTS.items()}
    line = {"nodes": n, "steps": K, "step_ms": S, "passes": ticks, "card": card(),
            "us_per_pass_timed": round(1000.0 * dev_ms / passes, 2), "us_per_pass_profiled_sum": round(sum(us.values()), 2),
            "parts_us_per_pass": parts, "saving_estimate_us": round(min(parts["C"], parts["TAIL"]) - parts["D"], 2),
            "kernel_us_per_pass": {k: round(v, 2) for k, v in us.items()}}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
