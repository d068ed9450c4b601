"""Node-sharded Handel: BASELINE config #3 (Handel 32 768 nodes, 8 192 suicide-Byzantine, AwsRegionNetworkLatency) run to
completion on 1, 2 and 4 shards, and the capacity sizes one GPU cannot hold (65 536 nodes on 2 GPUs, 131 072 on 4).

Per run: device-timed simulated-ms/s (CUDA events on every shard's stream; the slowest shard counts), init time (wall clock),
peak host RSS of the process, and device memory per shard (drop in free memory across network construction and init).

  python scripts/gpu_handel_sharded.py [--out DIR] [--capacity]
      one process; shards placed round-robin on the box's GPUs; every configuration runs in a child process of its own, so
      that its peak RSS and device memory are its own
  torchrun --nproc-per-node G scripts/gpu_handel_sharded.py --nodes N
      one shard per process and GPU (DistributedHandel; exchange-region handles through torch.distributed over gloo)

A size whose host or device memory the box cannot provide is reported as unmeasured, with the estimate that ruled it out."""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NB, NL = "AWS_SPEED=GAUSSIAN_TOR=0.00", "AwsRegionNetworkLatency"
MAX_MS = 20000


def params(n):
    from wittgenstein_b200 import HandelParameters

    return HandelParameters(n, int(n * 0.7425), 4, 50, 10, 20, 10, n // 4, NB, NL, 0, True, False)  # as scripts/gpu_handel32k.py


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return [x.strip() for x in q.stdout.strip().splitlines()]


def free_bytes(devices):
    import torch

    return {d: torch.cuda.mem_get_info(d)[0] for d in sorted(set(devices))}


def host_estimate(n, world, procs):
    """bytes of host memory a run needs at its peak: per shard the transposed rank table (N^2 ints) plus its own rank rows and
    emission lists (2 x N/G x N x 4 B); `procs` shards per process"""
    return procs * (4 * n * n + 2 * 4 * (n // world) * n)


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def run_one(n, world):
    """one configuration in this process: shards on the box's GPUs round-robin"""
    import torch

    from wittgenstein_b200 import Handel
    from wittgenstein_b200.sharded import ShardedHandel

    ng = torch.cuda.device_count()
    devices = [r % ng for r in range(world)]
    for d in sorted(set(devices)):
        torch.cuda.mem_get_info(d)  # CUDA context first: its memory is not the engine's
    before = free_bytes(devices)
    t0 = time.time()
    p = Handel(params(n), device=0) if world == 1 else ShardedHandel(params(n), world, devices=devices)
    p.init()
    net = p.network()
    net.msgs_size()  # ends in a device synchronise
    init_s = time.time() - t0
    after = free_bytes(devices)
    per_dev = {d: before[d] - after[d] for d in before}
    dev_mem = [per_dev[devices[r]] / devices.count(devices[r]) for r in range(world)]
    dev_ms = 0.0
    while p.continue_if() and net.time < MAX_MS:
        net.timer_start()
        net.run_ms(100)
        dev_ms += net.timer_stop_ms()
    out = {"workload": f"Handel {n} nodes, {n // 4} Byzantine (suicide), AWS", "shards": world, "gpus": len(set(devices)),
           "sim_ms": net.time, "completed": not p.continue_if(), "device_ms": round(dev_ms, 1),
           "sim_ms_per_s": round(net.time / (dev_ms / 1000.0), 1), "init_s": round(init_s, 1),
           "peak_host_rss_gb": round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2**20, 2),
           "device_gb_per_shard": [round(x / 2**30, 2) for x in dev_mem]}
    if world > 1:
        p.close()  # the read-backs above come first: closing destroys the shards' handles
    return out


def run_distributed(n):
    import torch
    import torch.distributed as dist

    from wittgenstein_b200.sharded import DistributedHandel

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    torch.cuda.mem_get_info(local)
    before = torch.cuda.mem_get_info(local)[0]
    t0 = time.time()
    p = DistributedHandel(params(n), dist, rank, world, local)
    p.init()
    net = p.network()
    net.msgs_size()
    init_s = time.time() - t0
    mem = before - torch.cuda.mem_get_info(local)[0]
    dev_ms = 0.0
    while p.continue_if() and net.time < MAX_MS:
        net.timer_start()
        net.run_ms(100)
        dev_ms += net.timer_stop_ms()
    rows = [None] * world
    dist.all_gather_object(rows, {"device_ms": dev_ms, "init_s": init_s, "mem": mem, "done": not p.local.continue_if(),
                                  "rss": resource.getrusage(resource.RUSAGE_SELF).ru_maxrss})
    if rank == 0:
        slow = max(r["device_ms"] for r in rows)
        print("RESULT " + json.dumps({"workload": f"Handel {n} nodes, {n // 4} Byzantine (suicide), AWS", "shards": world, "mode": "torchrun",
                                      "sim_ms": net.time, "completed": all(r["done"] for r in rows),
                                      "device_ms": round(slow, 1), "sim_ms_per_s": round(net.time / (slow / 1000.0), 1),
                                      "init_s": round(max(r["init_s"] for r in rows), 1),
                                      "peak_host_rss_gb_per_process": [round(r["rss"] / 2**20, 2) for r in rows],
                                      "device_gb_per_shard": [round(r["mem"] / 2**30, 2) for r in rows], "gpu": gpu_info()}), flush=True)
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=32768)
    ap.add_argument("--one", type=int, default=0, help="internal: run one configuration with this many shards in this process")
    ap.add_argument("--capacity", action="store_true", help="also 65 536 nodes on 2 GPUs and 131 072 on 4 where the box allows")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if "RANK" in os.environ and "LOCAL_RANK" in os.environ:
        run_distributed(a.nodes)
        return
    if a.one:
        print("RESULT " + json.dumps(run_one(a.nodes, a.one)), flush=True)
        return
    import torch

    ng = torch.cuda.device_count()
    plan = [(a.nodes, 1), (a.nodes, 2), (a.nodes, 4)]
    if a.capacity:
        plan += [(65536, 2), (131072, 4)]
    results = []
    info = gpu_info()
    print(json.dumps({"gpus": info, "host_mem_available_gb": round(mem_available() / 2**30, 1)}), flush=True)
    for n, world in plan:
        need = host_estimate(n, world, world)
        if n > a.nodes and ng < world:
            r = {"nodes": n, "shards": world, "unmeasured": f"needs {world} GPUs, the box has {ng}"}
        elif need > 0.9 * mem_available():
            r = {"nodes": n, "shards": world, "unmeasured": f"needs about {need / 2**30:.0f} GB of host memory in one process, "
                                                             f"{mem_available() / 2**30:.0f} GB available"}
        else:
            out = subprocess.run([sys.executable, "-X", "faulthandler", os.path.abspath(__file__), "--nodes", str(n), "--one", str(world)],
                                 capture_output=True, text=True)
            line = [x for x in out.stdout.splitlines() if x.startswith("RESULT ")]
            r = json.loads(line[-1][7:]) if line else {"nodes": n, "shards": world, "failed": f"exit code {out.returncode}",
                                                      "stdout": out.stdout[-1500:], "stderr": out.stderr[-3000:]}
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "handel_sharded.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
