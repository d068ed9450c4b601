# Slush / Snowflake on the device: init time and device memory, a device-timed run to quiescence (msgs.size() == 0), the
# passes whose draw indices were re-derived serially, a per-kernel profile (separate run), and the CPU restatement's time
# over a prefix window (compared bit for bit at its end, on a network of its own that is released before the timed one).
# usage: gpu_avalanche.py slush|snowflake NODES [--bcap B] [--prefix-ms P] [--wall-limit S]
# Parameters are the reference tests': Slush (N, M=7, K=7, A=4/7), Snowflake (N, M=5, K=7, A=4/7, B=3), RANDOM builder,
# NetworkLatencyByDistanceWJitter.
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tests.avalanche_parity import NB, NL, compare  # noqa: E402
from wittgenstein_b200 import Slush, SlushParameters, Snowflake, SnowflakeParameters  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("proto", choices=["slush", "snowflake"])
ap.add_argument("nodes", type=int)
ap.add_argument("--bcap", type=int, default=0, help="bucket capacity (0: the engine's default, max(16384, 3N))")
ap.add_argument("--prefix-ms", type=int, default=1000, help="window the CPU restatement runs (0: none)")
ap.add_argument("--wall-limit", type=float, default=600.0, help="stop the timed run after this many seconds of wall time")
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"card: {card}", flush=True)


def make():
    tun = {"bcap": args.bcap} if args.bcap else None
    if args.proto == "slush":
        return Slush(SlushParameters(args.nodes, 7, 7, 4.0 / 7.0, NB, NL), tunables=tun)
    return Snowflake(SnowflakeParameters(args.nodes, 5, 7, 4.0 / 7.0, 3, NB, NL), tunables=tun)


torch.cuda.init()
if args.prefix_ms:
    from tests.avalanche_oracle_lib import OracleSlush, OracleSnowflake

    q = make()
    q.init()
    o = OracleSlush(args.nodes, 7, 7, 4.0 / 7.0, NB, NL) if args.proto == "slush" else OracleSnowflake(args.nodes, 5, 7, 4.0 / 7.0, 3, NB, NL)
    o.init()
    oracle_ms = 0.0
    while o.time < args.prefix_ms:
        oracle_ms += o.run_timed(100)
        q.network().run_ms(100)
    bad = compare(q, o, f"t={o.time}")
    print(f"oracle (one CPU thread) over [0, {o.time}] ms: {oracle_ms / 1000:.2f} s, {o.deliveries()} deliveries; device state "
          f"{'bit-exact' if not bad else 'DIFFERS: ' + str(bad)}", flush=True)
    q.network().close()
    del q, o

free0, total = torch.cuda.mem_get_info()
t0 = time.time()
p = make()
p.init()
net = p.network()
net.msgs_size()  # synchronises
init_s = time.time() - t0
free1, _ = torch.cuda.mem_get_info()
print(f"{args.proto} N={args.nodes} bcap={net.stats()['bcap']}: init {init_s:.2f} s, device memory {(free0 - free1) / 2**30:.2f} GiB "
      f"of {total / 2**30:.1f}", flush=True)

net.timer_start()
t1 = time.time()
step = 100
while net.msgs_size() != 0 and time.time() - t1 < args.wall_limit:
    net.run_ms(step)
dev_ms = net.timer_stop_ms()
wall = time.time() - t1
st = net.stats()
quiet = net.msgs_size() == 0
print(f"run to t={net.time} ms ({'quiescent' if quiet else 'NOT quiescent: stopped at the wall limit'}): device {dev_ms:.1f} ms, "
      f"wall {wall:.2f} s -> {net.time / (dev_ms / 1000.0):.0f} simulated-ms/s, {st['deliveries']} deliveries "
      f"({st['deliveries'] / (dev_ms / 1000.0) / 1e6:.1f} M/s); serial passes {p.serial_passes()} of {net.time}; "
      f"max bucket {st['max_bucket']}; records {st['rec_top']}; launches {st['kernel_launches']}", flush=True)
s = p.scalars()
print(f"colours: {int((s['color'] == 1).sum())} x 1, {int((s['color'] == 2).sum())} x 2, {int((s['color'] == 0).sum())} uncoloured",
      flush=True)
net.close()
del p, net

p = make()
p.init()
net = p.network()
net.profile_enable(True)
t1 = time.time()
while net.msgs_size() != 0 and time.time() - t1 < args.wall_limit:
    net.run_ms(step)
prof = net.profile_read()
net.profile_enable(False)
tot = sum(v[0] for v in prof.values())
print(f"per-kernel ms over [0, {net.time}] ms (profiled run, total {tot:.1f}):",
      {k: (round(v[0], 1), v[1]) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0]) if v[1]}, flush=True)
