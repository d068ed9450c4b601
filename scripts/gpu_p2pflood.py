# P2PFlood on the device: init time and device memory, a device-timed run until every live node is done, deliveries/s, the
# passes whose draw indices were re-derived serially, the share of k_emit_peers in a per-kernel profile (separate run), and
# the CPU restatement's time over the same run (compared bit for bit at its end, on a network of its own that is released
# before the timed one).  The card's name and power limit are read in the same call.
# usage: gpu_p2pflood.py flood NODES [--bcap B] [--no-oracle]     floodTime(): NODES live nodes, peersCount 15, delays 1 / 1
#        gpu_p2pflood.py time [NODES] [--concurrency C]          P2PFlood.time(): N nodes, N messages, 13 peers, delays 1 / 0,
#                                                                  RunMultipleTimes over 5 seeds against sequential oracle runs
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tests.p2p_parity import compare  # noqa: E402
from wittgenstein_b200 import P2PFlood, P2PFloodParameters  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("mode", choices=["flood", "time"])
ap.add_argument("nodes", type=int, nargs="?", default=8192)
ap.add_argument("--bcap", type=int, default=0, help="bucket capacity (0: the engine's default, max(16384, 3N))")
ap.add_argument("--desc-cap", type=int, default=0)
ap.add_argument("--no-oracle", action="store_true")
ap.add_argument("--no-profile", action="store_true")
ap.add_argument("--concurrency", type=int, default=5)
ap.add_argument("--wall-limit", type=float, default=600.0)
args = ap.parse_args()

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(f"card: {card}; library {os.environ.get('WTG_LIB', 'default')}", flush=True)
torch.cuda.init()
tun = {k: v for k, v in (("bcap", args.bcap), ("desc_cap", args.desc_cap)) if v}


def done(net):
    return not (net.counters()[4][net.attrs()["down"] == 0] == 0).any()


if args.mode == "time":
    from tests.p2p_oracle_lib import OracleP2PFlood
    from wittgenstein_b200 import DoneAtStatGetter, MsgReceivedStatGetter, RunMultipleTimes, cont_until_done

    n = args.nodes
    rmt = RunMultipleTimes(P2PFlood(P2PFloodParameters(n, 0, 1, n, 1, 13, 0), tunables=tun), 5, 0, [DoneAtStatGetter(), MsgReceivedStatGetter()])
    t0 = time.time()
    res = rmt.run(cont_until_done, concurrency=args.concurrency)
    wall = time.time() - t0
    print(f"P2PFlood.time() N={n}: RunMultipleTimes 5 seeds, concurrency {args.concurrency}: wall {wall:.2f} s (inits included); "
          f"doneAt {res[0]}, msgReceived {res[1]}; end times {rmt.end_times}", flush=True)
    if not args.no_oracle:
        t0 = time.time()
        for seed in range(5):
            o = OracleP2PFlood(n, 0, 1, n, 1, 13, 0, seed=seed)
            o.init()
            while True:
                did = o.run_ms(10)
                if not (not did or (o.counters()[4] == 0).any()):
                    break
            assert o.time == rmt.end_times[seed], (seed, o.time, rmt.end_times[seed])
        print(f"oracle (one CPU thread), the 5 seeds one after the other: {time.time() - t0:.2f} s; end times equal", flush=True)
    sys.exit(0)


def make():
    return P2PFlood(P2PFloodParameters(args.nodes, 0, 1, 1, 1, 15, 1), tunables=tun or None)


if not args.no_oracle:
    from tests.p2p_oracle_lib import OracleP2PFlood

    q = make()
    q.init()
    o = OracleP2PFlood(args.nodes, 0, 1, 1, 1, 15, 1)
    o.init()
    oracle_ms = 0.0
    while not (o.counters()[4] > 0).all() and o.time < 50000:
        oracle_ms += o.run_timed(100)
        q.network().run_ms(100)
    bad = compare(q, o, f"t={o.time}", bitmaps=False)
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
print(f"floodTime N={args.nodes} bcap={net.stats()['bcap']} ring={net.stats()['ring']} avgPeers={p.avg_peers()}: init {init_s:.2f} s, "
      f"device memory {(free0 - free1) / 2**30:.2f} GiB of {total / 2**30:.1f}", flush=True)
net.timer_start()
t1 = time.time()
step = 100
while not done(net) and time.time() - t1 < args.wall_limit:
    net.run_ms(step)
dev_ms = net.timer_stop_ms()
st = net.stats()
print(f"run to t={net.time} ms ({'all live nodes done' if done(net) else 'NOT done: wall limit'}): device {dev_ms:.1f} ms -> "
      f"{net.time / (dev_ms / 1000.0):.0f} simulated-ms/s, {st['deliveries']} deliveries ({st['deliveries'] / (dev_ms / 1000.0) / 1e6:.1f} M/s); "
      f"serial passes {p.serial_passes()}; busiest ms {st['max_bucket']} envelopes; records {st['rec_top']}", flush=True)
net.close()
del p, net

if not args.no_profile:
    p = make()
    p.init()
    net = p.network()
    net.profile_enable(True)
    while not done(net):
        net.run_ms(step)
    prof = net.profile_read()
    net.profile_enable(False)
    tot = sum(v[0] for v in prof.values())
    print(f"per-kernel ms over [0, {net.time}] ms (profiled run, total {tot:.1f}; k_emit_peers {100 * prof['k_emit_peers'][0] / tot:.1f} %):",
          {k: (round(v[0], 2), v[1]) for k, v in sorted(prof.items(), key=lambda kv: -kv[1][0]) if v[1]}, flush=True)
