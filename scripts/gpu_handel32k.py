"""BASELINE config #3: Handel 32 768 nodes, 25 % Byzantine (suicide), AwsRegionNetworkLatency, 1 x H100.
Times the GPU engine to completion and checks the state against the oracle at t = 100 / 300 ms."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from wittgenstein_b200 import Handel, HandelParameters
from tests.oracle_lib import OracleHandel
from tests.test_gpu_parity import _handel_compare
n = int(sys.argv[1]) if len(sys.argv) > 1 else 32768
check_until = int(sys.argv[2]) if len(sys.argv) > 2 else 300
args = (n, int(n * 0.7425), 4, 50, 10, 20, 10, n // 4)
nb, nl = "AWS_SPEED=GAUSSIAN_TOR=0.00", "AwsRegionNetworkLatency"
t0 = time.time(); p = Handel(HandelParameters(*args, nb, nl, 0, True, False)); p.init(); p.network().msgs_size(); init_s = time.time() - t0
print("gpu init_s", round(init_s, 1), flush=True)
t0 = time.time(); o = OracleHandel(*args, nb, nl, 0, True); o.init(); print("oracle init_s", round(time.time() - t0, 1), flush=True)
net = p.network(); dev = 0.0; cpu = 0.0
while o.time < check_until:
    net.timer_start(); net.run_ms(100); dev += net.timer_stop_ms()
    cpu += o.run_timed(100, 1)
    bad = _handel_compare(p, o, f"t={o.time}", full=True)
    print("t", o.time, "gpu ms", round(dev, 1), "cpu s", round(cpu, 1), "parity", "OK" if not bad else bad, flush=True)
    if bad: sys.exit(1)
while p.continue_if() and net.time < 10000:
    net.timer_start(); net.run_ms(100); dev += net.timer_stop_ms()
print(json.dumps({"workload": f"Handel {n} nodes, {n//4} Byzantine (suicide), AWS", "sim_ms": net.time, "device_ms": dev, "sim_ms_per_s": net.time / (dev / 1000.0),
                  "init_s": init_s, "oracle_sim_ms_per_s_first_%d" % check_until: check_until / cpu, "stats": net.stats()}))
