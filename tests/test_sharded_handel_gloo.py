"""world_size-2 test of node-sharded Handel in its multi-process form on CPU (gloo): one shard per process (DistributedHandel),
exchange-region handles through torch.distributed; every rank's digests equal the oracle's for its id range, to completion."""
import json
import os
import subprocess
import sys

import numpy as np

from tests.test_sharded_gloo import _free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Range:
    """the oracle's read-backs restricted to the node ids [lo, lo + n), shaped like a shard's (tests.parity.handel_digests)"""

    def __init__(self, o, lo, n):
        self.o, self.lo, self.n = o, lo, n

    def network(self):
        return self

    def rng_state(self):
        return self.o.rng_state()

    def msgs_size(self):
        return self.o.msgs_live()

    def counters(self):
        return np.ascontiguousarray(self.o.counters()[:, self.lo:self.lo + self.n])

    def _cut(self, d):
        return {k: np.ascontiguousarray(v[self.lo:self.lo + self.n]) for k, v in d.items()}

    def scalars(self):
        return self._cut(self.o.scalars())

    def rows(self, w):
        return np.ascontiguousarray(self.o.rows(w)[self.lo:self.lo + self.n])

    def level_scalars(self):
        return self._cut(self.o.level_scalars())


def test_two_handel_shards_over_gloo():
    from tests.oracle_lib import OracleHandel
    from tests.parity import handel_digests

    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "sharded_handel_worker.py")]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    ranks = {}
    dec = json.JSONDecoder()
    pos = 0
    while True:
        i = out.stdout.find("RANKLINE ", pos)
        if i < 0:
            break
        r, _ = dec.raw_decode(out.stdout[i + 9:])
        ranks[r["rank"]] = r
        pos = i + 9
    assert sorted(ranks) == [0, 1]
    r0, r1 = ranks[0], ranks[1]
    assert r0["range"] == [0, 128] and r1["range"] == [128, 128] and r0["time"] == r1["time"]
    assert sorted(r0["digests"]) == sorted(r1["digests"]) and len(r0["digests"]) >= 4
    o = OracleHandel(256, 153, 4, 50, 10, 20, 10, 64, "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency", 0, True)
    o.init()
    while o.time < r0["time"]:
        o.run_ms(50)
        t = str(o.time)
        if t in r0["digests"]:
            for r in (r0, r1):
                lo, n = r["range"]
                want = handel_digests(_Range(o, lo, n), False)
                got = dict(r["digests"][t])
                # rd state is global; msgs.size() is per shard (the oracle's total is the sum of both)
                assert got["rng"] == want["rng"], t
                assert {k: got[k] for k in ("counters", "scalars", "rows", "levels")} == {k: want[k] for k in ("counters", "scalars", "rows", "levels")}, (t, r["rank"])
            assert r0["digests"][t]["msgs"] + r1["digests"][t]["msgs"] == o.msgs_live(), t
    assert not o.continue_if()
