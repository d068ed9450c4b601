"""Node-sharded CasperIMD (BASELINE config #4: "CasperIMD ... node-sharded across 4xH100"; DESIGN.md §8), host logic: the
same state-transition bodies and exchange protocol as the CUDA engine, compiled for the host (tests/emu), G shards driven by
G threads, checked bit for bit against the oracle — replicated block / attestation tables, sendAll records built on every
shard, the far-future calendar with ordering keys, and the per-pass "next event" minimum of the fast-forward.
The CUDA kernels of these stages run under -m gpu (tests/test_gpu_zz_sharded_casper.py)."""
import pytest

from tests import emu_lib
from tests.oracle_lib import OracleCasper
from tests.parity import compare_casper
from wittgenstein_b200 import CasperParemeters
from wittgenstein_b200.sharded import ShardedCasperIMD

RANDOM_NB, DIST_NL = "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"


def run_pair(args, world, steps, step, byz_delay=0, byz_kind="WF", votes=12, hook=None, atts_every=0):
    p = ShardedCasperIMD(CasperParemeters(*args), world, _api=emu_lib.api(), tunables={"casper_votes": votes})
    o = OracleCasper(*args)
    p.init(byz_delay, byz_kind); o.init(byz_delay, byz_kind)
    for k in range(steps):
        if hook:
            hook(k, p, o)
        assert p.network().run_ms(step) == o.run_ms(step), f"runMs return at t={o.time}"
        bad = compare_casper(p, o, f"t={o.time}", atts=bool(atts_every) and k % atts_every == atts_every - 1)
        assert not bad, bad
    assert not compare_casper(p, o, "end", atts=True)
    p.close()


@pytest.mark.parametrize("world", [2, 4])
def test_casper_sharded_vs_oracle(world):
    # 1 + 3 + 12 = 16 nodes: the id ranges are uneven (16 / 4 here, 16390 / 4 in config #4)
    run_pair((2, False, 3, 6, 1000, 1, None, None), world, 60, 2000, byz_delay=9000)


def test_casper_sharded_uneven_ranges_and_latency_models():
    # 1 + 2 + 20 = 23 nodes on 4 shards (6, 6, 6, 5) with the shipped builder / latency of config #4
    run_pair((4, False, 2, 5, 1000, 1, RANDOM_NB, DIST_NL), 4, 40, 4000)
    # AWS positions + Tor: long and varied latencies, many arrival groups per sendAll
    run_pair((3, False, 3, 7, 1000, 1, "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"), 2, 40, 3000, byz_delay=-3000)


@pytest.mark.parametrize("kind", ["plain", "SF", "NS"])
def test_casper_sharded_byzantine_producers(kind):
    run_pair((2, False, 3, 6, 1000, 1, None, None), 2, 40, 2000, byz_delay=0 if kind != "plain" else 3000, byz_kind=kind)


def test_casper_sharded_odd_slicing_and_stopped_nodes():
    def hook(k, p, o):
        if k == 5:
            p.network().stop_node(7); o.stop_node(7)
            p.network().stop_node(12); o.stop_node(12)
        if k == 25:
            p.network().start_node(7); o.start_node(7)

    run_pair((2, False, 3, 6, 1000, 1, None, None), 4, 90, 777, byz_delay=9000, hook=hook)


def test_casper_sharded_config4_shape_small():
    """config #4's shape at a size the host build runs in seconds: 1 + 5 producers + 64 x 4 attesters = 262 nodes on 4 shards
    (ranges 66, 66, 66, 64), shipped node builder / latency, two cycles of 4 slots"""
    run_pair((4, False, 5, 64, 1000, 1, RANDOM_NB, DIST_NL), 4, 16, 8000, votes=4, atts_every=8)
