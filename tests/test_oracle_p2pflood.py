"""The CPU restatement of P2PFlood (tests/p2p_oracle) pinned on the reference's own P2PFloodTest
(protocols/src/test/java/net/consensys/wittgenstein/protocols/P2PFloodTest.java): testSimpleRun :12-32, testLongRun :34-55
(the full network.run(2000)) and testCopy :57-78, peer lists included."""
import numpy as np

from tests.p2p_oracle_lib import OracleP2PFlood

RANDOM_NB = "RANDOM_SPEED=CONSTANT_TOR=0.00"  # RegistryNodeBuilders.name(RANDOM, true, 0)
AWS_NB = "AWS_SPEED=CONSTANT_TOR=0.00"


def _every_live_node_has_the_message(o, n):
    cnt, down, _ = o.received()
    assert len(cnt) == n
    assert (cnt[down] == 0).all() and (cnt[~down] == 1).all()


def test_simple_run():
    po = OracleP2PFlood(100, 10, 50, 1, 1, 10, 30, RANDOM_NB, "NetworkNoLatency")
    p = OracleP2PFlood(100, 10, 50, 1, 1, 10, 30, RANDOM_NB, "NetworkNoLatency")  # po.copy()
    p.init()
    p.run_ms(20 * 1000)
    po.init()
    _every_live_node_has_the_message(p, 100)


def test_long_run():
    p = OracleP2PFlood(4500, 4000, 500, 1, 1, 50, 300, AWS_NB, "AwsRegionNetworkLatency")
    p.init()
    p.run_ms(2000 * 1000)
    _every_live_node_has_the_message(p, 4500)
    assert max(len(p.peers(i)) for i in range(4500)) > 64  # the degrees the device engine must take


def test_copy():
    args = (2000, 10, 50, 1, 1, 10, 30, RANDOM_NB, "NetworkLatencyByDistanceWJitter")
    p1, p2 = OracleP2PFlood(*args), OracleP2PFlood(*args)
    p1.init()
    p1.run_ms(1000)
    p2.init()
    p2.run_ms(1000)
    assert (p1.counters()[4] == p2.counters()[4]).all()
    c1, d1, _ = p1.received()
    c2, d2, _ = p2.received()
    assert (c1 == c2).all() and (d1 == d2).all()
    for i in range(2000):
        assert np.array_equal(p1.peers(i), p2.peers(i))
    assert p1.avg_peers() == p2.avg_peers() >= 10
