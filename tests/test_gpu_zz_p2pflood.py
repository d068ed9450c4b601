"""P2PFlood on the device, through the C ABI, against the CPU restatement (tests/p2p_oracle): bit-exact time, network.rd
position, msgs.size(), node counters and received sets after every runMs window — a subset of the host-build matrix,
P2PFloodTest.testLongRun's configuration over its whole run, floodTime() at 65 536 nodes to completion, and 1 048 576 nodes
over its first 1.5 s (about 18 million deliveries)."""
import pytest

from tests.p2p_parity import AWS_NB, AWS_NL, NB, NL, NO_NL, compare, compare_graph, make, run_compare

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,dead,resend,msgs,peers,between,nl", [
    (100, 10, 50, 1, 10, 30, NO_NL),
    (100, 0, 1, 3, 1, 1, NL),
    (256, 0, 0, 7, 3, 0, NL),
    (300, 10, 500, 1, 10, 300, NL),
    (256, 5, 1, 65, 10, 1, NL),
    (4096, 0, 1, 1, 15, 1, NL),
])
def test_parity(n, dead, resend, msgs, peers, between, nl):
    p, o = make(None, n, dead, resend, msgs, peers, between, NB, nl)
    assert not compare_graph(p, o)
    bad = run_compare(p, o, [1, 3, 7, 13, 50, 200], limit_ms=120000)
    assert not bad, bad[:5]
    assert o.msgs_size() == 0


@pytest.mark.parametrize("seed,force", [(1, 0), (7, 1)])
def test_aws_seeds_and_serial_path(seed, force):
    p, o = make(None, 300, 10, 50, 3, 10, 30, AWS_NB, AWS_NL, seed=seed, tunables={"force_shuffle_serial": force})
    bad = run_compare(p, o, [1, 5, 11, 64], limit_ms=60000)
    assert not bad, bad[:5]
    assert (p.serial_passes() > 0) == bool(force)


def test_stop_and_partition():
    p, o = make(None, 400, 0, 20, 2, 10, 5)
    for _ in range(4):
        p.network().run_ms(15); o.run_ms(15)
    p.network().stop_node(11); o.stop_node(11)
    p.network().partition(0.5); o.partition(0.5)
    bad = run_compare(p, o, [7, 20], until_quiet=False, limit_ms=o.time + 200)
    assert not bad, bad[:5]
    p.network().end_partition(); o.end_partition()
    bad = run_compare(p, o, [50], limit_ms=60000)
    assert not bad, bad[:5]


def test_long_run():
    """P2PFloodTest.testLongRun: 4 500 nodes of which 4 000 dead, 50 peers (degrees near 100), 300 ms between sends, run(2000)"""
    p, o = make(None, 4500, 4000, 500, 1, 50, 300, "AWS_SPEED=CONSTANT_TOR=0.00", AWS_NL)
    assert not compare_graph(p, o)
    assert max(len(p.peers(i)) for i in range(4500)) > 64
    bad = run_compare(p, o, [100000], until_quiet=False, limit_ms=2000000)
    assert not bad, bad[:5]
    cnt = p.received_count()
    down = p.network().attrs()["down"] != 0
    assert (cnt[down] == 0).all() and (cnt[~down] == 1).all()


def test_flood_time_65536():
    """floodTime()'s parameters (P2PFlood.java:172-210) at 65 536 nodes until every live node is done"""
    p, o = make(None, 65536, 0, 1, 1, 15, 1, None, None)
    bad = run_compare(p, o, [10, 100], until_quiet=False, limit_ms=2000)
    assert not bad, bad[:5]
    assert (p.network().counters()[4] > 0).all()


def test_flood_time_1m_prefix():
    n = 1 << 20
    p, o = make(None, n, 0, 1, 1, 15, 1, None, None, tunables={"bcap": n // 4})
    bad = run_compare(p, o, [100], until_quiet=False, limit_ms=1500, bitmaps=False)
    assert not bad, bad[:5]
    assert p.network().stats()["deliveries"] == o.deliveries() > 10 * n
