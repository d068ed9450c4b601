"""P2PFlood on the host build of the device bodies (tests/emu) against the CPU restatement (tests/p2p_oracle), compared after
every runMs window: time, network.rd position, msgs.size(), the five node counters, every node's received count and (several
messages) bitmap, and the peer graph.  Covers the shuffle of every forward's peer list in the emit step (emitPeers), forwards
to an empty list (they still draw their seed), the far-future calendar of long delays between sends, and the serial
re-derivation of draw indices."""
import numpy as np
import pytest

from tests import emu_lib
from tests.p2p_oracle_lib import OracleP2PFlood
from tests.p2p_parity import AWS_NB, AWS_NL, NB, NL, NO_NL, compare, compare_graph, make, run_compare


@pytest.fixture(scope="module")
def api():
    return emu_lib.api()


# (nodes, dead, delayBeforeResent, msgCount, peersCount, delayBetweenSends, latency, tunables)
CASES = [
    (100, 10, 50, 1, 10, 30, NO_NL, None),   # P2PFloodTest.testSimpleRun
    (100, 0, 1, 1, 1, 1, NL, None),          # peersCount 1: many forwards go to an empty list
    (256, 0, 0, 7, 3, 0, NL, None),          # delay 0: MultipleDestEnvelope
    (512, 0, 1, 1, 15, 1, NL, None),         # floodTime()'s parameters
    (300, 10, 500, 1, 10, 300, NL, None),    # arrivals far beyond the ring: calendar and fast-forward
    (256, 0, 1, 64, 10, 1, NL, None),
    (256, 5, 1, 65, 10, 1, NL, None),        # a second bitmap word
    (256, 0, 0, 256, 10, 0, NL, {"bcap": 1 << 16}),
    (200, 0, 50, 0, 10, 30, NL, None),       # no message at all
    (1000, 0, 1, 1, 50, 1, NL, None),
    (4096, 0, 1, 1, 15, 1, NL, None),
]


@pytest.mark.parametrize("n,dead,resend,msgs,peers,between,nl,tun", CASES)
def test_parity(api, n, dead, resend, msgs, peers, between, nl, tun):
    p, o = make(api, n, dead, resend, msgs, peers, between, NB, nl, tunables=tun)
    assert not compare_graph(p, o)
    bad = run_compare(p, o, [1, 3, 7, 13, 50, 200], limit_ms=120000)
    assert not bad, bad[:5]
    assert o.msgs_size() == 0


def test_parity_aws_tor(api):
    p, o = make(api, 300, 10, 50, 1, 10, 30, AWS_NB, AWS_NL)
    assert not compare_graph(p, o)
    bad = run_compare(p, o, [1, 5, 11, 64], limit_ms=60000)
    assert not bad, bad[:5]


def test_empty_forwards_take_the_parallel_path(api):
    """with peersCount = 1 about a third of the forwards have no destination; each still draws its seed, and the
    optimistic draw indices account for it: no pass needs the serial re-derivation"""
    p, o = make(api, 400, 0, 1, 3, 1, 1)
    bad = run_compare(p, o, [2, 5], limit_ms=60000)
    assert not bad, bad[:5]
    assert p.serial_passes() == 0
    assert any(len(p.peers(i)) == 1 for i in range(400))


@pytest.mark.parametrize("seed", [1, 7])
@pytest.mark.parametrize("force", [0, 1])
def test_seeds_and_serial_path(api, seed, force):
    p, o = make(api, 300, 5, 1, 3, 10, 1, seed=seed, tunables={"force_shuffle_serial": force})
    bad = run_compare(p, o, [1, 9, 17], limit_ms=60000)
    assert not bad, bad[:5]
    assert (p.serial_passes() > 0) == bool(force)


def test_stop_and_partition_mid_run(api):
    p, o = make(api, 400, 0, 20, 2, 10, 5)
    for _ in range(4):
        p.network().run_ms(15); o.run_ms(15)
    for i in (3, 40, 77):
        p.network().stop_node(i); o.stop_node(i)
    bad = run_compare(p, o, [5], until_quiet=False, limit_ms=o.time + 40)
    assert not bad, bad[:5]
    p.network().partition(0.5); o.partition(0.5)
    bad = run_compare(p, o, [7, 20], until_quiet=False, limit_ms=o.time + 200)
    assert not bad, bad[:5]
    p.network().end_partition(); o.end_partition()
    p.network().start_node(40); o.start_node(40)
    bad = run_compare(p, o, [50], limit_ms=60000)
    assert not bad, bad[:5]


def test_peek_messages(api):
    """network.msgs.peekMessages() at two points of a run with delays between sends"""
    p, o = make(api, 300, 10, 50, 2, 10, 30)
    for t in (60, 400):
        p.network().run_ms(t - p.network().time); o.run_ms(t - o.time)
        tot, rows = p.network().peek_messages()
        otot, orows = o.peek_messages()
        assert tot == otot > 0
        for k in ("from", "to", "sent_at", "arriving_at"):
            assert np.array_equal(rows[k], orows[k]), (t, k)


def test_refusals(api):
    from wittgenstein_b200 import Network, P2PFlood, P2PFloodParameters, WtgError

    def init(*a):
        P2PFlood(P2PFloodParameters(*a), _api=api).init()

    with pytest.raises(WtgError, match="Wrong configuration"):
        init(50, 0, 1, 1, 1, 50, 1)
    with pytest.raises(WtgError, match="live nodes"):
        init(100, 10, 1, 91, 1, 10, 1)
    for bad in [(100, -1, 1, 1, 1, 10, 1), (100, 0, -1, 1, 1, 10, 1), (100, 0, 1, -1, 1, 10, 1), (100, 0, 1, 1, 1, -1, 1),
                (100, 0, 1, 1, 1, 10, -1), (0, 0, 1, 0, 1, 0, 1)]:
        with pytest.raises(WtgError, match="negative"):
            init(*bad)
    with pytest.raises(WtgError, match="delayBetweenSends"):
        init(100, 0, 1, 1, 1, 10, 1 << 20)
    with pytest.raises(WtgError, match="delayBeforeResent"):
        init(100, 0, 1 << 30, 1, 1, 10, 1)
    with pytest.raises(WtgError, match="degree"):  # peersCount 200 at 400 nodes: degrees well above 256
        init(400, 0, 1, 1, 1, 200, 1)
    with pytest.raises(WtgError, match="record arenas"):
        init(1 << 20, 0, 1, 1 << 12, 1, 15, 1)
    net = Network(api, shard=(0, 2))
    with pytest.raises(WtgError, match="node-sharded"):
        api.check(api.p2pflood_init(net.h, 64, 0, 1, 1, 10, 1))
    from wittgenstein_b200 import PingPong, PingPongParameters

    pp = PingPong(PingPongParameters(10), _api=api)
    pp.init()
    with pytest.raises(WtgError, match="not a P2PFlood"):
        api.check(api.p2p_avg_peers(pp.network().h))


def test_copy(api):  # P2PFloodTest.testCopy on the engine
    p1, o = make(api, 2000, 10, 50, 1, 10, 30)
    p2 = p1.copy()
    p2.init()
    p1.network().run_ms(1000)
    p2.network().run_ms(1000)
    o.run_ms(1000)
    assert not compare(p1, o) and not compare(p2, o)
    assert not compare_graph(p1, o) and not compare_graph(p2, o)


def test_run_multiple_times(api):
    """P2PFlood.time() at N = 128: RunMultipleTimes over 5 seeds (contUntilDone) equals the oracle run seed by seed"""
    from wittgenstein_b200 import DoneAtStatGetter, MsgReceivedStatGetter, P2PFlood, P2PFloodParameters, RunMultipleTimes, cont_until_done
    from wittgenstein_b200.run_multiple import avg, get_stats_on

    n = 128
    rmt = RunMultipleTimes(P2PFlood(P2PFloodParameters(n, 0, 1, n, 1, 13, 0), _api=api), 5, 0,
                           [DoneAtStatGetter(), MsgReceivedStatGetter()])
    res = rmt.run(cont_until_done, concurrency=1)
    done, rcv = [], []
    for seed in range(5):
        o = OracleP2PFlood(n, 0, 1, n, 1, 13, 0, seed=seed)
        o.init()
        while True:
            did = o.run_ms(10)
            if not (not did or (o.counters()[4] == 0).any()):
                break
        assert o.time == rmt.end_times[seed]
        done.append(get_stats_on(o.counters()[4]))
        rcv.append(get_stats_on(o.counters()[0]))
    assert res[0] == avg(done) and res[1] == avg(rcv)
