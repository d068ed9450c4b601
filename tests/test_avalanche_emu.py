"""Slush / Snowflake on the host build of the device bodies (tests/emu) against the CPU restatement, compared after every
runMs window: node state, counters, msgs.size() and the position of network.rd.  Covers the draw of every query's sample
in the emit step, including the serial re-derivation of a pass's draw indices that a discarded attempt (the sender itself
or a repeated id) forces."""
import pytest

from tests import emu_lib
from tests.avalanche_parity import AWS_NB, AWS_NL, NB, NL, compare, make, run_compare

PROTOS = ["slush", "snowflake"]


@pytest.fixture(scope="module")
def api():
    return emu_lib.api()


@pytest.mark.parametrize("proto", PROTOS)
@pytest.mark.parametrize("n,k", [(60, 1), (60, 20), (64, 2), (64, 7), (100, 1), (100, 2), (100, 7), (100, 20), (1000, 7), (1000, 20)])
def test_parity(api, proto, n, k):
    p, o = make(proto, api, n, k, NB, NL)
    bad = run_compare(p, o, [1, 3, 7, 13, 50], limit_ms=20000 if n < 1000 else 4000)
    assert not bad, bad[:5]


@pytest.mark.parametrize("proto", PROTOS)
@pytest.mark.parametrize("n,k", [(64, 7), (100, 20)])
def test_parity_aws(api, proto, n, k):
    p, o = make(proto, api, n, k, AWS_NB, AWS_NL)
    bad = run_compare(p, o, [1, 5, 11, 64], limit_ms=20000)
    assert not bad, bad[:5]


@pytest.mark.parametrize("proto", PROTOS)
@pytest.mark.parametrize("seed", [1, 7])
@pytest.mark.parametrize("force", [0, 1])
def test_seeds_and_serial_path(api, proto, seed, force):
    p, o = make(proto, api, 100, 7, NB, NL, seed=seed, tunables={"force_shuffle_serial": force})
    bad = run_compare(p, o, [1, 9, 17], limit_ms=20000)
    assert not bad, bad[:5]
    if force:
        assert p.serial_passes() > 0


@pytest.mark.parametrize("proto", PROTOS)
def test_collisions_reach_the_serial_path_unforced(api, proto):
    """at N = 100, K = 7 about a quarter of the queries draw more than K values: the serial path runs without any forcing"""
    p, o = make(proto, api, 100, 7, NB, NL)
    bad = run_compare(p, o, [10], limit_ms=20000)
    assert not bad, bad[:5]
    assert p.serial_passes() > 0


@pytest.mark.parametrize("proto", PROTOS)
def test_stop_node(api, proto):
    p, o = make(proto, api, 100, 7, NB, NL)
    for _ in range(8):
        p.network().run_ms(5); o.run_ms(5)
    for i in (3, 40):
        p.network().stop_node(i); o.stop_node(i)
    bad = run_compare(p, o, [3, 10], limit_ms=20000)
    assert not bad, bad[:5]


@pytest.mark.parametrize("proto", PROTOS)
def test_partition_mid_run(api, proto):
    """queries across the partition are lost: their Answer never completes and the node stops querying, as in the reference"""
    p, o = make(proto, api, 100, 7, NB, NL)
    for _ in range(10):
        p.network().run_ms(4); o.run_ms(4)
    p.network().partition(0.5); o.partition(0.5)
    bad = run_compare(p, o, [7, 20], limit_ms=20000)
    assert not bad, bad[:5]
    assert p.scalars()["pending"].sum() > 0
    p.network().end_partition(); o.end_partition()
    bad = run_compare(p, o, [50], until_quiet=False, limit_ms=o.time + 500)
    assert not bad, bad[:5]


def test_refusals(api):
    from wittgenstein_b200 import Network, Slush, SlushParameters, Snowflake, SnowflakeParameters, WtgError

    for n, k in [(100, 0), (100, 100), (100, 150), (200, 64), (1, 1)]:
        for p in (Slush(SlushParameters(n, 4, k, 0.5), _api=api), Snowflake(SnowflakeParameters(n, 4, k, 0.5, 3), _api=api)):
            with pytest.raises(WtgError):
                p.init()
    with pytest.raises(WtgError, match="K must be in"):
        Slush(SlushParameters(100, 4, 0, 0.5), _api=api).init()
    with pytest.raises(WtgError, match="B must be"):
        Snowflake(SnowflakeParameters(100, 4, 7, 0.5, -1), _api=api).init()
    net = Network(api, shard=(0, 2))
    with pytest.raises(WtgError, match="node-sharded"):
        api.check(api.slush_init(net.h, 64, 4, 7, 0.5))
    with pytest.raises(WtgError, match="node-sharded"):
        api.check(api.snowflake_init(net.h, 64, 4, 7, 0.5, 3))
    # the read-back refuses a network of another protocol
    import ctypes as C

    import numpy as np
    from wittgenstein_b200 import PingPong, PingPongParameters

    pp = PingPong(PingPongParameters(10), _api=api)
    pp.init()
    out = [np.zeros(10, np.int32) for _ in range(6)]
    with pytest.raises(WtgError, match="not a Slush or Snowflake"):
        api.check(api.avalanche_node_scalars(pp.network().h, *[x.ctypes.data_as(C.POINTER(C.c_int)) for x in out]))


@pytest.mark.parametrize("proto", PROTOS)
def test_copy(api, proto):  # SlushTest.testCopy / SnowflakeTest.testCopy on the engine
    p1, _ = make(proto, api, 60, 7, NB, NL, m=5)
    p2 = p1.copy()
    p2.init()
    p1.network().run_ms(200)
    p2.network().run_ms(200)
    a, b = p1.scalars(), p2.scalars()
    assert all((a[k] == b[k]).all() for k in a)
    assert p1.network().rng_state() == p2.network().rng_state()
    assert not compare(p1, _oracle_like(p2))


def _oracle_like(p):
    """a second engine run seen through the oracle's read-back names (for compare())"""
    net = p.network()

    class View:
        time = net.time
        rng_state = staticmethod(net.rng_state)
        msgs_size = staticmethod(net.msgs_size)
        counters = staticmethod(net.counters)
        scalars = staticmethod(p.scalars)

    return View()
