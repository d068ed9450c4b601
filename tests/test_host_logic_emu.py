"""CPU-side regression of the host logic (engine orchestration, init paths, C-ABI argument handling, read-backs) and of the
state-transition bodies shared between the CUDA kernels and the host debugging build (tests/emu): every protocol, a short
run, bit-for-bit against the oracle.  TEST INFRASTRUCTURE: the debugging build exports wtgemu_* symbols and is never loaded
by the product; the parity tests proper (-m gpu) run the CUDA path through the C ABI on an H100."""
import numpy as np
import pytest

from tests import emu_lib
from tests.oracle_lib import OracleCappos, OracleCasper, OracleGSF, OracleHandel, OraclePingPong, OracleSanFermin
from tests.parity import compare_casper, compare_gsf

NB, NL = "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"
AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"


@pytest.fixture(scope="module")
def api():
    return emu_lib.api()


def test_pingpong(api):
    from wittgenstein_b200 import PingPong, PingPongParameters

    p = PingPong(PingPongParameters(100, None, None), _api=api)
    o = OraclePingPong(100, None, None)
    p.init(); o.init()
    for _ in range(8):
        assert p.network().run_ms(50) == o.run_ms(50)
        assert (p.pongs() == o.pongs()).all() and (p.network().counters() == o.counters()).all()
    p.network().send(1, 3, [5, 6, 7], send_time=p.network().time + 4, delay_between=5)
    o.send(1, 3, [5, 6, 7], send_time=o.time + 4, delay_between=5)
    assert p.network().run_ms(300) == o.run_ms(300)
    assert (p.network().counters() == o.counters()).all() and p.network().rng_state() == o.rng_state()


def test_gsf(api):
    from wittgenstein_b200 import GSFSignature, GSFSignatureParameters

    args = (64, 52, 3, 20, 10, 10, 6, AWS_NB, AWS_NL)
    p = GSFSignature(GSFSignatureParameters(*args), _api=api)
    o = OracleGSF(*args, seed=3)
    p.network().set_seed(3)
    p.init(); o.init()
    for k in range(60):
        if k == 10:
            p.network().stop_node(9); o.stop_node(9)
        assert p.network().run_ms(10) == o.run_ms(10)
        bad = compare_gsf(p, o, f"t={o.time}")
        assert not bad, bad


@pytest.mark.parametrize("k", [1, 5])
def test_sanfermin(api, k):
    from wittgenstein_b200 import SanFerminSignature, SanFerminSignatureParameters

    p = SanFerminSignature(SanFerminSignatureParameters(64, 64, 2, 48, 300, k, False, None, None), _api=api)
    o = OracleSanFermin(64, 64, 2, 48, 300, k, None, None)
    p.init(); o.init()
    for _ in range(150):
        assert p.network().run_ms(10) == o.run_ms(10)
    a, b = p.scalars(), o.scalars()
    assert all((a[x] == b[x]).all() for x in a)
    assert (p.network().counters() == o.counters()).all() and p.network().rng_state() == o.rng_state()


def test_cappos(api):
    from wittgenstein_b200 import SanFerminCappos, SanFerminCapposParameters

    p = SanFerminCappos(SanFerminCapposParameters(128, 64, 2, 48, 150, 20, None, None), _api=api, tunables={"force_shuffle_serial": 1})
    o = OracleCappos(128, 64, 2, 48, 150, 20, None, None)
    p.init(); o.init()
    for _ in range(200):
        assert p.network().run_ms(10) == o.run_ms(10)
    a, b = p.scalars(), o.scalars()
    assert all((a[x] == b[x]).all() for x in a)
    assert (p.network().counters() == o.counters()).all() and p.network().rng_state() == o.rng_state()


@pytest.mark.parametrize("suicide,hidden", [(True, False), (False, True)])
def test_handel(api, suicide, hidden):
    from wittgenstein_b200 import Handel, HandelParameters

    args = (64, 40, 4, 50, 10, 20, 10, 16, NB, NL, 0, suicide)
    p = Handel(HandelParameters(*args, hidden), _api=api)
    o = OracleHandel(*args, hidden_byzantine=hidden)
    p.init(); o.init()
    for _ in range(120):
        assert p.network().run_ms(10) == o.run_ms(10)
    a, b = p.scalars(), o.scalars()
    assert all((a[x] == b[x]).all() for x in a)
    for w in range(6):
        assert (p.rows(w) == o.rows(w)).all()
    assert (p.network().counters() == o.counters()).all() and p.network().rng_state() == o.rng_state()


def test_casper(api):
    from wittgenstein_b200 import CasperIMD, CasperParemeters

    p = CasperIMD(CasperParemeters(2, False, 3, 6, 1000, 1, None, None), _api=api)
    o = OracleCasper(2, False, 3, 6, 1000, 1, None, None)
    p.network().set_tunable("casper_votes", 12)
    p.init(9000); o.init(9000)
    for k in range(60):
        if k == 20:
            p.network().partition(0.5); o.partition(0.5)
        if k == 30:
            p.network().end_partition(); o.end_partition()
        assert p.network().run_ms(2000) == o.run_ms(2000)
        bad = compare_casper(p, o, f"t={o.time}")
        assert not bad, bad
    assert not compare_casper(p, o, "end", atts=True)


def test_pingpong_caller_sends_to_many_destinations(api):
    """network.send(msg, from, dests) with more destinations than any handler uses (Network.java:352-362): 300 and 40 destinations,
    with and without delaysBetweenMessage, stopped nodes among them"""
    from wittgenstein_b200 import PingPong, PingPongParameters

    p = PingPong(PingPongParameters(400, None, None), _api=api)
    o = OraclePingPong(400, None, None)
    p.init(); o.init()
    p.network().run_ms(300); o.run_ms(300)
    for i in (5, 77, 399):
        p.network().stop_node(i); o.stop_node(i)
    d1 = [(7 * k + 3) % 400 for k in range(300)]
    p.network().send(1, 2, d1); o.send(1, 2, d1)
    d2 = list(range(399, 359, -1))
    p.network().send(1, 9, d2, send_time=p.network().time + 10, delay_between=3)
    o.send(1, 9, d2, send_time=o.time + 10, delay_between=3)
    assert p.network().msgs_size() == o.msgs_size()
    for _ in range(12):
        assert p.network().run_ms(50) == o.run_ms(50)
        assert (p.pongs() == o.pongs()).all() and (p.network().counters() == o.counters()).all()
    assert p.network().rng_state() == o.rng_state() and p.network().msgs_size() == o.msgs_size() == 0
