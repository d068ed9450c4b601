"""GSF's checkSigs of the next millisecond run ahead, beside the current millisecond's emission (DESIGN.md §4): host build of
the device logic against the oracle after every runMs, with the next pass's checkSigs placed before this pass's emission
(cond_ahead = 1) and after it (cond_ahead = 2), the two ends of what the device's two branches allow.  Windows of 1, 3, 4,
5 and 97 ms run the single-pass, first, middle and last pass shapes; stop / start and partitions change the network between
windows; EthScan latencies go through the far-future calendar."""
import pytest

from tests import emu_cond_ahead_lib
from tests.oracle_lib import OracleGSF
from tests.parity import compare_gsf
from wittgenstein_b200 import GSFSignature, GSFSignatureParameters

AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"
WINDOWS = [1, 3, 4, 5, 97]


def pair(args, seed, order, pool=0):
    p = GSFSignature(GSFSignatureParameters(*args), _api=emu_cond_ahead_lib.api())
    p.network().set_tunable("cond_ahead", order)
    if pool:
        p.network().set_tunable("pool_slots_per_node", pool)
    p.network().set_seed(seed)
    o = OracleGSF(*args, seed=seed)
    p.init(); o.init()
    return p, o


def step(p, o, ms, full=True):
    assert p.network().run_ms(ms) == o.run_ms(ms)
    bad = compare_gsf(p, o, f"t={o.time}", full=full)
    assert not bad, bad


@pytest.mark.parametrize("order", [1, 2])
@pytest.mark.parametrize("n,seed", [(64, 0), (64, 7), (512, 0), (512, 7)])
def test_cond_ahead_windows(n, seed, order):
    args = (n, int(0.8 * n), 3, 20, 10, 10, n // 10, AWS_NB, AWS_NL)
    p, o = pair(args, seed, order, pool=96)  # the partition holds signatures back: more pooled entries than the default
    for k in range(40):
        if k == 8:
            p.network().stop_node(n // 3); o.stop_node(n // 3)
        if k == 14:
            p.network().start_node(n // 3); o.start_node(n // 3)
        if k == 16:
            p.network().partition(0.5); o.partition(0.5)
        if k == 20:
            p.network().end_partition(); o.end_partition()
        step(p, o, WINDOWS[k % len(WINDOWS)])


@pytest.mark.parametrize("order", [1, 2])
def test_cond_ahead_4096(order):
    n = 4096
    args = (n, int(0.8 * n), 3, 20, 10, 10, n // 10, AWS_NB, AWS_NL)
    p, o = pair(args, 3, order)
    for k, ms in enumerate(WINDOWS * 3):
        step(p, o, ms, full=(k % 5 == 4))


@pytest.mark.parametrize("order", [1, 2])
def test_cond_ahead_far_calendar(order):
    n = 128
    args = (n, int(0.8 * n), 3, 20, 10, 10, n // 16, "RANDOM_SPEED=CONSTANT_TOR=0.00", "EthScanNetworkLatency")
    p, o = pair(args, 0, order)
    assert p.network().stats()["ring"] == 4096
    for k in range(30):
        step(p, o, WINDOWS[k % len(WINDOWS)] * 20, full=(k % 5 == 0))


def test_cond_ahead_off_matches():
    """cond_ahead = 0: every pass runs its own checkSigs, as node-sharded engines and the other protocols do"""
    args = (64, 52, 3, 20, 10, 10, 6, AWS_NB, AWS_NL)
    p, o = pair(args, 3, 0)
    for k in range(20):
        step(p, o, WINDOWS[k % len(WINDOWS)])


def test_cond_ahead_rejects_other_values():
    p = GSFSignature(GSFSignatureParameters(64, 52, 3, 20, 10, 10, 6, AWS_NB, AWS_NL), _api=emu_cond_ahead_lib.api())
    with pytest.raises(Exception):
        p.network().set_tunable("cond_ahead", 3)
