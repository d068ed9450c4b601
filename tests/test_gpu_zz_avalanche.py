"""Slush / Snowflake on the device, through the C ABI, against the CPU restatement (tests/avalanche_oracle): bit-exact node
state, counters, msgs.size() and network.rd position after every runMs window, including the serial re-derivation of a
pass's draw indices that sample collisions force, and 65 536 nodes over a prefix of the run."""
import pytest

from tests.avalanche_parity import AWS_NB, AWS_NL, NB, NL, compare, make, run_compare

pytestmark = pytest.mark.gpu

PROTOS = ["slush", "snowflake"]


@pytest.mark.parametrize("proto", PROTOS)
@pytest.mark.parametrize("n,k", [(60, 1), (64, 2), (100, 7), (100, 20), (1000, 7), (1000, 20)])
def test_parity(proto, n, k):
    p, o = make(proto, None, n, k, NB, NL)
    bad = run_compare(p, o, [1, 3, 7, 13, 50], limit_ms=20000)
    assert not bad, bad[:5]
    assert o.msgs_size() == 0


@pytest.mark.parametrize("proto", PROTOS)
@pytest.mark.parametrize("seed,force", [(1, 0), (7, 1)])
def test_parity_aws_seeds(proto, seed, force):
    p, o = make(proto, None, 100, 7, AWS_NB, AWS_NL, seed=seed, tunables={"force_shuffle_serial": force})
    bad = run_compare(p, o, [1, 5, 11, 64], limit_ms=20000)
    assert not bad, bad[:5]
    assert p.serial_passes() > 0


@pytest.mark.parametrize("proto", PROTOS)
def test_stop_and_partition(proto):
    p, o = make(proto, None, 100, 7, NB, NL)
    for _ in range(6):
        p.network().run_ms(5); o.run_ms(5)
    p.network().stop_node(11); o.stop_node(11)
    for _ in range(3):
        p.network().run_ms(5); o.run_ms(5)
    p.network().partition(0.5); o.partition(0.5)
    bad = run_compare(p, o, [7, 20], limit_ms=20000)
    assert not bad, bad[:5]


@pytest.mark.parametrize("proto", PROTOS)
def test_65536_nodes_prefix(proto):
    p, o = make(proto, None, 65536, 7, NB, NL)
    """the first second: every node is coloured by then and about a million answers have been delivered"""
    bad = run_compare(p, o, [100], until_quiet=False, limit_ms=1000)
    assert not bad, bad[:5]
    assert (p.scalars()["color"] > 0).all()
    assert p.network().stats()["deliveries"] == o.deliveries() > 500000


def test_error_paths():
    from wittgenstein_b200 import Network, Slush, SlushParameters, Snowflake, SnowflakeParameters, WtgError, _lib

    for n, k in [(100, 0), (100, 100), (200, 64)]:
        with pytest.raises(WtgError, match="K must be in"):
            Slush(SlushParameters(n, 4, k, 0.5)).init()
        with pytest.raises(WtgError, match="K must be in"):
            Snowflake(SnowflakeParameters(n, 4, k, 0.5, 3)).init()
    api = _lib.api()
    net = Network(api, shard=(0, 2))
    with pytest.raises(WtgError, match="node-sharded"):
        api.check(api.slush_init(net.h, 64, 4, 7, 0.5))
    net.close()
    # a run that outgrows the bucket capacity fails loudly instead of dropping arrivals
    p = Slush(SlushParameters(4096, 4, 20, 4.0 / 7.0, NB, NL), tunables={"bcap": 64})
    p.init()
    with pytest.raises(WtgError):
        for _ in range(100):
            p.network().run_ms(10)
