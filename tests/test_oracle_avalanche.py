"""The CPU restatement of Slush / Snowflake (tests/avalanche_oracle) against the reference's own tests: SlushTest and
SnowflakeTest (testSimple, testCopy), and both protocols running to quiescence."""
import pytest

from tests.avalanche_oracle_lib import OracleSlush, OracleSnowflake
from tests.avalanche_parity import NB, NL


def _one_colour(o):
    s = o.scalars()
    return (s["color"] == s["color"][0]).all()


def test_slush_simple():  # SlushTest.testSimple
    o = OracleSlush(100, 7, 7, 4.0 / 7.0, NB, NL)
    o.init()
    o.run(10)
    assert o.n == 100 and _one_colour(o)


def test_snowflake_simple():  # SnowflakeTest.testSimple
    o = OracleSnowflake(100, 5, 7, 4.0 / 7.0, 3, NB, NL)
    o.init()
    o.run(10)
    assert o.n == 100 and _one_colour(o)


@pytest.mark.parametrize("cls,extra,counter", [(OracleSlush, (), "round"), (OracleSnowflake, (3,), "cnt")])
def test_copy(cls, extra, counter):  # SlushTest.testCopy / SnowflakeTest.testCopy
    a = cls(60, 5, 7, 4.0 / 7.0, *extra, NB, NL)
    b = cls(60, 5, 7, 4.0 / 7.0, *extra, NB, NL)
    a.init(); a.run_ms(200)
    b.init(); b.run_ms(200)
    x, y = a.scalars(), b.scalars()
    for k in ("color", "nonce", counter):
        assert (x[k] == y[k]).all()


@pytest.mark.parametrize("cls,extra", [(OracleSlush, ()), (OracleSnowflake, (3,))])
def test_runs_to_quiescence(cls, extra):
    o = cls(100, 5, 7, 4.0 / 7.0, *extra, NB, NL)
    o.init()
    while o.msgs_size() != 0:
        assert o.time < 60000, "did not go quiet"
        o.run_ms(20)
        o.scalars()
        assert o.max_open <= 1, "more than one query of a node was pending"
    s = o.scalars()
    assert (s["pending"] == 0).all() and (s["color"] > 0).all()
    c = o.counters()
    assert c[0].sum() == c[1].sum()  # no message was lost: every send was received
