"""Node-sharded Handel on the device (DESIGN.md §8): G engines, one shard of the node ids each, with the pick exchange before
checkSigs' level draws and pooled payloads staged on the receiving shard — bit-exact against the oracle and against the
unsharded engine.  With one GPU the shards share it (separate streams); with several GPUs in the box each shard gets its own."""
import json
import os

import numpy as np
import pytest

from tests.oracle_lib import OracleHandel
from tests.test_sharded_handel_emu import check_init, compare, handel_args

pytestmark = pytest.mark.gpu


def devices_for(world):
    import torch

    n = torch.cuda.device_count()
    return [r % n for r in range(world)]


def sharded(args, hidden, world, devices=None, tunables=None):
    from wittgenstein_b200 import HandelParameters
    from wittgenstein_b200.sharded import ShardedHandel

    return ShardedHandel(HandelParameters(*args, hidden), world, devices=devices or devices_for(world), tunables=tunables)


@pytest.mark.parametrize("n,world,until,step,kind", [(256, 2, 600, 10, "suicide"), (512, 4, 400, 1, "hidden"), (1024, 8, 400, 10, "dead"),
                                                     (1024, 4, 300, 10, "hidden")])
def test_handel_sharded_small_vs_oracle(n, world, until, step, kind):
    args, hidden = handel_args(n, kind)
    p = sharded(args, hidden, world)
    o = OracleHandel(*args, hidden_byzantine=hidden)
    p.init()
    o.init()
    check_init(p, o)
    i = 0
    while o.time < until:
        assert p.network().run_ms(step) == o.run_ms(step)
        i += 1
        bad = compare(p, o, f"t={o.time}", full=(i % 5 == 0))
        assert not bad, bad
    p.close()


def test_handel_sharded_suicide_to_completion_vs_oracle():
    args, hidden = handel_args(512, "suicide")
    p = sharded(args, hidden, 4, tunables={"force_pick_serial": 1})
    o = OracleHandel(*args, hidden_byzantine=hidden)
    p.init()
    o.init()
    while o.continue_if() or p.continue_if():
        assert o.time < 5000, "the run did not complete"
        assert p.network().run_ms(20) == o.run_ms(20)
        bad = compare(p, o, f"t={o.time}", full=True)
        assert not bad, bad
    p.close()


def test_handel_sharded_4096_equals_unsharded_to_completion():
    """4 shards on one GPU against the unsharded engine: every read-back, rd state, msgs.size() and peekMessages"""
    from wittgenstein_b200 import Handel, HandelParameters

    args, hidden = handel_args(4096, "suicide")
    p = sharded(args, hidden, 4, devices=[0, 0, 0, 0])
    u = Handel(HandelParameters(*args, hidden))
    p.init()
    u.init()
    step = 0
    while u.continue_if() or p.continue_if():
        assert u.network().time < 6000, "the run did not complete"
        assert p.network().run_ms(25) == u.network().run_ms(25)
        step += 1
        pn, un = p.network(), u.network()
        t = un.time
        assert pn.rng_state() == un.rng_state() and pn.msgs_size() == un.msgs_size(), t
        assert (pn.counters() == un.counters()).all(), t
        a, b = p.scalars(), u.scalars()
        assert all((a[k] == b[k]).all() for k in a), t
        if step % 4 == 0:
            assert all((p.rows(w) == u.rows(w)).all() for w in range(6)), t
            a, b = p.level_scalars(), u.level_scalars()
            assert all((a[k] == b[k]).all() for k in a), t
            ta, ra = pn.peek_messages(1 << 20)
            tb, rb = un.peek_messages(1 << 20)
            assert ta == tb and all((ra[k] == rb[k]).all() for k in ra), t
    assert all((p.rows(w) == u.rows(w)).all() for w in range(6))
    for node in (0, 1234, 2048, 4095):
        assert (p.ranks(node) == u.ranks(node)).all()
        assert all((p.peers(node, lv) == u.peers(node, lv)).all() for lv in range(p.levels))
    p.close()


@pytest.mark.parametrize("world", [2, 4])
def test_handel_32768_config3_sharded_against_offline_oracle_digests(world):
    """BASELINE config #3 (Handel 32 768 nodes, 8 192 suicide-Byzantine, AWS latencies) on 2 and 4 shards: the concatenated
    read-backs against the oracle digests produced offline (tests/golden/make_handel32768.py) at every committed checkpoint"""
    from tests.parity import handel_digests

    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "handel32768_config3.json")
    fx = json.load(open(path))
    prm = fx["params"]
    p = sharded(tuple(prm[:8]) + (prm[8], prm[9], prm[10], prm[11]), prm[12], world)
    p.init()
    last = max(int(t) for t in fx["checkpoints"])
    assert last >= 300
    while p.network().time < last:
        p.network().run_ms(100)
        want = fx["checkpoints"].get(str(p.network().time))
        if want is not None:
            got = handel_digests(p, False)
            assert got == want, (world, p.network().time, {k: (got[k], want[k]) for k in got if got[k] != want[k]})
    p.close()
