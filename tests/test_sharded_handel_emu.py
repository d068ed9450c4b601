"""Node-sharded Handel (DESIGN.md §8), host logic: the same state-transition bodies, pick exchange and staging path as the CUDA
engine, compiled for the host (tests/emu), G shards driven by G threads of this process, checked against the oracle after every
runMs (rows and level scalars every few steps).  The CUDA kernels run under -m gpu (tests/test_gpu_zz_sharded_handel.py)."""
import numpy as np
import pytest

from tests import emu_handel_lib as emu_lib
from tests.oracle_lib import OracleHandel
from wittgenstein_b200 import HandelParameters, WtgError
from wittgenstein_b200.sharded import ShardedHandel

AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"


def handel_args(n, kind, nb=AWS_NB, nl=AWS_NL, desync=0):
    """(HandelParameters positional arguments, hidden_byzantine) of a run: kind is "suicide", "hidden" or "dead"."""
    return (n, int(n * 0.6), 4, 50, 10, 20, 10, n // 4, nb, nl, desync, kind == "suicide"), kind == "hidden"


def compare(p, o, tag, full):
    bad = []
    net = p.network()
    if net.time != o.time:
        bad.append(f"{tag}: time {net.time} vs {o.time}")
    if net.rng_state() != o.rng_state():
        bad.append(f"{tag}: rd state differs")
    if net.msgs_size() != o.msgs_live():
        bad.append(f"{tag}: msgs.size() {net.msgs_size()} vs {o.msgs_live()}")
    if not (net.counters() == o.counters()).all():
        bad.append(f"{tag}: counters differ")
    a, b = p.scalars(), o.scalars()
    bad += [f"{tag}: scalar {k} differs" for k in a if not (a[k] == b[k]).all()]
    if full:
        bad += [f"{tag}: row {w} differs" for w in range(6) if not (p.rows(w) == o.rows(w)).all()]
        a, b = p.level_scalars(), o.level_scalars()
        bad += [f"{tag}: level scalar {k} differs" for k in a if not (a[k] == b[k]).all()]
    return bad


def check_init(p, o):
    n = p.params.node_count
    nl = n // p.world
    for node in sorted({0, 1, n - 1} | {r * nl + nl // 2 for r in range(p.world)} | {r * nl for r in range(p.world)}):
        assert (p.ranks(node) == o.ranks(node)).all(), f"receptionRanks of node {node}"
        for lv in range(p.levels):
            assert (p.peers(node, lv) == o.peers(node, lv)).all(), f"emission list of node {node} level {lv}"


def run_pair(n, world, until, step, kind, seed=None, full_every=3, hook=None, tunables=None, **kw):
    args, hidden = handel_args(n, kind, **kw)
    p = ShardedHandel(HandelParameters(*args, hidden), world, _api=emu_lib.api(), tunables=tunables)
    o = OracleHandel(*args, hidden_byzantine=hidden, seed=seed)
    if seed is not None:
        p.network().set_seed(seed)
    p.init()
    o.init()
    check_init(p, o)
    i = 0
    while o.time < until:
        if hook:
            hook(p, o)
        assert p.network().run_ms(step) == o.run_ms(step)
        i += 1
        bad = compare(p, o, f"t={o.time}", full=(i % full_every == 0))
        assert not bad, bad
    p.close()
    return o


@pytest.mark.parametrize("n,world,until,step,kind", [(64, 2, 300, 1, "suicide"), (256, 4, 600, 10, "suicide"), (512, 8, 400, 10, "suicide"),
                                                     (256, 2, 500, 7, "hidden"), (1024, 4, 300, 10, "hidden"), (1024, 2, 120, 1, "dead"),
                                                     (2048, 8, 250, 10, "dead")])
def test_handel_sharded_vs_oracle(n, world, until, step, kind):
    run_pair(n, world, until, step, kind, full_every=1 if step == 10 else 5)


def test_handel_sharded_suicide_to_completion():
    """every live node reaches the threshold (Byzantine-suicide, 64 of 256 nodes down, 4 shards)"""
    o = run_pair(256, 4, 2000, 25, "suicide", full_every=4)
    assert (o.counters()[4][o.attrs()["down"] == 0] > 0).all()


def test_handel_sharded_desynchronized_start_tor():
    run_pair(512, 4, 500, 10, "suicide", seed=5, nb="AWS_SPEED=GAUSSIAN_TOR=0.33", desync=120)
    run_pair(256, 2, 400, 10, "dead", nb="RANDOM_SPEED=GAUSSIAN_TOR=0.33", nl=None, desync=60)


def test_handel_sharded_stop_start_partition():
    def hook(p, o):
        t = o.time
        if t == 0:
            live = np.flatnonzero(o.attrs()["down"] == 0)
            hook.a, hook.b = int(live[2]), int(live[-3])  # nodes of the first and the last shard
        if t == 100:
            for x in (p.network(), o):
                x.stop_node(hook.a)
                x.stop_node(hook.b)
        if t == 200:
            p.network().partition(0.4)
            o.partition(0.4)
        if t == 300:
            for x in (p.network(), o):
                x.end_partition()
                x.start_node(hook.a)

    run_pair(256, 4, 500, 10, "suicide", seed=2, hook=hook, full_every=2)


def test_handel_sharded_force_pick_serial():
    """the serial pick path, forced on every pass, gives the parallel path's state bit for bit (and the oracle's)"""
    args, hidden = handel_args(256, "hidden")
    runs = []
    for force in (0, 1):
        p = ShardedHandel(HandelParameters(*args, hidden), 4, _api=emu_lib.api(), tunables={"force_pick_serial": force})
        p.init()
        for _ in range(40):
            p.network().run_ms(10)
        runs.append((p.network().rng_state(), p.network().counters(), p.scalars(), [p.rows(w) for w in range(6)], p.level_scalars()))
        p.close()
    (r0, c0, s0, w0, l0), (r1, c1, s1, w1, l1) = runs
    assert r0 == r1 and (c0 == c1).all()
    assert all((s0[k] == s1[k]).all() for k in s0) and all((l0[k] == l1[k]).all() for k in l0)
    assert all((a == b).all() for a, b in zip(w0, w1))
    run_pair(128, 2, 300, 10, "suicide", tunables={"force_pick_serial": 1})


def test_handel_sharded_read_backs_of_other_shards_refused():
    args, hidden = handel_args(64, "dead")
    p = ShardedHandel(HandelParameters(*args, hidden), 2, _api=emu_lib.api())
    p.init()
    with pytest.raises(WtgError, match="another shard"):
        p.shards[0].peers(40, 3)
    with pytest.raises(WtgError, match="another shard"):
        p.shards[1].ranks(3)
    assert p.shards[1].scalars()["window"].shape == (32,)
    p.close()


def test_handel_sharded_ethscan_refused():
    args, hidden = handel_args(64, "suicide", nl="EthScanNetworkLatency")
    p = ShardedHandel(HandelParameters(*args, hidden), 2, _api=emu_lib.api())
    with pytest.raises(WtgError, match="far-future calendar"):
        p.init()
    p.close()
