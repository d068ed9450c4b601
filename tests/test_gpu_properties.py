"""Size-independent properties of the GPU engine at sizes the oracle cannot reach in seconds."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"


def popcount_rows(a):
    return np.unpackbits(a.view(np.uint8), axis=1).sum(axis=1)


def make(n, tun=None):
    from wittgenstein_b200 import GSFSignature, GSFSignatureParameters

    p = GSFSignature(GSFSignatureParameters(n, 0.85, 4, 50, 20, 10, 0.10, AWS_NB, AWS_NL), tunables=tun)
    p.init()
    return p


@pytest.mark.parametrize("n", [16384])
def test_gsf_invariants_and_determinism(n):
    a, b = make(n), make(n)
    prev = np.ones(n, np.int64)
    for i in range(12):
        a.network().run_ms(100)
        card = popcount_rows(a.verified()).astype(np.int64)
        assert (card == a.scalars()["card"]).all()          # cached cardinality == popcount of the row
        assert (card >= prev).all()                           # verified sets never shrink
        prev = card
        c = a.network().counters()
        assert c[1].sum() >= c[0].sum()                       # every received message was sent
        lv = a.level_scalars()
        assert (lv["card"].sum(axis=1)[a.network().attrs()["down"] == 0] == card[a.network().attrs()["down"] == 0]).all()
        # own signature always present
        ids = np.arange(n)
        assert ((a.verified()[ids, ids // 64] >> (ids % 64).astype(np.uint64)) & np.uint64(1)).all()
    # same seed + same runMs slicing -> identical state on a second engine (the reference's testCopy property;
    # a different slicing may legitimately differ: SURVEY.md A.1 rule 2)
    for i in range(12):
        b.network().run_ms(100)
    assert (a.verified() == b.verified()).all()
    assert (a.network().counters() == b.network().counters()).all()
    assert a.network().rng_state() == b.network().rng_state()
    down = a.network().attrs()["down"] == 1
    assert (prev[down] == 1).all()


@pytest.mark.gpu
def test_run_multiple_times_concurrent_equals_sequential_and_oracle():
    """RunMultipleTimes (C/RunMultipleTimes.java:41-85): seeds in flight concurrently give the sequential result, and the
    averaged stats equal the oracle's over the same seeds."""
    import numpy as np

    from tests.oracle_lib import OracleGSF
    from wittgenstein_b200 import (DoneAtStatGetter, GSFSignature, GSFSignatureParameters, MsgReceivedStatGetter, RunMultipleTimes)
    from wittgenstein_b200.run_multiple import avg, get_stats_on

    args = (256, 204, 4, 50, 20, 10, 25, "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency")
    p = GSFSignature(GSFSignatureParameters(*args))
    cont = lambda c: c.continue_if()  # noqa: E731
    r_seq = RunMultipleTimes(p, 4, 0, [DoneAtStatGetter(), MsgReceivedStatGetter()])
    seq = r_seq.run(cont, concurrency=1)
    r_con = RunMultipleTimes(p, 4, 0, [DoneAtStatGetter(), MsgReceivedStatGetter()])
    con = r_con.run(cont, concurrency=4)
    assert seq == con and r_seq.end_times == r_con.end_times
    done, recv = [], []
    for seed in range(4):
        o = OracleGSF(*args, seed=seed)
        o.init()
        while True:
            did = o.run_ms(10)
            live = o.attrs()["down"] == 0
            more = bool(((o.scalars()["card"] < args[1]) & live).any())
            if not ((not did) or more):
                break
        assert o.time == r_seq.end_times[seed]
        c = o.counters()
        done.append(get_stats_on(c[4][live]))
        recv.append(get_stats_on(c[0][live]))
    assert avg(done) == seq[0] and avg(recv) == seq[1]


@pytest.mark.gpu
def test_progress_per_time_rounds():
    """ProgressPerTime (C/ProgressPerTime.java:52-129): per-round series sampled every 10 ms and the averaged counters, concurrent
    rounds equal to sequential ones and to the oracle's runs of the same seeds."""
    from tests.oracle_lib import OracleGSF
    from wittgenstein_b200 import DoneAtStatGetter, GSFSignature, GSFSignatureParameters, ProgressPerTime
    from wittgenstein_b200.run_multiple import get_stats_on

    args = (128, 100, 3, 20, 10, 10, 8, "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter")
    tmpl = GSFSignature(GSFSignatureParameters(*args))
    cont = lambda c: c.continue_if()  # noqa: E731
    a = ProgressPerTime(tmpl, DoneAtStatGetter(), 3)
    sa = a.run(cont, concurrency=1)
    b = ProgressPerTime(tmpl, DoneAtStatGetter(), 3)
    sb = b.run(cont, concurrency=3)
    assert [[(t, s.min, s.max, s.avg) for t, s in r] for r in sa] == [[(t, s.min, s.max, s.avg) for t, s in r] for r in sb]
    assert a.average == b.average
    sums = {"msg_rcvd": 0, "done_at": 0}
    for seed in range(3):
        o = OracleGSF(*args, seed=seed)
        o.init()
        lines = []
        while True:
            o.run_ms(10)
            live = o.attrs()["down"] == 0
            st = get_stats_on(o.counters()[4][live])
            lines.append((o.time, st.min, st.max, st.avg))
            if not bool(((o.scalars()["card"] < args[1]) & live).any()):
                break
        assert lines == [(t, s.min, s.max, s.avg) for t, s in sa[seed]]
        sums["msg_rcvd"] += get_stats_on(o.counters()[0][live]).avg
        sums["done_at"] += get_stats_on(o.counters()[4][live]).avg
    assert a.average["msg_rcvd"] == sums["msg_rcvd"] // 3 and a.average["done_at"] == sums["done_at"] // 3


def test_gsf_65536_prefix_vs_oracle():
    """The metric configuration itself (BASELINE.json: GSFSignature, 65 536 nodes, the largest power of two whose engine
    state fits an 80 GB H100) against the oracle: bit-exact state after [0, 300] ms with runMs(10) slicing — pooled payload
    levels up to 17 (4 KiB blocks), 3N-entry buckets.  Needs ~40 GB of host memory for the oracle's peer tables; skipped on
    smaller hosts."""
    import os

    import psutil

    from tests import parity
    from tests.oracle_lib import OracleGSF

    n = 65536
    if psutil.virtual_memory().available < 40 * 2**30:
        pytest.skip("host memory too small for the oracle at 65536 nodes")
    o = OracleGSF(n, int(0.85 * n), 4, 50, 20, 10, int(0.10 * n), AWS_NB, AWS_NL)
    o.init_fast(min(64, os.cpu_count() or 1))
    p = make(n)
    for _ in range(30):
        p.network().run_ms(10)
        o.run_ms(10)
    bad = parity.compare_gsf(p, o, "t=300", full=True)
    assert not bad, bad


def test_handel_32768_config3_against_offline_oracle_digests():
    """BASELINE config #3 (Handel 32 768 nodes, 8 192 suicide-Byzantine, AWS latencies): the device run against digests of the
    oracle's state produced offline (tests/golden/make_handel32768.py; the oracle needs minutes per simulated second here),
    every 100 ms up to the last committed checkpoint — past the start of the Byzantine phase."""
    import json
    import os

    from tests.parity import handel_digests
    from wittgenstein_b200 import Handel, HandelParameters

    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "handel32768_config3.json")
    if not os.path.exists(path):
        pytest.skip("no offline digests committed")
    fx = json.load(open(path))
    prm = fx["params"]
    p = Handel(HandelParameters(*prm[:8], prm[8], prm[9], prm[10], prm[11], prm[12]))
    p.init()
    last = max(int(t) for t in fx["checkpoints"])
    assert last >= 300
    while p.network().time < last:
        p.network().run_ms(100)
        want = fx["checkpoints"].get(str(p.network().time))
        if want is not None:
            got = handel_digests(p, False)
            assert got == want, (p.network().time, {k: (got[k], want[k]) for k in got if got[k] != want[k]})


def test_casper_16390_config4_prefix_vs_oracle():
    """BASELINE config #4 (CasperIMD 64-slot cycles, 5 producers, 256 attesters per slot = 16 390 nodes) against the oracle
    through the first 40 000 ms (5 slots: 1 280 votes x 16 390 destinations), every 4 000 ms"""
    from tests.oracle_lib import OracleCasper
    from tests.parity import compare_casper
    from wittgenstein_b200 import CasperIMD, CasperParemeters

    nb, nl = "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"
    p = CasperIMD(CasperParemeters(64, False, 5, 256, 1000, 1, nb, nl))
    o = OracleCasper(64, False, 5, 256, 1000, 1, nb, nl)
    p.init(0); o.init(0)
    while o.time < 40000:
        assert p.network().run_ms(4000) == o.run_ms(4000)
        bad = compare_casper(p, o, f"t={o.time}")
        assert not bad, bad
