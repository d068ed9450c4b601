"""Every engine arena at its exact capacity — TEST INFRASTRUCTURE shared by the host-build and device tests.

A configuration is an ordinary run through the public tunables: a protocol, a fixed runMs schedule and the arenas that bind in
it.  `minimum(cfg, api, key)` finds the smallest value of one capacity tunable with which the run completes; `check_boundary` then
runs that value against the oracle (bit-exact after every window) and the next smaller value the engine actually uses (the run
must fail with that arena's error, and stay failed).  Where a high-water stat gives the minimum exactly, `stat_minimum` states
the arena's rule and the search must land on it."""
import re
from dataclasses import dataclass, field
from typing import Callable, Optional

from tests.oracle_lib import OracleCappos, OracleCasper, OracleGSF, OracleHandel, OraclePingPong
from tests.parity import compare_casper, compare_gsf

NB, NL = "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"
AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"

# the engine rounds these up (wtg_engine.hpp): qcap to a warp, desc_cap to whole stripes (ARENA_STRIPES), CasperIMD's block
# table to 64-bit words
STEP = {"qcap": 32, "desc_cap": 64, "casper_blocks": 64}

# the error each arena raises when it is too small (throwDeviceError, and the init-time upload checks for the buckets)
ERROR = {
    "bcap": r"time-bucket capacity exceeded|bucket capacity too small",
    "qcap": r"toVerify queue capacity exceeded",
    "pool_slots_per_node": r"payload pool exhausted",
    "desc_cap": r"descriptor arena exceeded",
    "rec_cap": r"multi-destination record arena exceeded",
    "far_cap": r"far-future calendar exceeded",
    "casper_votes": r"situation not supported by the device path \(detail 3\)",  # attestation table full
    "casper_blocks": r"situation not supported by the device path \(detail 2\)",  # block table full
}


def effective(key, v):
    """the capacity the engine allocates for tunable value v"""
    s = STEP.get(key, 1)
    return (v + s - 1) // s * s


@dataclass
class Config:
    name: str
    make: Callable            # (api, tunables, oracle: bool) -> (protocol, oracle or None), both initialised
    windows: list             # runMs schedule
    keys: list                # the arenas that bind in this run
    compare: Callable         # (p, o, tag, full) -> list of differences
    host_api: str = "emu"     # "emu" or "cond_ahead": which host build runs it
    tunables: dict = field(default_factory=dict)  # fixed tunables of the configuration (cond_ahead, ...)
    after_init: Optional[Callable] = None  # (p, o) -> None: host sends issued after init, on both sides
    rec_dest: Optional[Callable] = None    # rec_cap -> destination-arena capacity, for the rec_cap rule
    queue_reserve: bool = False  # GSF: the onNewSig that reached max_queue stored one entry (see stat_minimum)
    quiet: bool = False       # the schedule ends with msgs.size() == 0 (far-future calendars: every bucket has been processed)


def _gsf(n, thr, pairing, timeout, period, acc, dead, nb, nl, seed=None):
    from wittgenstein_b200 import GSFSignature, GSFSignatureParameters

    args = (n, thr, pairing, timeout, period, acc, dead, nb, nl)

    def make(api, tun, oracle):
        p = GSFSignature(GSFSignatureParameters(*args), _api=api)
        for k, v in tun.items():
            p.network().set_tunable(k, v)
        if seed is not None:
            p.network().set_seed(seed)
        o = OracleGSF(*args, seed=seed) if oracle else None
        p.init()
        if o:
            o.init()
        return p, o
    return make


def _handel_compare(p, o, tag, full=True):
    bad = []
    if p.network().rng_state() != o.rng_state():
        bad.append(f"{tag}: rd state")
    if p.network().msgs_size() != o.msgs_live():
        bad.append(f"{tag}: msgs.size()")
    if not (p.network().counters() == o.counters()).all():
        bad.append(f"{tag}: counters")
    a, b = p.scalars(), o.scalars()
    bad += [f"{tag}: {k}" for k in a if not (a[k] == b[k]).all()]
    if full:
        bad += [f"{tag}: rows {w}" for w in range(6) if not (p.rows(w) == o.rows(w)).all()]
        l1, l2 = p.level_scalars(), o.level_scalars()
        bad += [f"{tag}: level {k}" for k in l1 if not (l1[k] == l2[k]).all()]
    return bad


def _handel(n, thr, down, nb, nl, byz, hidden, seed=None):
    from wittgenstein_b200 import Handel, HandelParameters

    args = (n, thr, 4, 50, 10, 20, 10, down, nb, nl, 0, byz)

    def make(api, tun, oracle):
        p = Handel(HandelParameters(*args, hidden), _api=api)
        for k, v in tun.items():
            p.network().set_tunable(k, v)
        if seed is not None:
            p.network().set_seed(seed)
        o = OracleHandel(*args, seed=seed, hidden_byzantine=hidden) if oracle else None
        p.init()
        if o:
            o.init()
        return p, o
    return make


def _scalars_compare(p, o, tag, full=True):
    bad = []
    net = p.network()
    if net.rng_state() != o.rng_state():
        bad.append(f"{tag}: rd state")
    if net.msgs_size() != (o.msgs_live() if hasattr(o, "msgs_live") else o.msgs_size()):
        bad.append(f"{tag}: msgs.size()")
    if not (net.counters() == o.counters()).all():
        bad.append(f"{tag}: counters")
    a, b = p.scalars(), o.scalars()
    bad += [f"{tag}: {k}" for k in a if not (a[k] == b[k]).all()]
    return bad


def _cappos(n, k):
    from wittgenstein_b200 import SanFerminCappos, SanFerminCapposParameters

    args = (n, n // 2, 2, 48, 150, k, None, None)

    def make(api, tun, oracle):
        p = SanFerminCappos(SanFerminCapposParameters(*args), _api=api, tunables=tun)
        o = OracleCappos(*args) if oracle else None
        p.init()
        if o:
            o.init()
        return p, o
    return make


def _pingpong(n):
    from wittgenstein_b200 import PingPong, PingPongParameters

    def make(api, tun, oracle):
        p = PingPong(PingPongParameters(n, None, None), _api=api)
        for k, v in tun.items():
            p.network().set_tunable(k, v)
        o = OraclePingPong(n, None, None) if oracle else None
        p.init()
        if o:
            o.init()
        return p, o
    return make


def _pingpong_compare(p, o, tag, full=True):
    bad = []
    net = p.network()
    if net.rng_state() != o.rng_state():
        bad.append(f"{tag}: rd state")
    if net.msgs_size() != o.msgs_size():
        bad.append(f"{tag}: msgs.size()")
    if not (net.counters() == o.counters()).all():
        bad.append(f"{tag}: counters")
    if not (p.pongs() == o.pongs()).all():
        bad.append(f"{tag}: pongs")
    return bad


def _pingpong_sends(p, o):
    """caller sends either side of MAX_ACC (16): 17 destinations go through emitBigMulti, 16 through the warp emitter; some
    spaced by delaysBetweenMessage"""
    for side in (p.network(), o):
        if side is None:
            continue
        t = side.time
        for k in range(12):
            dests = [(37 * k + 11 * j + 5) % 300 for j in range(16 + k % 2)]
            side.send(1, k, dests)
            side.send(1, 100 + k, dests, send_time=t + 3 + k, delay_between=k % 4)


def _casper(cyc, apr):
    from wittgenstein_b200 import CasperIMD, CasperParemeters

    args = (cyc, False, 3, apr, 1000, 1, None, None)

    def make(api, tun, oracle):
        p = CasperIMD(CasperParemeters(*args), _api=api)
        for k, v in tun.items():
            p.network().set_tunable(k, v)
        o = OracleCasper(*args) if oracle else None
        p.init(9000)
        if o:
            o.init(9000)
        return p, o
    return make


def _p2pflood(n, peers, seed):
    from tests.p2p_oracle_lib import OracleP2PFlood
    from wittgenstein_b200 import P2PFlood, P2PFloodParameters

    args = (n, 0, 1, 1, 1, peers, 1, NB, NL)

    def make(api, tun, oracle):
        p = P2PFlood(P2PFloodParameters(*args), _api=api, tunables=tun)
        p.network().set_seed(seed)
        o = OracleP2PFlood(*args, seed=seed) if oracle else None
        p.init()
        if o:
            o.init()
        return p, o
    return make


def _p2p_compare(p, o, tag, full=True):
    from tests.p2p_parity import compare

    return compare(p, o, tag, bitmaps=False)


def _slush(n, k):
    from tests.avalanche_oracle_lib import OracleSlush
    from wittgenstein_b200 import Slush, SlushParameters

    args = (n, 4, k, 4.0 / 7.0, NB, NL)

    def make(api, tun, oracle):
        p = Slush(SlushParameters(*args), _api=api, tunables=tun)
        o = OracleSlush(*args) if oracle else None
        p.init()
        if o:
            o.init()
        return p, o
    return make


def _avalanche_compare(p, o, tag, full=True):
    from tests.avalanche_parity import compare

    return compare(p, o, tag)


CONFIGS = [
    # seed 7: the queue's high-water mark (96) is a whole number of warps and was reached by an onNewSig that stored one
    # entry, so the reservation of a second entry is what makes qcap 128
    *[Config(f"gsf256_aws_cond{c}", _gsf(256, 204, 4, 50, 20, 10, 25, AWS_NB, AWS_NL, seed=7), [10] * 150,
             ["bcap", "qcap", "pool_slots_per_node", "desc_cap"], compare_gsf, host_api="cond_ahead", tunables={"cond_ahead": c},
             queue_reserve=True)
      for c in (0, 1)],
    Config("gsf256_ethscan", _gsf(256, 204, 3, 20, 10, 10, 25, NB, "EthScanNetworkLatency"), [100] * 30,
           ["far_cap", "pool_slots_per_node"], compare_gsf, host_api="cond_ahead", tunables={"cond_ahead": 1}),
    Config("handel1024_suicide_aws", _handel(1024, 760, 256, "AWS_SPEED=GAUSSIAN_TOR=0.00", AWS_NL, True, False), [10] * 100,
           ["qcap", "bcap", "pool_slots_per_node"], _handel_compare),
    Config("handel1024_hidden_aws", _handel(1024, 700, 256, "AWS_SPEED=GAUSSIAN_TOR=0.00", AWS_NL, False, True, seed=3), [10] * 100,
           ["bcap", "pool_slots_per_node"], _handel_compare),
    Config("cappos512_k50", _cappos(512, 50), [10] * 100, ["rec_cap", "desc_cap"], _scalars_compare,
           rec_dest=lambda rc: rc * 51 // 2 + 512 + 1024),  # capposInit: rec_cap x (candidateCount + 1) / 2 + N + 1024
    Config("pingpong300_sends", _pingpong(300), [7] * 60, ["rec_cap", "bcap"], _pingpong_compare, after_init=_pingpong_sends,
           rec_dest=lambda rc: rc * 4 + 300 + 1024),  # allocCommon's default: rec_cap x 4 + N + 1024
    Config("p2pflood1024_peers150", _p2pflood(1024, 150, 1), [1, 3, 7, 13, 50] * 40, ["bcap"], _p2p_compare, quiet=True),
    Config("casper3x20", _casper(3, 20), [4000] * 150, ["rec_cap", "casper_votes", "casper_blocks"],
           lambda p, o, tag, full: compare_casper(p, o, tag, atts=full), tunables={"casper_votes": 30}),
    Config("slush1024", _slush(1024, 7), [1, 3, 7, 13, 50] * 4, ["bcap"], _avalanche_compare),
]
BY_NAME = {c.name: c for c in CONFIGS}
CASES = [(c.name, k) for c in CONFIGS for k in c.keys]


@dataclass
class Outcome:
    error: Optional[str]          # None: the whole schedule ran
    stats: dict                   # stats() after a completed run
    diffs: list                   # mismatches with the oracle (oracle runs only)
    at_init: bool = False         # the error came from init(): there is no network to run again
    again: Optional[str] = None   # the error of one more runMs after a failed one
    p: object = None              # the protocol object of a completed run


def run(cfg, api, key=None, value=None, oracle=False):
    """a fresh engine with `key` = `value`, through the whole schedule (against the oracle after every window if `oracle`)"""
    from wittgenstein_b200 import WtgError

    tun = dict(cfg.tunables)
    if key is not None:
        tun[key] = value
    try:
        p, o = cfg.make(api, tun, oracle)
    except WtgError as e:
        return Outcome(str(e), {}, [], at_init=True)
    diffs = []
    try:
        if cfg.after_init:
            cfg.after_init(p, o)
        for i, ms in enumerate(cfg.windows):
            r = p.network().run_ms(ms)
            if o is not None:
                if r != o.run_ms(ms):
                    diffs.append(f"t={o.time}: runMs result")
                diffs += cfg.compare(p, o, f"t={o.time}", i + 1 == len(cfg.windows))
                if diffs:
                    break
    except WtgError as e:
        try:
            p.network().run_ms(1)
            again = None
        except WtgError as e2:
            again = str(e2)
        return Outcome(str(e), {}, diffs, again=again)
    if cfg.quiet:
        assert p.network().msgs_size() == 0, f"{cfg.name}: the schedule ends with envelopes in flight"
    return Outcome(None, p.network().stats(), diffs, p=p)


_minima = {}


def minimum(cfg, api, key):
    """the smallest value of `key` with which the schedule completes: galloping, then bisection over the values the engine
    distinguishes (multiples of STEP); memoised per library"""
    memo = (id(api), cfg.name, key)
    if memo in _minima:
        return _minima[memo]
    s = STEP.get(key, 1)
    lo, hi = 0, 1  # in units of s: lo fails (0 stands for nothing), hi is the probe
    while run(cfg, api, key, hi * s).error is not None:
        lo, hi = hi, hi * 2
        assert hi * s < 1 << 26, f"{cfg.name}: {key} does not complete even at {hi * s}"
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if run(cfg, api, key, mid * s).error is None:
            hi = mid
        else:
            lo = mid
    _minima[memo] = hi * s
    return hi * s


def stat_minimum(cfg, key, st):
    """the minimum that the high-water stats of a completed run give (default_stats), by the arena's rule; None where no
    stat covers the arena"""
    if key == "bcap":
        # max_bucket is the fill of a bucket when it is processed; the buckets still ahead when the run ends count too
        return max(st["max_bucket"], st["pending_bucket"])
    if key == "qcap":
        q = st["max_queue"]
        if cfg.name.startswith("handel"):
            return effective(key, q)  # len + 1 > qcap: the queue holds every entry it was asked for
        # GSF's onNewSig reserves two entries (len + 2 > qcap) and stores one or two: the call that reached max_queue
        # needed max_queue + 1 if it stored one, max_queue if it stored two
        return effective(key, q + 1 if cfg.queue_reserve else q)
    if key == "rec_cap" and cfg.rec_dest is not None:
        # bump arenas: ri >= recCap and off + cnt > recDestCap, with recDestCap a function of rec_cap
        need = st["rec_top"]
        while cfg.rec_dest(need) < st["rec_dest_top"]:
            need += 1
        return need
    return None


def check_boundary(cfg, api, key, cstar):
    """c* runs bit-exact against the oracle; the next smaller value the engine uses fails with this arena's error, no other,
    and the network stays failed"""
    at = run(cfg, api, key, cstar, oracle=True)
    assert at.error is None, f"{cfg.name}: {key}={cstar} failed: {at.error}"
    assert not at.diffs, f"{cfg.name}: {key}={cstar} differs from the oracle: {at.diffs[:5]}"
    if key in ("bcap", "qcap"):
        assert at.stats[key] == cstar, f"{cfg.name}: the engine uses {key}={at.stats[key]}, expected {cstar}"
    below = cstar - STEP.get(key, 1)
    assert below > 0, f"{cfg.name}: {key} never binds (minimum {cstar})"
    under = run(cfg, api, key, below)
    assert under.error is not None, f"{cfg.name}: {key}={below} completed"
    assert re.search(ERROR[key], under.error), f"{cfg.name}: {key}={below} raised another error: {under.error}"
    others = [o for o, pat in ERROR.items() if o != key and re.search(pat, under.error)]
    assert not others, f"{cfg.name}: {key}={below}: {under.error} names {others}"
    assert not re.search(r"internal|CUDA|cuda", under.error), under.error
    if not under.at_init:
        assert under.again is not None and re.search(ERROR[key], under.again), \
            f"{cfg.name}: {key}={below}: the next runMs gave {under.again!r}"
    return at


def default_stats(cfg, api):
    """stats() of a run with the default capacities, with pending_bucket: the fullest bucket not processed yet (runs that
    end quiet have none; the others keep no far-future calendar, so msgs.size() at an arrival time is its bucket's fill)"""
    out = run(cfg, api)
    assert out.error is None, f"{cfg.name} fails with the default capacities: {out.error}"
    net = out.p.network()
    st = dict(out.stats)
    st["pending_bucket"] = 0
    if "bcap" in cfg.keys and not cfg.quiet:
        st["pending_bucket"] = max(net.msgs_size_at(net.time + k) for k in range(1, st["ring"]))
    return st


def p2p_max_degree(p):
    return max(len(p.peers(i)) for i in range(p.params.node_count))
