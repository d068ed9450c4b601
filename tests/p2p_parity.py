"""P2PFlood parity helpers shared by the host-build and device tests — TEST INFRASTRUCTURE ONLY."""
import numpy as np

from tests.p2p_oracle_lib import OracleP2PFlood

NB, NL = "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"
NO_NL = "NetworkNoLatency"
AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"


def make(api, n, dead=0, resend=1, msgs=1, peers=10, between=1, nb=NB, nl=NL, seed=None, tunables=None):
    """(device-side P2PFlood, oracle) with the same parameters, both initialised"""
    from wittgenstein_b200 import P2PFlood, P2PFloodParameters

    p = P2PFlood(P2PFloodParameters(n, dead, resend, msgs, 1, peers, between, nb, nl), _api=api, tunables=tunables)
    o = OracleP2PFlood(n, dead, resend, msgs, 1, peers, between, nb, nl, seed=seed)
    if seed is not None:
        p.network().set_seed(seed)
    p.init()
    o.init()
    return p, o


def compare_graph(p, o):
    bad = [f"peers of {i}" for i in range(p.params.node_count) if not np.array_equal(p.peers(i), o.peers(i))]
    if p.avg_peers() != o.avg_peers():
        bad.append(f"avgPeers {p.avg_peers()} != {o.avg_peers()}")
    return bad


def compare(p, o, where="", bitmaps=None):
    """the differences between the device-side state and the oracle's, as a list of names (empty: bit-exact)"""
    bad = []
    net = p.network()
    if net.time != o.time:
        bad.append(f"time {net.time} != {o.time}")
    if net.rng_state() != o.rng_state():
        bad.append("rng state")
    if net.msgs_size() != o.msgs_size():
        bad.append(f"msgs.size() {net.msgs_size()} != {o.msgs_size()}")
    if not (net.counters() == o.counters()).all():
        bad.append("node counters")
    cnt, _, bits = o.received()
    if not np.array_equal(p.received_count(), cnt):
        bad.append("received counts")
    if bitmaps is None:
        bitmaps = p.params.msg_count > 1
    if bitmaps:
        for i in range(p.params.node_count):
            mine = p.received(i)
            theirs = np.unpackbits(bits[i].view(np.uint8), bitorder="little")[:p.params.msg_count].astype(bool)
            if not np.array_equal(mine, theirs):
                bad.append(f"received bitmap of {i}")
                break
    return [f"{where}: {x}" for x in bad]


def run_compare(p, o, slices, limit_ms=60000, until_quiet=True, bitmaps=None):
    """runMs over `slices` (cycled) on both sides, comparing after every window, until both are quiet (msgs.size() == 0)
    or `limit_ms` have run; returns the differences (empty: bit-exact all along)"""
    i = 0
    while o.time < limit_ms:
        ms = slices[i % len(slices)]
        i += 1
        r1, r2 = p.network().run_ms(ms), o.run_ms(ms)
        bad = compare(p, o, f"t={o.time}", bitmaps)
        if r1 != r2:
            bad.append(f"t={o.time}: runMs result {r1} != {r2}")
        if bad:
            return bad
        if until_quiet and o.msgs_size() == 0:
            break
    return []
