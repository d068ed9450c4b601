"""Slush / Snowflake parity helpers shared by the host-build and device tests — TEST INFRASTRUCTURE ONLY."""
from tests.avalanche_oracle_lib import OracleSlush, OracleSnowflake

NB, NL = "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"
AWS_NB, AWS_NL = "AWS_SPEED=GAUSSIAN_TOR=0.33", "AwsRegionNetworkLatency"


def make(proto, api, n, k, nb, nl, seed=None, tunables=None, m=4, a=4.0 / 7.0, b=3):
    """(device-side protocol object, oracle) with the same parameters, both initialised"""
    from wittgenstein_b200 import Slush, SlushParameters, Snowflake, SnowflakeParameters

    if proto == "slush":
        p = Slush(SlushParameters(n, m, k, a, nb, nl), _api=api, tunables=tunables)
        o = OracleSlush(n, m, k, a, nb, nl, seed=seed)
    else:
        p = Snowflake(SnowflakeParameters(n, m, k, a, b, nb, nl), _api=api, tunables=tunables)
        o = OracleSnowflake(n, m, k, a, b, nb, nl, seed=seed)
    if seed is not None:
        p.network().set_seed(seed)
    p.init()
    o.init()
    return p, o


def compare(p, o, where=""):
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
    a, b = p.scalars(), o.scalars()
    bad += [k for k in a if not (a[k] == b[k]).all()]
    return [f"{where}: {x}" for x in bad]


def run_compare(p, o, slices, until_quiet=True, limit_ms=60000):
    """runMs over `slices` (cycled) on both sides, comparing after every window, until both are quiet (msgs.size() == 0)
    or `limit_ms` have run; returns the differences (empty: bit-exact all along)"""
    i = 0
    while o.time < limit_ms:
        ms = slices[i % len(slices)]
        i += 1
        r1, r2 = p.network().run_ms(ms), o.run_ms(ms)
        bad = compare(p, o, f"t={o.time}")
        if r1 != r2:
            bad.append(f"t={o.time}: runMs result {r1} != {r2}")
        if bad:
            return bad
        if until_quiet and o.msgs_size() == 0:
            break
    return []
