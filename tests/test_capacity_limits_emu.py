"""Every engine arena at its exact capacity, on the host build of the device logic (tests/emu): for each configuration and each
arena that binds in it, the smallest capacity that completes the run compares bit-exact with the oracle after every runMs, the
next smaller capacity the engine uses fails with that arena's error and stays failed, and where a high-water stat covers the
arena the minimum is the one its rule gives (tests/capacity_limits.py)."""
import pytest

from tests import capacity_limits as cl
from tests import emu_cond_ahead_lib, emu_lib
from wittgenstein_b200 import WtgError


def host_api(cfg):
    return emu_cond_ahead_lib.api() if cfg.host_api == "cond_ahead" else emu_lib.api()


@pytest.mark.parametrize("name,key", cl.CASES)
def test_capacity_boundary(name, key):
    cfg = cl.BY_NAME[name]
    api = host_api(cfg)
    cstar = cl.minimum(cfg, api, key)
    cl.check_boundary(cfg, api, key, cstar)
    rule = cl.stat_minimum(cfg, key, cl.default_stats(cfg, api))
    assert rule is None or cstar == rule, f"{name}: {key} minimum {cstar}, the stats give {rule}"


@pytest.mark.parametrize("key", ["bcap", "qcap", "pool_slots_per_node", "desc_cap"])
def test_gsf_minima_equal_for_both_checksigs_orders(key):
    """checkSigs of t + 1 beside the emission of t (cond_ahead = 1) evicts from the pool and samples it where the serial
    order does (DESIGN.md §4): every arena needs exactly what it needs with cond_ahead = 0"""
    c0, c1 = cl.BY_NAME["gsf256_aws_cond0"], cl.BY_NAME["gsf256_aws_cond1"]
    assert cl.minimum(c0, host_api(c0), key) == cl.minimum(c1, host_api(c1), key)


def test_p2pflood_degree_at_the_emit_warp_limit():
    """peersCount 150 at 1 024 nodes: seed 1 reaches degree 254, which the emit warp takes; seed 2 reaches 261, which init
    refuses with its degree message"""
    cfg = cl.BY_NAME["p2pflood1024_peers150"]
    p, _ = cfg.make(emu_lib.api(), {}, False)
    assert cl.p2p_max_degree(p) == 254
    with pytest.raises(WtgError, match="degree 261"):
        cl._p2pflood(1024, 150, 2)(emu_lib.api(), {}, False)


def test_p2pflood_record_arenas_never_bind():
    """P2PFlood sizes its record arenas exactly at init (one record per node and message): rec_cap does not reach them"""
    cfg = cl.BY_NAME["p2pflood1024_peers150"]
    out = cl.run(cfg, emu_lib.api(), "rec_cap", 1)
    assert out.error is None, out.error
    assert out.stats["rec_top"] <= 1024
