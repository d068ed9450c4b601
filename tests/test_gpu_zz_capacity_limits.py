"""Every engine arena at its exact capacity on the device, through the C ABI (tests/capacity_limits.py): the minimum of each
(configuration, arena) runs bit-exact against the oracle, the next smaller capacity fails with that arena's error, and the
minimum equals the host build's.  Every arena here fills deterministically, so a device minimum that differs from the host
build's is a device-side check or stat that is off.  The bucket check of most protocols (the multisplit's scan) and the
32-lane warp emitters exist only in device code."""
import pytest

from tests import capacity_limits as cl
from tests import emu_cond_ahead_lib, emu_lib
from wittgenstein_b200 import WtgError

pytestmark = pytest.mark.gpu


def host_api(cfg):
    return emu_cond_ahead_lib.api() if cfg.host_api == "cond_ahead" else emu_lib.api()


@pytest.mark.parametrize("name,key", cl.CASES)
def test_capacity_boundary(name, key):
    cfg = cl.BY_NAME[name]
    cstar = cl.minimum(cfg, None, key)
    cl.check_boundary(cfg, None, key, cstar)
    st = cl.default_stats(cfg, None)
    rule = cl.stat_minimum(cfg, key, st)
    assert rule is None or cstar == rule, f"{name}: {key} minimum {cstar}, the stats give {rule}"
    assert cstar == cl.minimum(cfg, host_api(cfg), key), f"{name}: {key} minimum differs between device and host build"
    host = cl.default_stats(cfg, host_api(cfg))
    for k in ("max_bucket", "max_queue", "rec_top", "rec_dest_top"):
        assert st[k] == host[k], f"{name}: {k} {st[k]} on the device, {host[k]} on the host build"


@pytest.mark.parametrize("key", ["bcap", "qcap", "pool_slots_per_node", "desc_cap"])
def test_gsf_minima_equal_for_both_checksigs_orders(key):
    c0, c1 = cl.BY_NAME["gsf256_aws_cond0"], cl.BY_NAME["gsf256_aws_cond1"]
    assert cl.minimum(c0, None, key) == cl.minimum(c1, None, key)


def test_p2pflood_degree_at_the_emit_warp_limit():
    cfg = cl.BY_NAME["p2pflood1024_peers150"]
    p, _ = cfg.make(None, {}, False)
    assert cl.p2p_max_degree(p) == 254
    with pytest.raises(WtgError, match="degree 261"):
        cl._p2pflood(1024, 150, 2)(None, {}, False)
