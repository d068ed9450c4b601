"""ctypes loader for the C-ABI shared library (include/wtg.h).

The library is hand-written CUDA for sm_90a (H100; wittgenstein_b200/csrc).  There is no CPU
fallback: if the shared library is missing or no CUDA device is visible, creating a network
raises.  Build it with `python -c "import __graft_entry__ as g; g.build()"`.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("WTG_LIB") or os.path.join(_HERE, "libwtg_b200.so")  # WTG_LIB: a differently built copy of the same library (kernel experiments)


class WtgError(RuntimeError):
    """Raised where the reference throws IllegalArgumentException / IllegalStateException."""


class Api:
    """Typed view over the C ABI.  `prefix` exists so the test-suite's debugging build can expose the
    same entry points under another name; the product always uses `wtg_`."""

    _SIGS = {
        "last_error": (C.c_char_p, []),
        "create": (C.c_void_p, []),
        "create_on": (C.c_void_p, [C.c_int]),
        "destroy": (None, [C.c_void_p]),
        "shard_create": (C.c_void_p, [C.c_int, C.c_int, C.c_int]),
        "shard_export": (C.c_int, [C.c_void_p, C.POINTER(C.c_ubyte)]),
        "shard_link": (C.c_int, [C.c_void_p, C.POINTER(C.c_ubyte)]),
        "shard_range": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
        "device": (C.c_int, [C.c_void_p]),
        "set_seed": (C.c_int, [C.c_void_p, C.c_longlong]),
        "set_network_latency": (C.c_int, [C.c_void_p, C.c_char_p]),
        "set_network_latency_measured": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]),
        "set_node_builder": (C.c_int, [C.c_void_p, C.c_char_p]),
        "set_msg_discard_time": (C.c_int, [C.c_void_p, C.c_int]),
        "set_tunable": (C.c_int, [C.c_void_p, C.c_char_p, C.c_longlong]),
        "pingpong_init": (C.c_int, [C.c_void_p, C.c_int]),
        "gsf_init": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "sanfermin_construct": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "sanfermin_init": (C.c_int, [C.c_void_p]),
        "sanfermin_node_scalars": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 7 + [C.POINTER(C.c_longlong)]),
        "casper_construct": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "casper_init": (C.c_int, [C.c_void_p, C.c_int]),
        "casper_init_byz": (C.c_int, [C.c_void_p, C.c_int, C.c_int]),
        "casper_block_count": (C.c_int, [C.c_void_p]),
        "casper_blocks": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 5),
        "casper_block_attestations": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_int]),
        "casper_node_state": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 5 + [C.POINTER(C.c_ulonglong)]),
        "casper_heads": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "casper_byz": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "cappos_init": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "cappos_node_scalars": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 6 + [C.POINTER(C.c_longlong)]),
        "java_shuffle": (C.c_int, [C.c_ulonglong, C.c_int, C.POINTER(C.c_int)]),
        "slush_init": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double]),
        "snowflake_init": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int]),
        "avalanche_node_scalars": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 6),
        "serial_passes": (C.c_longlong, [C.c_void_p]),
        "p2pflood_init": (C.c_int, [C.c_void_p] + [C.c_int] * 6),
        "p2p_peer_count": (C.c_int, [C.c_void_p, C.c_int]),
        "p2p_peers": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int]),
        "p2p_avg_peers": (C.c_int, [C.c_void_p]),
        "p2pflood_received": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_ulonglong)]),
        "handel_init": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "handel_node_scalars": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "handel_rows": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_ulonglong)]),
        "handel_level_scalars": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 3),
        "handel_peers": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int]),
        "handel_ranks": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int)]),
        "handel_levels": (C.c_int, [C.c_void_p]),
        "send": (C.c_int, [C.c_void_p, C.c_int, C.c_ulonglong, C.c_int, C.POINTER(C.c_int), C.c_int]),
        "send_all": (C.c_int, [C.c_void_p, C.c_int, C.c_ulonglong, C.c_int]),
        "send_at": (C.c_int, [C.c_void_p, C.c_int, C.c_ulonglong, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int]),
        "run_ms": (C.c_int, [C.c_void_p, C.c_int]),
        "time": (C.c_int, [C.c_void_p]),
        "node_count": (C.c_int, [C.c_void_p]),
        "msgs_size": (C.c_int, [C.c_void_p]),
        "msgs_size_at": (C.c_int, [C.c_void_p, C.c_int]),
        "peek_messages": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 6 + [C.c_int]),
        "stop_node": (C.c_int, [C.c_void_p, C.c_int]),
        "start_node": (C.c_int, [C.c_void_p, C.c_int]),
        "partition": (C.c_int, [C.c_void_p, C.c_float]),
        "end_partition": (C.c_int, [C.c_void_p]),
        "rng_state": (C.c_ulonglong, [C.c_void_p]),
        "node_counters": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong)]),
        "node_attrs": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                 C.POINTER(C.c_double), C.POINTER(C.c_ubyte)]),
        "pingpong_pongs": (C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
        "gsf_levels": (C.c_int, [C.c_void_p]),
        "gsf_verified": (C.c_int, [C.c_void_p, C.POINTER(C.c_ulonglong)]),
        "gsf_rows": (C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_ulonglong)]),
        "gsf_node_scalars": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 5),
        "gsf_level_scalars": (C.c_int, [C.c_void_p] + [C.POINTER(C.c_int)] * 3),
        "gsf_peers": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_int), C.c_int]),
        "stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_longlong)]),
        "timer_start": (C.c_int, [C.c_void_p]),
        "timer_stop_ms": (C.c_double, [C.c_void_p]),
        "profile_enable": (C.c_int, [C.c_void_p, C.c_int]),
        "profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_longlong), C.POINTER(C.c_char_p), C.c_int]),
    }

    def __init__(self, path=LIB_PATH, prefix="wtg_"):
        if not os.path.exists(path):
            raise WtgError(
                f"{path} not found: the CUDA extension is not built (run __graft_entry__.build()); "
                "wittgenstein_b200 has no CPU fallback")
        self.lib = C.CDLL(path)
        self.prefix = prefix
        for name, (res, args) in self._SIGS.items():
            fn = getattr(self.lib, prefix + name)
            fn.restype = res
            fn.argtypes = args
            setattr(self, name, fn)

    def symbols(self):
        return [self.prefix + n for n in self._SIGS]

    def check(self, rc):
        if rc < 0:
            raise WtgError(self.last_error().decode())
        return rc


_api = None


def api():
    global _api
    if _api is None:
        _api = Api()
    return _api
