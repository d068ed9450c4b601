"""ctypes binding of the CPU restatement of P2PFlood (tests/p2p_oracle) — TEST INFRASTRUCTURE ONLY.

The restatement sits on the oracle's core (oracle/core.hpp: Network, Node, Message, java.util.Random) and is compiled on
first use.  Only tests/ and scripts/ may import this module; the product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC_DIR = os.path.join(ROOT, "tests", "p2p_oracle")
ORACLE_DIR = os.path.join(ROOT, "oracle")
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    so = os.path.join(SRC_DIR, "libwtg_p2p_oracle.so")
    srcs = [os.path.join(SRC_DIR, f) for f in ("p2pflood.hpp", "capi.cpp")]
    srcs += [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".hpp", ".inc"))]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wextra", "-ffp-contract=off", "-fno-fast-math",
                               "-o", so, os.path.join(SRC_DIR, "capi.cpp")])
    lib = C.CDLL(so)
    lib.wpf_last_error.restype = C.c_char_p
    lib.wpf_create.restype = C.c_void_p
    lib.wpf_create.argtypes = [C.c_int] * 7 + [C.c_char_p, C.c_char_p]
    for name in ("wpf_destroy", "wpf_init", "wpf_time", "wpf_msgs_size", "wpf_avg_peers"):
        getattr(lib, name).argtypes = [C.c_void_p]
    lib.wpf_set_seed.argtypes = [C.c_void_p, C.c_int64]
    lib.wpf_run_ms.argtypes = [C.c_void_p, C.c_int]
    lib.wpf_run_timed.restype = C.c_double
    lib.wpf_run_timed.argtypes = [C.c_void_p, C.c_int]
    lib.wpf_net_ctl.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.wpf_rng_state.restype = C.c_uint64
    lib.wpf_rng_state.argtypes = [C.c_void_p]
    lib.wpf_deliveries.restype = C.c_int64
    lib.wpf_deliveries.argtypes = [C.c_void_p]
    lib.wpf_peer_count.argtypes = [C.c_void_p, C.c_int]
    lib.wpf_peers.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    lib.wpf_node_counters.argtypes = [C.c_void_p, C.c_void_p]
    lib.wpf_received.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
    lib.wpf_peek_messages.argtypes = [C.c_void_p] * 5 + [C.c_int]
    _lib = lib
    return lib


def _b(s):
    return None if s is None else s.encode()


class OracleP2PFlood:
    """protocols/P2PFlood.java through the CPU restatement."""

    def __init__(self, node_count=100, dead_node_count=10, delay_before_resent=50, msg_count=1, msg_to_receive=1, peers_count=10,
                 delay_between_sends=30, node_builder=None, latency=None, seed=None):
        self.lib = load()
        self.n = node_count
        self.msg_count = msg_count
        self.h = C.c_void_p(self.lib.wpf_create(node_count, dead_node_count, delay_before_resent, msg_count, msg_to_receive, peers_count,
                                                delay_between_sends, _b(node_builder), _b(latency)))
        if not self.h:
            raise ValueError(self.lib.wpf_last_error().decode())
        if seed is not None:
            self.lib.wpf_set_seed(self.h, C.c_int64(seed))

    def __del__(self):
        try:
            self.lib.wpf_destroy(self.h)
        except Exception:  # noqa: BLE001
            pass

    def _check(self, r):
        if r < 0:
            raise RuntimeError(self.lib.wpf_last_error().decode())
        return r

    def init(self):
        self._check(self.lib.wpf_init(self.h))

    def run_ms(self, ms):
        return bool(self._check(self.lib.wpf_run_ms(self.h, ms)))

    def run_timed(self, ms):
        """runMs(ms) and the host time it took, in ms"""
        t = self.lib.wpf_run_timed(self.h, ms)
        if t < 0:
            raise RuntimeError(self.lib.wpf_last_error().decode())
        return t

    @property
    def time(self):
        return self.lib.wpf_time(self.h)

    def msgs_size(self):
        return self.lib.wpf_msgs_size(self.h)

    def deliveries(self):
        return int(self.lib.wpf_deliveries(self.h))

    def rng_state(self):
        return int(self.lib.wpf_rng_state(self.h))

    def counters(self):
        out = np.zeros((5, self.n), np.int64)
        self.lib.wpf_node_counters(self.h, out.ctypes.data)
        return out

    def received(self):
        """(count[N], down[N], bits[N][words]) — bits: which originating messages (init's draw order) each node holds"""
        words = max(1, (self.msg_count + 63) // 64)
        cnt = np.zeros(self.n, np.int32)
        down = np.zeros(self.n, np.uint8)
        bits = np.zeros((self.n, words), np.uint64)
        self.lib.wpf_received(self.h, cnt.ctypes.data, down.ctypes.data, bits.ctypes.data, words)
        return cnt, down.astype(bool), bits

    def peers(self, i):
        k = self.lib.wpf_peer_count(self.h, int(i))
        out = np.zeros(max(k, 1), np.int32)
        self.lib.wpf_peers(self.h, int(i), out.ctypes.data)
        return out[:k]

    def avg_peers(self):
        return self.lib.wpf_avg_peers(self.h)

    def peek_messages(self, cap=1 << 16):
        """network.msgs.peekMessages(): (total, dict of from, to, sent_at, arriving_at) sorted by (arrivingAt, from, to, sentAt)"""
        a = [np.zeros(cap, np.int32) for _ in range(4)]
        total = self.lib.wpf_peek_messages(self.h, *[x.ctypes.data for x in a], int(cap))
        k = min(total, cap)
        return total, dict(zip(["from", "to", "sent_at", "arriving_at"], [x[:k] for x in a]))

    def _c(self, op, arg=0):
        self._check(self.lib.wpf_net_ctl(self.h, op, int(arg)))

    def stop_node(self, i):
        self._c(0, i)

    def start_node(self, i):
        self._c(1, i)

    def partition(self, part):
        self._c(2, round(part * 10000))

    def end_partition(self):
        self._c(3)
