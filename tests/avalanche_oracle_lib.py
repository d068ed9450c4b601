"""ctypes binding of the CPU restatement of Slush / Snowflake (tests/avalanche_oracle) — TEST INFRASTRUCTURE ONLY.

The restatement sits on the oracle's core (oracle/core.hpp: Network, Node, Message, java.util.Random) and is compiled on
first use.  Only tests/ and scripts/ may import this module; the product package never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC_DIR = os.path.join(ROOT, "tests", "avalanche_oracle")
ORACLE_DIR = os.path.join(ROOT, "oracle")
_lib = None


def load():
    global _lib
    if _lib is not None:
        return _lib
    so = os.path.join(SRC_DIR, "libwtg_avalanche_oracle.so")
    srcs = [os.path.join(SRC_DIR, f) for f in ("avalanche.hpp", "capi.cpp")]
    srcs += [os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith((".hpp", ".inc"))]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wextra", "-ffp-contract=off", "-fno-fast-math",
                               "-o", so, os.path.join(SRC_DIR, "capi.cpp")])
    lib = C.CDLL(so)
    lib.wav_last_error.restype = C.c_char_p
    lib.wav_create.restype = C.c_void_p
    lib.wav_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_char_p, C.c_char_p]
    for name in ("wav_destroy", "wav_init", "wav_time", "wav_msgs_size", "wav_node_counters", "wav_node_scalars"):
        getattr(lib, name).argtypes = None
    lib.wav_set_seed.argtypes = [C.c_void_p, C.c_int64]
    lib.wav_run_ms.argtypes = [C.c_void_p, C.c_int]
    lib.wav_run_timed.restype = C.c_double
    lib.wav_run_timed.argtypes = [C.c_void_p, C.c_int]
    lib.wav_net_ctl.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.wav_rng_state.restype = C.c_uint64
    lib.wav_msgs_live.restype = C.c_int64
    lib.wav_deliveries.restype = C.c_int64
    _lib = lib
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _b(s):
    return None if s is None else s.encode()


class _OracleAvalanche:
    _counter = None
    _b = -1

    def __init__(self, nodes_av, m, k, a, b, node_builder, latency, seed=None):
        self.lib = load()
        self.n = nodes_av
        self.h = C.c_void_p(self.lib.wav_create(nodes_av, m, k, float(a), b, _b(node_builder), _b(latency)))
        if not self.h:
            raise ValueError(self.lib.wav_last_error().decode())
        if seed is not None:
            self.lib.wav_set_seed(self.h, C.c_int64(seed))

    def __del__(self):
        try:
            self.lib.wav_destroy(self.h)
        except Exception:  # noqa: BLE001
            pass

    def _check(self, r):
        if r < 0:
            raise RuntimeError(self.lib.wav_last_error().decode())
        return r

    def init(self):
        self._check(self.lib.wav_init(self.h))

    def run_ms(self, ms):
        return bool(self._check(self.lib.wav_run_ms(self.h, ms)))

    def run(self, seconds):
        return self.run_ms(seconds * 1000)

    def run_timed(self, ms):
        """runMs(ms) and the host time it took, in ms"""
        t = self.lib.wav_run_timed(self.h, ms)
        if t < 0:
            raise RuntimeError(self.lib.wav_last_error().decode())
        return t

    @property
    def time(self):
        return self.lib.wav_time(self.h)

    def msgs_size(self):
        return self.lib.wav_msgs_size(self.h)

    def msgs_live(self):
        return self.lib.wav_msgs_live(self.h)

    def deliveries(self):
        return int(self.lib.wav_deliveries(self.h))

    def rng_state(self):
        return int(self.lib.wav_rng_state(self.h))

    def counters(self):
        out = np.zeros((5, self.n), np.int64)
        self.lib.wav_node_counters(self.h, _p(out, C.c_int64))
        return out

    def scalars(self):
        """per node: color, nonce, round / cnt, pending, found1, found2 — the keys of Slush / Snowflake.scalars()"""
        a = [np.zeros(self.n, np.int32) for _ in range(6)]
        self.max_open = self.lib.wav_node_scalars(self.h, *[_p(v, C.c_int32) for v in a])
        return dict(zip(["color", "nonce", self._counter, "pending", "found1", "found2"], a))

    def stop_node(self, i):
        self._check(self.lib.wav_net_ctl(self.h, 0, int(i)))

    def start_node(self, i):
        self._check(self.lib.wav_net_ctl(self.h, 1, int(i)))

    def partition(self, part):
        self._check(self.lib.wav_net_ctl(self.h, 2, round(part * 10000)))

    def end_partition(self):
        self._check(self.lib.wav_net_ctl(self.h, 3, 0))


class OracleSlush(_OracleAvalanche):
    """protocols/Slush.java through the CPU restatement."""

    _counter = "round"

    def __init__(self, nodes_av=100, m=4, k=7, a=4.0, node_builder=None, latency=None, seed=None):
        super().__init__(nodes_av, m, k, a, -1, node_builder, latency, seed)


class OracleSnowflake(_OracleAvalanche):
    """protocols/Snowflake.java through the CPU restatement."""

    _counter = "cnt"

    def __init__(self, nodes_av=100, m=4, k=7, a=4.0, b=7, node_builder=None, latency=None, seed=None):
        if b < 0:
            raise ValueError("B must be >= 0")
        super().__init__(nodes_av, m, k, a, b, node_builder, latency, seed)
