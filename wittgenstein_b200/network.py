"""Host-side mirror of the reference's `Network` surface for the accelerated path.

Reference: core/src/main/java/net/consensys/wittgenstein/core/Network.java — `rd.setSeed` (:32),
`setNetworkLatency` (:665-677), `runMs` / `run` (:306-338), `time` (:49), `msgs.size()` /
`msgs.sizeAt` (:204-220), `partition` / `endPartition` (:693-707), `Node.stop/start`
(core/Node.java:120-127), per-node counters (core/Node.java:72-79).
Every method is a thin call through the C ABI declared in include/wtg.h.
"""
import ctypes as C
import threading

import numpy as np

from . import _lib
from ._lib import WtgError


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


_tls = threading.local()


def set_thread_device(device):
    """Networks created by this thread from now on live on CUDA device `device` (None: the library's default).  Lets one
    process spread independent runs — RunMultipleTimes / ProgressPerTime seeds — over several GPUs, one thread per run."""
    _tls.device = device


class Network:
    def __init__(self, _api=None, device=None, shard=None):
        """shard = (rank, world): this object is one node-id shard of a network spread over `world` engines (sharded.py)."""
        self.api = _api or _lib.api()
        if device is None:
            device = getattr(_tls, "device", None)
        self.shard = shard
        if shard is not None:
            self.h = C.c_void_p(self.api.shard_create(int(shard[0]), int(shard[1]), -1 if device is None else int(device)))
        else:
            self.h = C.c_void_p(self.api.create() if device is None else self.api.create_on(int(device)))
        if not self.h:
            raise WtgError(self.api.last_error().decode())

    # ---- node-sharded networks ----
    def shard_range(self):
        """(first id, count) of the nodes this engine owns; node-indexed read-backs cover exactly these."""
        a, b = C.c_int(0), C.c_int(0)
        self.api.check(self.api.shard_range(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def shard_export(self):
        buf = (C.c_ubyte * 128)()
        self.api.check(self.api.shard_export(self.h, buf))
        return bytes(buf)

    def shard_link(self, handles):
        """handles: the 128-byte exports of all shards in rank order (shards of this process are mapped directly, shards of
        other processes through CUDA IPC)."""
        blob = (C.c_ubyte * (128 * len(handles))).from_buffer_copy(b"".join(handles))
        self.api.check(self.api.shard_link(self.h, blob))

    @property
    def device(self):
        return self.api.device(self.h)

    @property
    def local_count(self):
        return self.shard_range()[1] if self.shard is not None else self.node_count

    def close(self):
        if getattr(self, "h", None):
            self.api.destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- configuration ----
    def set_seed(self, seed):
        """network.rd.setSeed(seed) — before Protocol.init() (RunMultipleTimes.java:47)."""
        self.api.check(self.api.set_seed(self.h, int(seed)))

    def set_network_latency(self, name):
        """RegistryNetworkLatencies.getByName(name); None -> NetworkLatencyByDistanceWJitter."""
        self.api.check(self.api.set_network_latency(self.h, None if name is None else name.encode()))

    def set_network_latency_measured(self, proportions, values):
        p = np.asarray(proportions, np.int32)
        v = np.asarray(values, np.int32)
        self.api.check(self.api.set_network_latency_measured(self.h, _p(p, C.c_int), _p(v, C.c_int), len(p)))

    def set_node_builder(self, name):
        self.api.check(self.api.set_node_builder(self.h, None if name is None else name.encode()))

    def set_msg_discard_time(self, ms):
        self.api.check(self.api.set_msg_discard_time(self.h, int(ms)))

    def set_tunable(self, key, value):
        self.api.check(self.api.set_tunable(self.h, key.encode(), int(value)))

    # ---- sends issued by the caller (Network.java:341-366) ----
    def send(self, msg_type, from_id, to, payload=0, send_time=None, delay_between=0):
        """network.send(msg, from, to) / send(msg, from, dests): `to` is a node id or a list of ids.  With
        `send_time` (> time): send(msg, sendTime, from, to) / send(msg, sendTime, from, dests, delaysBetweenMessage)."""
        dests = np.asarray([to] if np.isscalar(to) else list(to), np.int32)
        if send_time is None:
            self.api.check(self.api.send(self.h, int(msg_type), C.c_ulonglong(int(payload)), int(from_id), _p(dests, C.c_int), len(dests)))
        else:
            self.api.check(self.api.send_at(self.h, int(msg_type), C.c_ulonglong(int(payload)), int(from_id), _p(dests, C.c_int), len(dests),
                                            int(send_time), int(delay_between)))

    def send_all(self, msg_type, from_id, payload=0):
        """network.sendAll(msg, from)"""
        self.api.check(self.api.send_all(self.h, int(msg_type), C.c_ulonglong(int(payload)), int(from_id)))

    # ---- run ----
    def run_ms(self, ms):
        return bool(self.api.check(self.api.run_ms(self.h, int(ms))))

    def run(self, seconds):
        return self.run_ms(seconds * 1000)

    @property
    def time(self):
        return self.api.time(self.h)

    @property
    def node_count(self):
        return self.api.node_count(self.h)

    def msgs_size(self):
        return self.api.check(self.api.msgs_size(self.h))

    def msgs_size_at(self, t):
        return self.api.check(self.api.msgs_size_at(self.h, int(t)))

    def peek_messages(self, cap=1 << 16):
        """network.msgs.peekMessages() (Network.java:279-286): (total, rows) with rows = dict of int32 arrays from, to, sent_at,
        arriving_at, kind, msg_type, sorted by arrival; at most `cap` rows."""
        a = [np.zeros(cap, np.int32) for _ in range(6)]
        total = self.api.check(self.api.peek_messages(self.h, *[_p(x, C.c_int) for x in a], int(cap)))
        k = min(total, cap)
        return total, dict(zip(["from", "to", "sent_at", "arriving_at", "kind", "msg_type"], [x[:k] for x in a]))

    def stop_node(self, node_id):
        self.api.check(self.api.stop_node(self.h, int(node_id)))

    def start_node(self, node_id):
        self.api.check(self.api.start_node(self.h, int(node_id)))

    def partition(self, part):
        self.api.check(self.api.partition(self.h, float(part)))

    def end_partition(self):
        self.api.check(self.api.end_partition(self.h))

    def rng_state(self):
        return int(self.api.rng_state(self.h))

    # ---- read-back ----
    def counters(self):
        """rows: msgReceived, msgSent, bytesSent, bytesReceived, doneAt (int64, [5, N])."""
        out = np.zeros((5, self.local_count), np.int64)
        self.api.check(self.api.node_counters(self.h, _p(out, C.c_longlong)))
        return out

    def attrs(self):
        n = self.node_count
        x = np.zeros(n, np.int32); y = np.zeros(n, np.int32); e = np.zeros(n, np.int32); c = np.zeros(n, np.int32)
        s = np.zeros(n, np.float64); d = np.zeros(n, np.uint8)
        self.api.check(self.api.node_attrs(self.h, _p(x, C.c_int), _p(y, C.c_int), _p(e, C.c_int), _p(c, C.c_int),
                                           _p(s, C.c_double), _p(d, C.c_ubyte)))
        return dict(x=x, y=y, extra=e, city=c, speed=s, down=d)

    def stats(self):
        out = np.zeros(26, np.int64)
        self.api.check(self.api.stats(self.h, _p(out, C.c_longlong)))
        keys = ["deliveries", "tasks", "cond_runs", "draws", "eval_entries", "eval_words", "updates", "cycles", "sends",
                "multi_sends", "send_words", "events", "max_queue", "max_bucket", "max_inbox", "rec_top", "rec_dest_top",
                "kernel_launches", "min_pool_free", "init_draws", "ring", "bcap", "qcap", "peer_bits", "update_words", "reevaluated"]
        return dict(zip(keys, out.tolist()))

    # ---- measurement hooks ----
    def timer_start(self):
        self.api.check(self.api.timer_start(self.h))

    def timer_stop_ms(self):
        return float(self.api.timer_stop_ms(self.h))

    def profile_enable(self, on=True, split_scans=False):
        """split_scans: profile_read reports the delivery dispatch's scan A as k_scan_a_partial / k_scan_a_final; by default
        it is added into k_scan_partial / k_scan_final, which scan B (and Handel's draw scan) report"""
        self.api.check(self.api.profile_enable(self.h, (2 if split_scans else 1) if on else 0))

    def profile_read(self):
        cap = 64
        ms = (C.c_double * cap)()
        cnt = (C.c_longlong * cap)()
        names = (C.c_char_p * cap)()
        k = self.api.check(self.api.profile_read(self.h, ms, cnt, names, cap))
        return {names[i].decode(): (ms[i], cnt[i]) for i in range(k)}
