"""Host-side mirrors of the reference protocols whose `Message.action` bodies run as device
state-transition kernels: same constructor parameters, `init()`, `network()`, `copy()`.

Reference: protocols/src/main/java/net/consensys/wittgenstein/protocols/PingPong.java and
GSFSignature.java; core/Protocol.java:7-22.
"""
import ctypes as C

import numpy as np

from ._lib import WtgError
from .network import Network, _p


class PingPongParameters:
    """PingPong.PingPongParameters (PingPong.java:34-50)."""

    def __init__(self, node_ct=1000, node_builder_name=None, network_latency_name=None):
        self.node_ct = node_ct
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class PingPong:
    def __init__(self, params=None, _api=None):
        self.params = params or PingPongParameters()
        self._api = _api
        self._net = Network(_api)
        self._net.set_node_builder(self.params.node_builder_name)  # RegistryNodeBuilders.getByName (PingPong.java:54)
        self._net.set_network_latency(self.params.network_latency_name)  # :55-56

    def network(self):
        return self._net

    def copy(self):
        return PingPong(self.params, self._api)

    def init(self):
        self._net.api.check(self._net.api.pingpong_init(self._net.h, int(self.params.node_ct)))

    def pongs(self):
        out = np.zeros(self._net.node_count, np.int32)
        self._net.api.check(self._net.api.pingpong_pongs(self._net.h, _p(out, C.c_int)))
        return out


class GSFSignatureParameters:
    """GSFSignature.GSFSignatureParameters (GSFSignature.java:27-107); ratios are accepted like the
    second constructor (:86-106) when threshold / nodes_down are floats."""

    def __init__(self, node_count=32768 // 32, threshold=None, pairing_time=3, timeout_per_level_ms=50, period_duration_ms=10,
                 accelerated_calls_count=10, nodes_down=0, node_builder_name=None, network_latency_name=None):
        if threshold is None:
            threshold = int(node_count * 0.99)
        if isinstance(threshold, float):
            threshold = int(threshold * node_count)
        if isinstance(nodes_down, float):
            nodes_down = int(nodes_down * node_count)
        if nodes_down >= node_count or nodes_down < 0 or threshold > node_count or nodes_down + threshold > node_count:
            raise WtgError(f"nodeCount={node_count}, threshold={threshold}")  # :69-74
        self.node_count = node_count
        self.threshold = threshold
        self.pairing_time = pairing_time
        self.timeout_per_level_ms = timeout_per_level_ms
        self.period_duration_ms = period_duration_ms
        self.accelerated_calls_count = accelerated_calls_count
        self.nodes_down = nodes_down
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class GSFSignature:
    def __init__(self, params, _api=None, tunables=None, shard=None, device=None):
        self.params = params
        self._api = _api
        self._tunables = dict(tunables or {})
        self._net = Network(_api, device=device, shard=shard)
        self._net.set_node_builder(params.node_builder_name)  # GSFSignature.java:111
        self._net.set_network_latency(params.network_latency_name)  # :112-113
        for k, v in self._tunables.items():
            self._net.set_tunable(k, v)

    def network(self):
        return self._net

    def copy(self):
        return GSFSignature(self.params, self._api, self._tunables)

    def init(self):
        p = self.params
        arr = np.array([p.node_count, p.threshold, p.pairing_time, p.timeout_per_level_ms, p.period_duration_ms,
                        p.accelerated_calls_count, p.nodes_down], np.int32)
        self._net.api.check(self._net.api.gsf_init(self._net.h, _p(arr, C.c_int)))
        self.levels = self._net.api.gsf_levels(self._net.h)
        self.words = max(1, p.node_count // 64)
        self.rows_local = self._net.local_count  # a shard reads back its own nodes

    # ---- read-back of node state (GSFNode fields) ----
    def verified(self):
        """verifiedSignatures of every node: uint64 [N, N/64]; bit i of the set = bit i%64 of word i//64."""
        out = np.zeros((self.rows_local, self.words), np.uint64)
        self._net.api.check(self._net.api.gsf_verified(self._net.h, _p(out, C.c_ulonglong)))
        return out

    def rows(self, which):
        """0 verified, 1 individualSignatures (union over levels), 2 indivVerifiedSig (union over levels)."""
        out = np.zeros((self.rows_local, self.words), np.uint64)
        self._net.api.check(self._net.api.gsf_rows(self._net.h, int(which), _p(out, C.c_ulonglong)))
        return out

    def scalars(self):
        n = self.rows_local
        a = [np.zeros(n, np.int32) for _ in range(5)]
        self._net.api.check(self._net.api.gsf_node_scalars(self._net.h, *[_p(v, C.c_int) for v in a]))
        return dict(pairing=a[0], sig_checked=a[1], sig_queue_size=a[2], to_verify=a[3], card=a[4])

    def level_scalars(self):
        n, L = self.rows_local, self.levels
        a = [np.zeros((n, L), np.int32) for _ in range(3)]
        self._net.api.check(self._net.api.gsf_level_scalars(self._net.h, *[_p(v, C.c_int) for v in a]))
        return dict(pos=a[0], remaining=a[1], card=a[2])

    def peers(self, node, level):
        cap = max(1, self.params.node_count)
        out = np.zeros(cap, np.int32)
        k = self._net.api.check(self._net.api.gsf_peers(self._net.h, node, level, _p(out, C.c_int), cap))
        return out[:k].copy()

    def continue_if(self):
        """GSFSignature.newConfIf (:670-682): some live node is still below the threshold."""
        card = self.scalars()["card"]
        down = self._net.attrs()["down"]
        if self._net.shard is not None:
            n0, nl = self._net.shard_range()
            down = down[n0:n0 + nl]
        return bool(((card < self.params.threshold) & (down == 0)).any())


class SanFerminSignatureParameters:
    """SanFerminSignature.SanFerminSignatureParameters (SanFerminSignature.java:41-110)."""

    def __init__(self, node_count=32768 // 32, threshold=32768 // 32, pairing_time=2, signature_size=48, reply_timeout=300,
                 candidate_count=1, shuffled_lists=False, node_builder_name=None, network_latency_name=None):
        self.node_count = node_count
        self.threshold = threshold
        self.pairing_time = pairing_time
        self.signature_size = signature_size
        self.reply_timeout = reply_timeout
        self.candidate_count = candidate_count
        self.shuffled_lists = shuffled_lists  # unused by the reference as well
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class SanFerminSignature:
    """The reference builds its nodes in the constructor (SanFerminSignature.java:112-129); so does this mirror."""

    def __init__(self, params, _api=None):
        self.params = params
        self._api = _api
        self._net = Network(_api)
        self._net.set_node_builder(params.node_builder_name)
        self._net.set_network_latency(params.network_latency_name)
        arr = np.array([params.node_count, params.threshold, params.pairing_time, params.signature_size, params.reply_timeout,
                        params.candidate_count], np.int32)
        self._net.api.check(self._net.api.sanfermin_construct(self._net.h, _p(arr, C.c_int)))

    def network(self):
        return self._net

    def copy(self):
        return SanFerminSignature(self.params, self._api)

    def init(self):
        self._net.api.check(self._net.api.sanfermin_init(self._net.h))

    def scalars(self):
        n = self.params.node_count
        a = [np.zeros(n, np.int32) for _ in range(7)]
        t = np.zeros(n, np.int64)
        self._net.api.check(self._net.api.sanfermin_node_scalars(self._net.h, *[_p(v, C.c_int) for v in a], _p(t, C.c_longlong)))
        d = dict(zip(["agg", "cpl", "done", "threshold_done", "sent_requests", "received_requests", "swapping"], a))
        d["threshold_at"] = t
        return d


class CasperParemeters:
    """CasperIMD.CasperParemeters (CasperIMD.java:18-71; the reference's spelling)."""

    SLOT_DURATION = 8000

    def __init__(self, cycle_length=4, random_on_ties=True, block_producers_count=2, attesters_per_round=20,
                 block_construction_time=1000, attestation_construction_time=1, node_builder_name=None, network_latency_name=None):
        self.cycle_length = cycle_length
        self.random_on_ties = random_on_ties
        self.block_producers_count = block_producers_count
        self.attesters_per_round = attesters_per_round
        self.attesters_count = attesters_per_round * cycle_length
        self.block_construction_time = block_construction_time
        self.attestation_construction_time = attestation_construction_time
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class CasperIMD:
    """CasperIMD (protocols/CasperIMD.java).  The constructor adds the observer (node 0, :81-88); init(byz_delay) is
    init(new ByzBlockProducerWF(byz_delay, genesis)) (:472-508): node 1 is the Byzantine producer, then the other
    producers, then the attesters.  Blocks are identified by their creation rank (genesis = 0)."""

    def __init__(self, params, _api=None, tunables=None, shard=None, device=None):
        self.params = params
        self._api = _api
        self._net = Network(_api, device=device, shard=shard)
        self._net.set_node_builder(params.node_builder_name)
        self._net.set_network_latency(params.network_latency_name)
        for k, v in dict(tunables or {}).items():
            self._net.set_tunable(k, v)
        arr = np.array([params.cycle_length, 1 if params.random_on_ties else 0, params.block_producers_count,
                        params.attesters_per_round, params.block_construction_time, params.attestation_construction_time], np.int32)
        self._net.api.check(self._net.api.casper_construct(self._net.h, _p(arr, C.c_int)))

    def network(self):
        return self._net

    def copy(self):
        return CasperIMD(self.params, self._api)

    def node_count(self):
        return 1 + self.params.block_producers_count + self.params.attesters_count

    BYZ_KINDS = {"plain": 3, "SF": 4, "NS": 5, "WF": 6}  # ByzBlockProducer, ...SF, ...NS, ...WF (CasperIMD.java:511-707)

    def init(self, byz_delay=0, byz_kind="WF"):
        self._net.api.check(self._net.api.casper_init_byz(self._net.h, self.BYZ_KINDS[byz_kind], int(byz_delay)))

    def blocks(self):
        a = self._net.api
        nb = a.check(a.casper_block_count(self._net.h))
        v = [np.zeros(nb, np.int32) for _ in range(5)]
        a.check(a.casper_blocks(self._net.h, *[_p(x, C.c_int) for x in v]))
        return dict(zip(["height", "parent", "producer", "proposal_time", "included"], v))

    def block_attestations(self, block):
        a = self._net.api
        cap = 1 << 16
        while True:
            att, h = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
            k = a.check(a.casper_block_attestations(self._net.h, int(block), _p(att, C.c_int), _p(h, C.c_int), cap))
            if k <= cap:
                return sorted(zip(att[:k].tolist(), h[:k].tolist()))
            cap = k

    def node_state(self):
        n = self._net.local_count  # a shard reads back its own nodes
        v = [np.zeros(n, np.int32) for _ in range(5)]
        hs = np.zeros(n, np.uint64)
        a = self._net.api
        a.check(a.casper_node_state(self._net.h, *[_p(x, C.c_int) for x in v], _p(hs, C.c_ulonglong)))
        d = dict(zip(["head", "atts_received", "heads_with_atts", "blocks_received", "to_reevaluate"], v))
        d["att_hash"] = hs
        return d

    def heads(self):
        out = np.zeros(self._net.local_count, np.int32)
        self._net.api.check(self._net.api.casper_heads(self._net.h, _p(out, C.c_int)))
        return out

    def byz(self):
        out = np.zeros(9, np.int32)
        self._net.api.check(self._net.api.casper_byz(self._net.h, _p(out, C.c_int)))
        return dict(zip(["to_send", "h", "late", "on_time", "delay", "on_direct_father", "on_older_ancestor", "inc_not_the_best_father",
                         "skipped"], out.tolist()))


class SanFerminCapposParameters:
    """SanFerminCappos.SanFerminParameters (SanFerminCappos.java:43-104)."""

    def __init__(self, node_count=32768 // 16, threshold=32768 // 32, pairing_time=2, signature_size=48, timeout=150, candidate_count=50,
                 node_builder_name=None, network_latency_name=None):
        self.node_count = node_count
        self.threshold = threshold
        self.pairing_time = pairing_time
        self.signature_size = signature_size
        self.timeout = timeout
        self.candidate_count = candidate_count
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class SanFerminCappos:
    """SanFerminCappos (protocols/SanFerminCappos.java); nodes are built by init() (:120-134)."""

    def __init__(self, params, _api=None, tunables=None):
        self.params = params
        self._api = _api
        self._tunables = dict(tunables or {})
        self._net = Network(_api)
        self._net.set_node_builder(params.node_builder_name)
        self._net.set_network_latency(params.network_latency_name)
        for k, v in self._tunables.items():
            self._net.set_tunable(k, v)

    def network(self):
        return self._net

    def copy(self):
        return SanFerminCappos(self.params, self._api, self._tunables)

    def init(self):
        p = self.params
        arr = np.array([p.node_count, p.threshold, p.pairing_time, p.signature_size, p.timeout, p.candidate_count], np.int32)
        self._net.api.check(self._net.api.cappos_init(self._net.h, _p(arr, C.c_int)))

    def scalars(self):
        n = self.params.node_count
        a = [np.zeros(n, np.int32) for _ in range(6)]
        t = np.zeros(n, np.int64)
        self._net.api.check(self._net.api.cappos_node_scalars(self._net.h, *[_p(v, C.c_int) for v in a], _p(t, C.c_longlong)))
        d = dict(zip(["cpl", "sigs", "done", "threshold_done", "swapping", "cache_mask"], a))
        d["threshold_at"] = t
        return d


class SlushParameters:
    """Slush.SlushParameters (Slush.java:14-52); the defaults are the JSON constructor's (100, 4, 7, 4)."""

    def __init__(self, nodes_av=100, m=4, k=7, a=4.0, node_builder_name=None, network_latency_name=None):
        self.nodes_av = nodes_av
        self.m = m
        self.k = k
        self.a = a
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class SnowflakeParameters:
    """Snowflake.SnowflakeParameters (Snowflake.java:18-61); the defaults are the JSON constructor's (100, 4, 7, 4, 7)."""

    def __init__(self, nodes_av=100, m=4, k=7, a=4.0, b=7, node_builder_name=None, network_latency_name=None):
        self.nodes_av = nodes_av
        self.m = m
        self.k = k
        self.a = a
        self.b = b
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class _Avalanche:
    """Slush / Snowflake (protocols/Slush.java, Snowflake.java): nodes are built by init(), which also sends the first two
    queries (node 0 with colour 1, node 1 with colour 2)."""

    def __init__(self, params, _api=None, tunables=None):
        self.params = params
        self._api = _api
        self._tunables = dict(tunables or {})
        self._net = Network(_api)
        self._net.set_node_builder(params.node_builder_name)
        self._net.set_network_latency(params.network_latency_name)
        for k, v in self._tunables.items():
            self._net.set_tunable(k, v)

    def network(self):
        return self._net

    def copy(self):
        return type(self)(self.params, self._api, self._tunables)

    def scalars(self):
        """per node: color, nonce, round (Slush) / cnt (Snowflake), pending, found1, found2 (colorsFound of the open query)"""
        n = self.params.nodes_av
        a = [np.zeros(n, np.int32) for _ in range(6)]
        self._net.api.check(self._net.api.avalanche_node_scalars(self._net.h, *[_p(v, C.c_int) for v in a]))
        return dict(zip(["color", "nonce", self._counter, "pending", "found1", "found2"], a))

    def serial_passes(self):
        """pipeline passes whose draw indices were re-derived serially (a query's sample discarded an attempt)"""
        return self._net.api.check(self._net.api.serial_passes(self._net.h))


class Slush(_Avalanche):
    _counter = "round"

    def init(self):
        p = self.params
        self._net.api.check(self._net.api.slush_init(self._net.h, int(p.nodes_av), int(p.m), int(p.k), float(p.a)))


class Snowflake(_Avalanche):
    _counter = "cnt"

    def init(self):
        p = self.params
        self._net.api.check(self._net.api.snowflake_init(self._net.h, int(p.nodes_av), int(p.m), int(p.k), float(p.a), int(p.b)))


class P2PFloodParameters:
    """P2PFlood.P2PFloodParameters (P2PFlood.java:46-109); the defaults are the JSON constructor's (100, 10, 50, 1, 1, 10, 30).
    msg_to_receive is kept for scenario code: the protocol itself never reads it."""

    def __init__(self, node_count=100, dead_node_count=10, delay_before_resent=50, msg_count=1, msg_to_receive=1, peers_count=10,
                 delay_between_sends=30, node_builder_name=None, network_latency_name=None):
        self.node_count = node_count
        self.dead_node_count = dead_node_count
        self.delay_before_resent = delay_before_resent
        self.msg_count = msg_count
        self.msg_to_receive = msg_to_receive
        self.peers_count = peers_count
        self.delay_between_sends = delay_between_sends
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name


class P2PFlood:
    """protocols/P2PFlood.java on a P2PNetwork (core/P2PNetwork.java, minimum = true): init() builds the nodes (the first
    dead_node_count stopped), the peer graph, and sends msg_count messages from distinct live nodes to their peers.  Not
    available on a node-sharded network."""

    def __init__(self, params=None, _api=None, tunables=None):
        self.params = params or P2PFloodParameters()
        self._api = _api
        self._tunables = dict(tunables or {})
        self._net = Network(_api)
        self._net.set_node_builder(self.params.node_builder_name)
        self._net.set_network_latency(self.params.network_latency_name)
        for k, v in self._tunables.items():
            self._net.set_tunable(k, v)

    def network(self):
        return self._net

    def copy(self):
        return P2PFlood(self.params, self._api, self._tunables)

    def init(self):
        p = self.params
        self._net.api.check(self._net.api.p2pflood_init(self._net.h, int(p.node_count), int(p.dead_node_count), int(p.delay_before_resent),
                                                        int(p.msg_count), int(p.peers_count), int(p.delay_between_sends)))

    def peers(self, i):
        """P2PNode.peers of node i, in the reference's order (link creation)"""
        api = self._net.api
        k = api.check(api.p2p_peer_count(self._net.h, int(i)))
        out = np.zeros(max(k, 1), np.int32)
        api.check(api.p2p_peers(self._net.h, int(i), _p(out, C.c_int), k))
        return out[:k]

    def avg_peers(self):
        """P2PNetwork.avgPeers()"""
        return self._net.api.check(self._net.api.p2p_avg_peers(self._net.h))

    def received_count(self):
        """getMsgReceived(-1).size() of every node"""
        out = np.zeros(self.params.node_count, np.int32)
        self._net.api.check(self._net.api.p2pflood_received(self._net.h, _p(out, C.c_int), 0, None))
        return out

    def received(self, i):
        """which originating messages (init's draw order) node i has received: a bool array of msg_count"""
        cnt = np.zeros(self.params.node_count, np.int32)
        words = max(1, (int(self.params.msg_count) + 63) // 64)
        bits = np.zeros(words, np.uint64)
        self._net.api.check(self._net.api.p2pflood_received(self._net.h, _p(cnt, C.c_int), int(i), _p(bits, C.c_ulonglong)))
        return np.unpackbits(bits.view(np.uint8), bitorder="little")[:self.params.msg_count].astype(bool)

    def serial_passes(self):
        """pipeline passes whose draw indices were re-derived serially (a shuffle's nextInt rejected)"""
        return self._net.api.check(self._net.api.serial_passes(self._net.h))


class HandelParameters:
    """Handel.HandelParameters (Handel.java:22-142); window = WindowParameters() (16, 1, 128, ScoringExp(2, 4))."""

    def __init__(self, node_count=32, threshold=None, pairing_time=3, level_wait_time=50, extra_cycle=10,
                 dissemination_period_ms=10, fast_path=10, nodes_down=0, node_builder_name=None, network_latency_name=None,
                 desynchronized_start=0, byzantine_suicide=False, hidden_byzantine=False):
        if threshold is None:
            threshold = int(node_count * 0.99)
        if nodes_down >= node_count or nodes_down < 0 or threshold > node_count or nodes_down + threshold > node_count:
            raise WtgError(f"nodeCount={node_count}, threshold={threshold}")  # :112-117
        if bin(node_count).count("1") != 1:
            raise WtgError("We support only power of two nodes in this simulation")  # :118-120
        if byzantine_suicide and hidden_byzantine:
            raise WtgError("Only one attack at a time")  # :122-124
        self.node_count = node_count
        self.threshold = threshold
        self.pairing_time = pairing_time
        self.level_wait_time = level_wait_time
        self.extra_cycle = extra_cycle
        self.dissemination_period_ms = dissemination_period_ms
        self.fast_path = fast_path
        self.nodes_down = nodes_down
        self.node_builder_name = node_builder_name
        self.network_latency_name = network_latency_name
        self.desynchronized_start = desynchronized_start
        self.byzantine_suicide = byzantine_suicide
        self.hidden_byzantine = hidden_byzantine


class Handel:
    def __init__(self, params, _api=None, tunables=None, shard=None, device=None):
        """shard = (rank, world): this object is one node-id shard of a network spread over `world` engines (sharded.py);
        its node-indexed read-backs cover its own ids."""
        self.params = params
        self._api = _api
        self._tunables = dict(tunables or {})
        self._net = Network(_api, device=device, shard=shard)
        self._net.set_network_latency(params.network_latency_name)  # Handel.java:214-215
        for k, v in self._tunables.items():
            self._net.set_tunable(k, v)

    def network(self):
        return self._net

    def copy(self):
        return Handel(self.params, self._api, self._tunables)

    def init(self):
        p = self.params
        self._net.set_node_builder(p.node_builder_name)  # :958
        arr = np.array([p.node_count, p.threshold, p.pairing_time, p.level_wait_time, p.extra_cycle, p.dissemination_period_ms,
                        p.fast_path, p.nodes_down, p.desynchronized_start, int(p.byzantine_suicide), int(p.hidden_byzantine)], np.int32)
        self._net.api.check(self._net.api.handel_init(self._net.h, _p(arr, C.c_int)))
        self.levels = self._net.api.handel_levels(self._net.h)
        self.words = max(1, p.node_count // 64)
        self.rows_local = self._net.local_count  # a shard reads back its own nodes

    def scalars(self):
        n = self.rows_local
        out = np.zeros((9, n), np.int32)
        self._net.api.check(self._net.api.handel_node_scalars(self._net.h, _p(out, C.c_int)))
        keys = ["start_at", "pairing", "sigs_checked", "sig_queue_size", "msg_filtered", "window", "added_cycle", "total_sig_size", "queued"]
        return {k: out[i] for i, k in enumerate(keys)}

    def rows(self, which):
        out = np.zeros((self.rows_local, self.words), np.uint64)
        self._net.api.check(self._net.api.handel_rows(self._net.h, int(which), _p(out, C.c_ulonglong)))
        return out

    def level_scalars(self):
        n, L = self.rows_local, self.levels
        a = [np.zeros((n, L), np.int32) for _ in range(3)]
        self._net.api.check(self._net.api.handel_level_scalars(self._net.h, *[_p(v, C.c_int) for v in a]))
        return dict(pos=a[0], outgoing_finished=a[1], suicide_biz_after=a[2])

    def peers(self, node, level):
        """emission list of `node` at `level`; on a sharded network only for the shard's own nodes"""
        out = np.zeros(max(1, self.params.node_count), np.int32)
        k = self._net.api.check(self._net.api.handel_peers(self._net.h, node, level, _p(out, C.c_int), self.params.node_count))
        return out[:k].copy()

    def ranks(self, node):
        """receptionRanks of `node`; on a sharded network only for the shard's own nodes"""
        out = np.zeros(self.params.node_count, np.int32)
        self._net.api.check(self._net.api.handel_ranks(self._net.h, node, _p(out, C.c_int)))
        return out

    def continue_if(self):
        """Handel.newContIf (:1044-1053); a shard answers for its own nodes."""
        c = self._net.counters()
        down = self._net.attrs()["down"]
        if self._net.shard is not None:
            n0, nl = self._net.shard_range()
            down = down[n0:n0 + nl]
        sc = self.scalars()
        return bool((((c[4] == 0) | (sc["added_cycle"] > 0)) & (down == 0)).any())
