"""One simulation spread over several engines by node id (DESIGN.md §8): shard r owns the ids [r*N/G, (r+1)*N/G).

Two ways to drive the same C ABI (include/wtg.h, `wtg_shard_*`):

* `ShardedGSFSignature`, `ShardedHandel`, `ShardedCasperIMD` — all shards in this process, one host thread per shard (the
  engines may sit on different GPUs of the box, or share one): what a single-process caller such as the reference's JVM
  would do through JNI.
* `DistributedGSFSignature`, `DistributedHandel`, `DistributedCasperIMD` — one shard per process (torchrun: one rank per GPU); the 128-byte handles (CUDA IPC) of the
  exchange regions travel through `torch.distributed`, after that the data path is peer stores between the GPUs'
  kernels — no collective call per tick.

Every shard is configured with identical calls; node-indexed read-backs are concatenated in rank order, so the result
has the layout of the unsharded protocol object (and is compared with it / the oracle by the tests).
"""
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .protocols import CasperIMD, GSFSignature, Handel


class _ShardedNetwork:
    def __init__(self, owner):
        self._o = owner

    def _each(self, fn):
        return self._o._each(fn)

    def set_seed(self, seed):
        self._each(lambda s: s.network().set_seed(seed))

    def set_tunable(self, k, v):
        self._each(lambda s: s.network().set_tunable(k, v))

    def run_ms(self, ms):
        return any(self._each(lambda s: s.network().run_ms(ms)))

    @property
    def time(self):
        return self._o.shards[0].network().time

    @property
    def node_count(self):
        return self._o.shards[0].network().node_count

    def rng_state(self):
        st = set(self._each(lambda s: s.network().rng_state()))
        assert len(st) == 1, "shards disagree on the rd state"
        return st.pop()

    def msgs_size(self):
        return sum(self._each(lambda s: s.network().msgs_size()))

    def counters(self):
        return np.concatenate(self._each(lambda s: s.network().counters()), axis=1)

    def peek_messages(self, cap=1 << 16):
        """network.msgs.peekMessages(): every pending arrival is reported by exactly one shard; merged and sorted like the
        unsharded read-back (arrivingAt, from, to, sentAt)"""
        parts = self._each(lambda s: s.network().peek_messages(cap))
        total = sum(p[0] for p in parts)
        rows = {k: np.concatenate([p[1][k] for p in parts]) for k in parts[0][1]}
        order = np.lexsort((rows["sent_at"], rows["to"], rows["from"], rows["arriving_at"]))
        return total, {k: v[order] for k, v in rows.items()}

    def attrs(self):
        return self._o.shards[0].network().attrs()

    def stop_node(self, i):
        self._each(lambda s: s.network().stop_node(i))

    def start_node(self, i):
        self._each(lambda s: s.network().start_node(i))

    def partition(self, part):
        self._each(lambda s: s.network().partition(part))

    def end_partition(self):
        self._each(lambda s: s.network().end_partition())

    def stats(self):
        sts = self._each(lambda s: s.network().stats())
        out = dict(sts[0])
        for k in ("deliveries", "tasks", "cond_runs", "eval_entries", "eval_words", "updates", "cycles", "sends", "multi_sends",
                  "send_words", "update_words", "reevaluated", "kernel_launches"):
            out[k] = sum(st[k] for st in sts)
        for k in ("max_queue", "max_bucket", "max_inbox"):
            out[k] = max(st[k] for st in sts)
        return out

    def timer_start(self):
        self._each(lambda s: s.network().timer_start())

    def timer_stop_ms(self):
        return max(self._each(lambda s: s.network().timer_stop_ms()))


class ShardedGSFSignature:
    """GSFSignature over `world` node-id shards driven from this process (one thread per shard)."""

    def __init__(self, params, world, devices=None, _api=None, tunables=None):
        self.params = params
        self.world = world
        self.devices = list(devices) if devices is not None else [None] * world
        self.shards = [GSFSignature(params, _api, tunables, shard=(r, world), device=self.devices[r]) for r in range(world)]
        self._pool = ThreadPoolExecutor(max_workers=world)
        self._net = _ShardedNetwork(self)

    def _each(self, fn):
        return list(self._pool.map(fn, self.shards))

    def network(self):
        return self._net

    def init(self):
        self._each(lambda s: s.init())
        handles = [s.network().shard_export() for s in self.shards]
        self._each(lambda s: s.network().shard_link(handles))
        self.levels = self.shards[0].levels
        self.words = self.shards[0].words

    def verified(self):
        return np.concatenate(self._each(lambda s: s.verified()), axis=0)

    def rows(self, which):
        return np.concatenate(self._each(lambda s: s.rows(which)), axis=0)

    def scalars(self):
        parts = self._each(lambda s: s.scalars())
        return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}

    def level_scalars(self):
        parts = self._each(lambda s: s.level_scalars())
        return {k: np.concatenate([p[k] for p in parts], axis=0) for k in parts[0]}

    def peers(self, node, level):
        nl = self.params.node_count // self.world
        return self.shards[node // nl].peers(node, level)

    def continue_if(self):
        return any(self._each(lambda s: s.continue_if()))

    def close(self):
        self._pool.shutdown(wait=True)
        for s in self.shards:
            s.network().close()


class ShardedHandel:
    """Handel (BASELINE config #3) over `world` node-id shards driven from this process (one thread per shard).  Every shard
    runs the whole host init; the level draws of checkSigs are ordered over the shards by the pick exchange, and pooled
    payloads for another shard's nodes go through its staging area (DESIGN.md §8)."""

    def __init__(self, params, world, devices=None, _api=None, tunables=None):
        self.params = params
        self.world = world
        self.devices = list(devices) if devices is not None else [None] * world
        self.shards = [Handel(params, _api, tunables, shard=(r, world), device=self.devices[r]) for r in range(world)]
        self._pool = ThreadPoolExecutor(max_workers=world)
        self._net = _ShardedNetwork(self)

    def _each(self, fn):
        return list(self._pool.map(fn, self.shards))

    def network(self):
        return self._net

    def init(self):
        self._each(lambda s: s.init())
        handles = [s.network().shard_export() for s in self.shards]
        self._each(lambda s: s.network().shard_link(handles))
        self.levels = self.shards[0].levels
        self.words = self.shards[0].words

    def _owner(self, node):
        return self.shards[node // (self.params.node_count // self.world)]

    def scalars(self):
        parts = self._each(lambda s: s.scalars())
        return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}

    def rows(self, which):
        return np.concatenate(self._each(lambda s: s.rows(which)), axis=0)

    def level_scalars(self):
        parts = self._each(lambda s: s.level_scalars())
        return {k: np.concatenate([p[k] for p in parts], axis=0) for k in parts[0]}

    def peers(self, node, level):
        return self._owner(node).peers(node, level)

    def ranks(self, node):
        return self._owner(node).ranks(node)

    def continue_if(self):
        return any(self._each(lambda s: s.continue_if()))

    def close(self):
        self._pool.shutdown(wait=True)
        for s in self.shards:
            s.network().close()


class ShardedCasperIMD:
    """CasperIMD (BASELINE config #4) over `world` node-id shards driven from this process (one thread per shard): ids split
    into `world` contiguous ranges; the block and attestation tables are replicated (their creator stores into every copy),
    a sendAll is published once and every shard builds the same sorted record; the fast-forward over idle milliseconds takes the
    minimum of the shards' next events at the start of every pass (DESIGN.md §8)."""

    def __init__(self, params, world, devices=None, _api=None, tunables=None):
        self.params = params
        self.world = world
        self.devices = list(devices) if devices is not None else [None] * world
        self.shards = [CasperIMD(params, _api, tunables, shard=(r, world), device=self.devices[r]) for r in range(world)]
        self._pool = ThreadPoolExecutor(max_workers=world)
        self._net = _ShardedNetwork(self)

    def _each(self, fn):
        return list(self._pool.map(fn, self.shards))

    def network(self):
        return self._net

    def node_count(self):
        return self.shards[0].node_count()

    def init(self, byz_delay=0, byz_kind="WF"):
        self._each(lambda s: s.init(byz_delay, byz_kind))
        handles = [s.network().shard_export() for s in self.shards]
        self._each(lambda s: s.network().shard_link(handles))

    def blocks(self):
        return self.shards[0].blocks()  # replicated table

    def block_attestations(self, block):
        return self.shards[0].block_attestations(block)

    def node_state(self):
        parts = self._each(lambda s: s.node_state())
        return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}

    def heads(self):
        return np.concatenate(self._each(lambda s: s.heads()))

    def byz(self):
        return self.shards[0].byz()  # node 1 (the Byzantine producer) lives on shard 0

    def close(self):
        self._pool.shutdown(wait=True)
        for s in self.shards:
            s.network().close()


class DistributedCasperIMD:
    """This process's shard of a CasperIMD network spread over the ranks of a torch.distributed group (one GPU each): the
    handles of the exchange regions travel once through `torch.distributed`; the data path is peer stores between kernels."""

    def __init__(self, params, dist, rank, world, device, tunables=None, _api=None):
        self.params, self.dist, self.rank, self.world = params, dist, rank, world
        self.local = CasperIMD(params, _api, tunables, shard=(rank, world), device=device)

    def network(self):
        return self.local.network()

    def init(self, byz_delay=0, byz_kind="WF"):
        self.local.init(byz_delay, byz_kind)
        mine = self.local.network().shard_export()
        handles = [None] * self.world
        self.dist.all_gather_object(handles, mine)
        self.local.network().shard_link(handles)
        self.dist.barrier()

    def heads(self):
        """heads of this shard's nodes"""
        return self.local.heads()

    def all_heads(self):
        parts = [None] * self.world
        self.dist.all_gather_object(parts, self.local.heads())
        return np.concatenate(parts)

    def blocks(self):
        return self.local.blocks()


class DistributedGSFSignature:
    """This process's shard of a GSFSignature network spread over the ranks of a torch.distributed group (one GPU each)."""

    def __init__(self, params, dist, rank, world, device, tunables=None, _api=None):
        self.params, self.dist, self.rank, self.world = params, dist, rank, world
        self.local = GSFSignature(params, _api, tunables, shard=(rank, world), device=device)

    def network(self):
        return self.local.network()

    def init(self):
        self.local.init()
        mine = self.local.network().shard_export()
        handles = [None] * self.world
        self.dist.all_gather_object(handles, mine)
        self.local.network().shard_link(handles)
        self.dist.barrier()
        self.levels, self.words = self.local.levels, self.local.words

    def scalars(self):
        return self.local.scalars()

    def continue_if(self):
        """some live node of some shard is still below the threshold"""
        import torch

        dev = f"cuda:{self.local.network().device}" if self.dist.get_backend() == "nccl" else "cpu"
        t = torch.tensor([1 if self.local.continue_if() else 0], dtype=torch.int32, device=dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return bool(t.item())


class DistributedHandel:
    """This process's shard of a Handel network spread over the ranks of a torch.distributed group (one GPU each)."""

    def __init__(self, params, dist, rank, world, device, tunables=None, _api=None):
        self.params, self.dist, self.rank, self.world = params, dist, rank, world
        self.local = Handel(params, _api, tunables, shard=(rank, world), device=device)

    def network(self):
        return self.local.network()

    def init(self):
        self.local.init()
        mine = self.local.network().shard_export()
        handles = [None] * self.world
        self.dist.all_gather_object(handles, mine)
        self.local.network().shard_link(handles)
        self.dist.barrier()
        self.levels, self.words = self.local.levels, self.local.words

    def continue_if(self):
        """Handel.newContIf over all shards: some live node of some shard has not finished (or still has extra cycles)"""
        parts = [None] * self.world
        self.dist.all_gather_object(parts, self.local.continue_if())
        return any(parts)
