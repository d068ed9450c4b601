// wittgenstein_b200 — CUDA backend (sm_90a, H100): the kernels of the tick pipeline and the C ABI.
//
// One simulated millisecond = one pass of these kernels over SoA state resident in HBM:
//   k_begin -> { C: k_cond_mark / k_cond_nodes<scan> / k_cond_score / k_cond_nodes<select> (conditional tasks)
//              | D: k_dispatch_count -> pair scan A -> k_dispatch_scatter }
//   -> k_node_msgs (thread per node) / k_node_tasks (warp per node) -> pair scan B -> k_emit (seed / latency / arrival)
//   -> { multisplit (count, column scan, stable scatter into the time ring) | k_free } -> k_end
// The two chains inside braces run as two branches (two streams, fork / join edges in the tick graph) for unsharded
// GSF and Handel engines in mode 1; otherwise, and in the profiled pass, one after the other in the order written.
// Unsharded GSF in mode 1 goes one step further inside a runMs window: C of the next millisecond runs beside this
// millisecond's emission (k_free -> k_cond_begin -> C | scan B -> k_emit -> multisplit), and the next pass starts at D.
// All sizes are read from the device control block, so a whole runMs window is enqueued without
// a host round trip.  See DESIGN.md §4 for why this reproduces the reference's sequential order, and for what each
// branch writes.
#include <cuda_runtime.h>
#include <unistd.h>

#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "wtg_engine.hpp"

namespace wtg {

#define CUDA_OK(x)                                                                                       \
  do {                                                                                                   \
    cudaError_t e_ = (x);                                                                                \
    if (e_ != cudaSuccess) throw std::runtime_error(std::string("CUDA: ") + cudaGetErrorString(e_) + " at " #x); \
  } while (0)

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 4;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

// condAhead: the pass's checkSigs has already run beside the previous pass's emission (k_begin), or the next pass's runs
// beside this one's (k_end)
__global__ void k_begin(Dev d, int mode, bool condAhead) {  // one warp
  if (threadIdx.x >= 32) return;
  if (d.ffwd && mode == 1) {
    CoopWarp c;
    tickBeginFfwd(d, c);
  } else if (d.farCap > 0 && !d.ffwd) {
    CoopWarp c;
    tickBeginFar(d, c, mode, condAhead);
  } else if (threadIdx.x == 0) {
    tickBegin(d, mode, condAhead);
  }
}
__global__ void k_end(Dev d, int mode, bool condAhead) {
  if (threadIdx.x == 0) tickEnd(d, mode, condAhead);
}
// clock and counters of the next pass's checkSigs, which runs ahead (one thread: a few hundred bytes)
__global__ void k_cond_begin(Dev d) {
  if (threadIdx.x == 0) condBegin(d);
}

// ---- conditional tasks (checkSigs): scan -> score -> select ---------------------------------------
// append node n to a striped list (stripe = global warp index & 63; a stripe receives at most listStripeCap nodes),
// with a 64-bit payload per entry when `words` is given
__device__ __forceinline__ void listAppend(const Dev& d, bool active, int n, int* cnt, int* list, u64* words = nullptr, u64 word = 0) {
  CoopWarp c;
  unsigned m = c.ballot(active);
  if (!m) return;
  int stripe = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) & (ARENA_STRIPES - 1);
  int base = 0;
  if (c.lane() == 0) base = atomicAdd(&cnt[stripe], c.count(m));
  base = c.bcast(base, 0);
  if (active) {
    size_t at = (size_t)stripe * d.listStripeCap + base + c.rank(m);
    list[at] = n;
    if (words) words[at] = word;
  }
}
// conditional-task bookkeeping, one thread per node -> list of due nodes
__global__ void __launch_bounds__(256) k_cond_mark(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x;
  int n = d.n0 + blk * blockDim.x + threadIdx.x;
  bool due = false;
  if (n < d.n0 + d.nLoc) due = d.proto == PROTO_HANDEL ? hCondMark(d, n) : gsfCondMark(d, n);
  listAppend(d, due, n, d.ctl->dueCnt, d.dueList);
}
// one warp per due node, blocks assigned to list stripes
template <int PHASE>
__global__ void __launch_bounds__(256) k_cond_nodes(Dev d) {
  extern __shared__ uint32_t keepAll[];
  __shared__ HScratch scratch[8];
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int stripe = blk & (ARENA_STRIPES - 1);
  const int cnt = d.ctl->dueCnt[stripe];
  const int warp = threadIdx.x >> 5;
  const int sub = (blk >> 6) * 8 + warp;
  const int nsub = (nBlk >> 6) * 8;
  const int* list = d.dueList + (size_t)stripe * d.listStripeCap;
  CoopWarp c;
  for (int t = sub; t < cnt; t += nsub) {
    int n = list[t];
    if (PHASE == 0) {
      if (d.proto == PROTO_HANDEL)
        hCondScanQueue(d, c, n);
      else
        gsfCondScanQueue(d, c, n);
    } else {
      if (d.proto == PROTO_HANDEL)
        hCondSelect(d, c, n, &scratch[warp]);
      else
        gsfCondSelect(d, c, n, keepAll + (size_t)warp * (size_t)(d.qcap / 32));
    }
  }
}
// blocks are assigned to arena stripes (blockIdx & 63), so an item is found without walking the 64 counters
__global__ void __launch_bounds__(256) k_cond_score(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int per = d.workCap / ARENA_STRIPES;
  const int stripe = blk & (ARENA_STRIPES - 1);
  int cnt = d.ctl->workCnt[stripe];
  if (cnt > per) cnt = per;
  const int warpsPerBlock = blockDim.x >> 5;
  const int sub = (blk >> 6) * warpsPerBlock + (threadIdx.x >> 5);
  const int nsub = (nBlk >> 6) * warpsPerBlock;
  CoopWarp c;
  const uint32_t* wl = d.workList + (size_t)stripe * per;
  for (int t = sub; t < cnt; t += nsub) {
    uint32_t it = wl[t];
    if (d.proto == PROTO_HANDEL)
      hScoreItem(d, c, it);
    else
      gsfScoreItem(d, c, it);
  }
}
// ---- Handel conditional pass (checkSigs): scan -> score -> select -> draw scan -> pick ---------------------
// does any nextInt(k) of this pass hit java.util.Random's rejection loop?  (probability ~ k / 2^31 per draw)
__global__ void k_hpick_check(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  for (int n = d.n0 + blk * blockDim.x + threadIdx.x; n < d.n0 + d.nLoc; n += nBlk * blockDim.x)
    if (d.hCandK[n] > 0 && (d.forcePickSerial || hCondPick(d, n, (u64)d.hDrawBase[n], false) > d.condDraws[n])) d.ctl->hReject = 1;
}
__global__ void k_hpick_apply(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  if (!d.ctl->hReject) {
    for (int n = d.n0 + blk * blockDim.x + threadIdx.x; n < d.n0 + d.nLoc; n += nBlk * blockDim.x) hCondPick(d, n, (u64)d.hDrawBase[n], true);
  } else if (blk == 0 && threadIdx.x == 0) {  // a rejection shifts every later draw: redo the picks in node order
    u64 idx = 0;
    for (int n = d.n0; n < d.n0 + d.nLoc; ++n) idx += (u64)hCondPick(d, n, idx, true);
  }
}
// node-sharded: the pick exchange (wtg_handel.cuh).  Publication: the k of every local pick into every shard's region; a
// shard in error still publishes its header (which carries the error)
__global__ void k_hpick_publish(Dev d) {
  const int blk = blockIdx.x, nBlk = gridDim.x;
  if (!d.ctl->error)
    for (int n = d.n0 + blk * blockDim.x + threadIdx.x; n < d.n0 + d.nLoc; n += nBlk * blockDim.x) hPickPublish(d, n);
  if (blk == 0 && threadIdx.x == 0) hPickPublishHeader(d);
}
// after the wait: replay every pick of the shards up to this one on its presumed position
__global__ void k_hpick_xcheck(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  if (blk == 0 && threadIdx.x == 0) hPickHeaders(d);
  const int upTo = hPicksBelow(d, d.rank + 1);
  for (int t = blk * blockDim.x + threadIdx.x; t < upTo; t += nBlk * blockDim.x)
    if (hPickRejects(d, t)) d.ctl->hReject = 1;
}
__global__ void k_hpick_xapply(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  if (!d.ctl->hReject) {
    const u64 below = (u64)hPicksBelow(d, d.rank);
    for (int n = d.n0 + blk * blockDim.x + threadIdx.x; n < d.n0 + d.nLoc; n += nBlk * blockDim.x) hCondPick(d, n, below + (u64)d.hDrawBase[n], true);
  } else if (blk == 0 && threadIdx.x == 0) {  // a rejection shifts every later draw, on this shard and above
    hPickSerial(d);
  }
}

// ---- dispatch -----------------------------------------------------------------------------
__global__ void k_dispatch_count(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int nEv = d.ctl->nEv;
  if (d.allCap > 0) {  // sendAll protocols: a warp per bucket entry
    CoopWarp c;
    int gw = (blk * blockDim.x + threadIdx.x) >> 5, nw = (nBlk * blockDim.x) >> 5;
    for (int i = gw; i < nEv; i += nw) dispatchCountCoop(d, c, i);
    return;
  }
  for (int i = blk * blockDim.x + threadIdx.x; i < nEv; i += nBlk * blockDim.x) dispatchCount(d, i);
}
__global__ void k_dispatch_scatter(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int nEv = d.ctl->nEv;
  if (d.allCap > 0) {
    CoopWarp c;
    int gw = (blk * blockDim.x + threadIdx.x) >> 5, nw = (nBlk * blockDim.x) >> 5;
    for (int i = gw; i < nEv; i += nw) dispatchScatterCoop(d, c, i);
    return;
  }
  for (int i = blk * blockDim.x + threadIdx.x; i < nEv; i += nBlk * blockDim.x) dispatchScatter(d, i);
}

// ---- handlers: warp per node ----------------------------------------------------------------
// pass 1: one thread per node.  GSF / PingPong: message deliveries (they commute with the node's tasks, see
// nodeProcess); SanFermin: everything (all handlers are scalar).  Leaves nodeTasks[n] = 1 when a warp is needed.
__global__ void __launch_bounds__(256) k_node_msgs(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x;
  int n = d.n0 + blk * blockDim.x + threadIdx.x;
  int flag = 0;
  u64 word = ~0ULL;
  if (n < d.n0 + d.nLoc && d.inboxFill[n] > 0) {
    CoopSerial cs;
    if (d.proto == PROTO_SANFERMIN || d.proto == PROTO_CAPPOS || d.proto == PROTO_SLUSH || d.proto == PROTO_SNOWFLAKE ||
        d.proto == PROTO_P2PFLOOD)
      nodeProcess(d, cs, n, 0);
    else if (d.proto == PROTO_GSF || d.proto == PROTO_PINGPONG) {
      u64 w = 0;
      int tasks = nodeProcess(d, cs, n, 1, &w);
      flag = tasks > 0 ? 1 : 0;
      if (tasks == 1) word = w;
    }
    else if (d.proto == PROTO_CASPER) {  // an inbox of attestations only is scalar work; blocks and tasks get a warp
      const u64* in = d.inbox + d.inboxOff[n];
      const Ev* bucket = d.buckets + (size_t)(d.ctl->tick & (d.ring - 1)) * (size_t)d.bcap;
      int cnt = d.inboxFill[n];
      bool simple = true;
      for (int r = 0; r < cnt && simple; ++r) {
        const Ev& ev = bucket[inboxEntry(in[r])];
        uint32_t meta = ev.kind == EV_MULTI ? d.rec[ev.aux].meta : ev.meta;
        simple = (ev.kind == EV_MSG || ev.kind == EV_MULTI) && meta == CM_ATT;
      }
      if (simple)
        nodeProcess(d, cs, n, 0);
      else
        flag = 1;
    } else
      flag = 1;
  }
  listAppend(d, flag != 0, n, d.ctl->taskCnt, d.taskList, d.taskWord, word);
}
// pass 2: one warp per node that has tasks (updateVerifiedSignatures / doCycle / ...), or, for protocols whose
// events do not commute (Handel), all of the node's events in reference order; blocks assigned to list stripes.
// Three blocks per SM = at most 80 registers per thread.  GSFSignature 65 536 nodes on an H100 80GB HBM3 (400 W), simulated-ms/s:
// 80 registers 4 643-4 667 over five runs, 64 (spills ~1 KB) 4 756 and 4 643 in two, 128 4 559 in one: no budget is clearly faster
__global__ void __launch_bounds__(256, 3) k_node_tasks(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const bool split = d.proto == PROTO_GSF || d.proto == PROTO_PINGPONG;
  const int stripe = blk & (ARENA_STRIPES - 1);
  const int cnt = d.ctl->taskCnt[stripe];
  const int sub = (blk >> 6) * 8 + (threadIdx.x >> 5);
  const int nsub = (nBlk >> 6) * 8;
  const int* list = d.taskList + (size_t)stripe * d.listStripeCap;
  const u64* words = d.taskWord + (size_t)stripe * d.listStripeCap;
  CoopWarp c;
  for (int t = sub; t < cnt; t += nsub) {
    const int n = list[t];
    const u64 w = words[t];
    if (split && w != ~0ULL)
      nodeSingleTask(d, c, n, w);
    else
      nodeProcess(d, c, n, split ? 2 : 0);
  }
}
// CasperIMD, after the parallel handler pass (one warp; both are rare): nodes that hit a fork-choice tie run in processing
// order with their exact draw index (randomOnTies), and several blocks created in one millisecond get their ids in
// processing order
__global__ void k_casper_fixups(Dev d) {
  const int blk = blockIdx.x;
  if (d.ctl->error || blk != 0 || threadIdx.x >= 32) return;
  CoopWarp c;
  if (d.cRandomTies && d.ctl->tieCnt > 0) casperResolveTies(d, c);
  if (d.G == 1 && d.cg->createdThisTick > 1) casperRenumber(d, c);
}
// ---- pair scans ---------------------------------------------------------------------------
__device__ __forceinline__ Pair pairAdd(Pair x, Pair y) {
  Pair r;
  r.a = x.a + y.a;
  r.b = x.b + y.b;
  return r;
}
// exclusive scan of one value per thread across the block; returns the block total in `total`
__device__ __forceinline__ Pair blockExclusive(Pair v, Pair& total) {
  __shared__ Pair warpSums[33];
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  Pair inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    int ta = __shfl_up_sync(0xffffffffu, inc.a, o), tb = __shfl_up_sync(0xffffffffu, inc.b, o);
    if (lane >= o) {
      inc.a += ta;
      inc.b += tb;
    }
  }
  __syncthreads();  // warpSums may still be read by a previous call
  if (lane == 31) warpSums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    Pair w;
    w.a = lane < nw ? warpSums[lane].a : 0;
    w.b = lane < nw ? warpSums[lane].b : 0;
    Pair wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int ta = __shfl_up_sync(0xffffffffu, wi.a, o), tb = __shfl_up_sync(0xffffffffu, wi.b, o);
      if (lane >= o) {
        wi.a += ta;
        wi.b += tb;
      }
    }
    Pair ex;
    ex.a = wi.a - w.a;
    ex.b = wi.b - w.b;
    warpSums[lane] = ex;
    if (lane == 31) warpSums[32] = wi;
  }
  __syncthreads();
  total = warpSums[32];
  Pair base = warpSums[warp];
  Pair r;
  r.a = base.a + inc.a - v.a;
  r.b = base.b + inc.b - v.b;
  return r;
}

__global__ void __launch_bounds__(SCAN_THREADS) k_scan_partial(Dev d, int which) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int M = scanCount(d, which);
  int nTiles = (M + SCAN_TILE - 1) / SCAN_TILE;
  for (int tile = blk; tile < nTiles; tile += nBlk) {
    int j0 = tile * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    Pair s;
    s.a = 0;
    s.b = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k)
      if (j0 + k < M) s = pairAdd(s, scanLoad(d, which, j0 + k));
    Pair total;
    blockExclusive(s, total);
    if (threadIdx.x == 0) {
      d.scanPartial[2 * tile] = total.a;
      d.scanPartial[2 * tile + 1] = total.b;
    }
    __syncthreads();
  }
}
// second (last) scan kernel: every block first sums the partials of the tiles before its own (a few hundred
// pairs at most), then scans its tile; the block of the last tile also publishes the totals.
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_final(Dev d, int which) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int M = scanCount(d, which);
  int nTiles = (M + SCAN_TILE - 1) / SCAN_TILE;
  if (nTiles == 0 && blk == 0 && threadIdx.x == 0) {
    Pair z;
    z.a = 0;
    z.b = 0;
    scanTotals(d, which, z);
  }
  for (int tile = blk; tile < nTiles; tile += nBlk) {
    Pair pre;
    pre.a = 0;
    pre.b = 0;
    for (int t = threadIdx.x; t < tile; t += SCAN_THREADS) {
      pre.a += d.scanPartial[2 * t];
      pre.b += d.scanPartial[2 * t + 1];
    }
    Pair tileBase;
    blockExclusive(pre, tileBase);  // tileBase = sum over all threads
    int j0 = tile * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    Pair v[SCAN_ITEMS];
    Pair s;
    s.a = 0;
    s.b = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
      if (j0 + k < M)
        v[k] = scanLoad(d, which, j0 + k);
      else {
        v[k].a = 0;
        v[k].b = 0;
      }
      s = pairAdd(s, v[k]);
    }
    Pair total;
    Pair ex = blockExclusive(s, total);
    ex = pairAdd(ex, tileBase);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; ++k) {
      if (j0 + k < M) scanStore(d, which, j0 + k, ex);
      ex = pairAdd(ex, v[k]);
    }
    if (tile == nTiles - 1 && threadIdx.x == 0) scanTotals(d, which, pairAdd(tileBase, total));
    __syncthreads();
  }
}

// ---- shuffled multi-sends: optimistic draw indices, checked; re-derived serially when a rejection shifted them ----
__global__ void k_shuffle_check(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int per = d.descCap / ARENA_STRIPES;
  const int stripe = blk & (ARENA_STRIPES - 1);
  int cnt = d.ctl->descCnt[stripe];
  if (cnt > per) cnt = per;
  const int sub = (blk >> 6) * blockDim.x + threadIdx.x;
  const int nsub = (nBlk >> 6) * blockDim.x;
  for (int j = sub; j < cnt; j += nsub) shuffleCheck(d, stripe * per + j);
}
__global__ void k_shuffle_serial(Dev d) {
  if (d.ctl->error) return;
  shuffleSerial(d);
}

// ---- node-sharded runs: the two exchanges of a pass (wtg_shard.cuh) --------------------------------------------
// exchange 1, publication: every item of this shard (key, prefix of slots / draws) into every shard's copy of this shard's
// list — peer stores over NVLink; a shard in error still publishes its header (which carries the error) so that the
// others stop at once
__global__ void __launch_bounds__(256) k_x1_publish(Dev d) {
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int n = d.ctl->error ? -1 : d.ctl->nItems;
  for (int i = blk * blockDim.x + threadIdx.x; i <= n; i += nBlk * blockDim.x) xPublishItem(d, i);
  if (blk == 0 && threadIdx.x == 0) xPublishHeader(d);
}
// signal the end of this shard's publication of `phase` to every shard, then wait for all of theirs (one block:
// spinning must not occupy the machine — shards may share a GPU in the tests)
__global__ void k_x_sync(Dev d, int phase) {
  if (threadIdx.x == 0) xSignal(d, phase);  // stream order: the publishing kernel has completed
  __syncthreads();
  if (threadIdx.x < d.G && threadIdx.x != d.rank) xWaitOne(d, phase, threadIdx.x);
}
// exchange 1, evaluation: global totals, and for every local item that created something the creation indices / draws
// of the other shards that come first
__global__ void __launch_bounds__(256) k_x1_offsets(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int n = d.ctl->nItems;
  for (int i = blk * blockDim.x + threadIdx.x; i < n; i += nBlk * blockDim.x) xOffsets(d, i);
}
__global__ void k_x1_totals(Dev d) {
  if (d.ctl->error) return;
  xTotals(d);
}
// exchange 2, after the wait: pooled payloads that arrived in the staging area move into pool slabs (warp per envelope)
__global__ void __launch_bounds__(256) k_x2_ingest(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int G = d.ctl->totalSlots;
  CoopWarp c;
  const int gw = (blk * blockDim.x + threadIdx.x) >> 5, nw = (nBlk * blockDim.x) >> 5;
  for (int g0 = gw * 32; g0 < G; g0 += nw * 32) {
    int g = g0 + c.lane();
    unsigned m = c.ballot(g < G && xNeedsIngest(d, g));
    while (m) {
      int src = c.first(m);
      m &= m - 1;
      xIngest(d, c, g0 + src);
    }
  }
}

// ---- emit ------------------------------------------------------------------------------------
__global__ void k_emit(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  // conditional-task inserts (one per node) ...
  for (int i = blk * blockDim.x + threadIdx.x; i < d.nLoc; i += nBlk * blockDim.x) emitCond(d, d.n0 + i);
  // ... then the handlers' descriptors, blocks assigned to arena stripes
  const int per = d.descCap / ARENA_STRIPES;
  const int stripe = blk & (ARENA_STRIPES - 1);
  int cnt = d.ctl->descCnt[stripe];
  if (cnt > per) cnt = per;
  const int sub = (blk >> 6) * blockDim.x + threadIdx.x;
  const int nsub = (nBlk >> 6) * blockDim.x;
  for (int j = sub; j < cnt; j += nsub) emitDesc(d, stripe * per + j);
}

// sendAll descriptors: one warp each (arrival per destination, stable counting sort by arrival)
__global__ void __launch_bounds__(128) k_emit_all(Dev d) {
  __shared__ int hist[4][ALL_HIST];
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int cnt = d.ctl->allCnt;
  if (cnt > d.allCap) cnt = d.allCap;
  const int warp = threadIdx.x >> 5;
  if (warp >= 4) return;  // four histograms per block
  const int gw = blk * 4 + warp, nw = nBlk * 4;
  CoopWarp c;
  for (int j = gw; j < cnt; j += nw) emitAll(d, c, d.allList[j], d.allTmp + (size_t)gw * d.N, hist[warp]);
}
// P2PFlood forwards (DESC_PEERS descriptors): one warp each — the peer list and its shuffle in shared memory, arrivals, the
// stably ranked record (wtg_p2p.cuh)
__global__ void __launch_bounds__(128) k_emit_peers(Dev d) {
  __shared__ uint32_t list[4][PEERS_MAX];
  __shared__ int arr[4][PEERS_MAX];
  if (d.ctl->error) return;
  const int warp = threadIdx.x >> 5;
  const int gw = blockIdx.x * 4 + warp, nw = gridDim.x * 4;
  int cnt = d.ctl->peerCnt;
  if (cnt > d.descCap) cnt = d.descCap;
  CoopWarp c;
  for (int j = gw; j < cnt; j += nw) emitPeers(d, c, d.peerList[j], list[warp], arr[warp]);
}
// node-sharded sendAll (CasperIMD): the descriptors are published to every shard before the envelope exchange ...
__global__ void __launch_bounds__(128) k_x_all_publish(Dev d) {
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int cnt = d.ctl->error ? 0 : d.ctl->allCnt;
  if (cnt > d.xAllCap) cnt = 0;  // xPublishAllCount reports the overflow
  for (int j = blk * blockDim.x + threadIdx.x; j < cnt; j += nBlk * blockDim.x) xPublishAll(d, j);
  if (blk == 0 && threadIdx.x == 0) xPublishAllCount(d);
}
// ... and after it every shard builds every sendAll of the pass: the same sorted record in the same slot (replicated records)
__global__ void __launch_bounds__(128) k_x_all_build(Dev d) {
  __shared__ int hist[4][ALL_HIST];
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int cnt = xAllTotal(d);
  const int warp = threadIdx.x >> 5;
  if (warp >= 4) return;
  const int gw = blk * 4 + warp, nw = nBlk * 4;
  CoopWarp c;
  for (int k = gw; k < cnt; k += nw) xBuildAll(d, c, k, d.allTmp + (size_t)gw * d.N, hist[warp]);
}

// ---- multisplit: stable distribution of the new envelopes into the time ring -----------------
// A block of Dev.msWarps warps handles a chunk of msWarps * MS_SUB consecutive envelopes (creation order); warp w owns the w-th
// sub-chunk of MS_SUB envelopes.  count: per-warp histograms over the ring bins in shared memory -> one row of totals per
// chunk.  scan: running offset per bin over the chunks.  scatter: the histograms again, turned into each warp's first
// position per bin (chunk offset + the lower warps' counts); then MS_SUB / 32 rounds of match-any ranked placement per warp.
constexpr int MS_SUB = 256;  // envelopes per warp
constexpr int MS_ROUNDS = MS_SUB / 32;
// warps per block = Dev.msWarps (8 unless the ring is so long that 8 histograms do not fit in shared memory); chunk = msWarps * MS_SUB
__device__ __forceinline__ void msZero(int* hist, int ring, int warps) {
  for (int i = threadIdx.x * 4; i < warps * ring; i += blockDim.x * 4) *reinterpret_cast<int4*>(hist + i) = make_int4(0, 0, 0, 0);
}
// this warp's targets of the chunk (kept in registers) and their histogram
__device__ __forceinline__ void msWarpHistogram(const Dev& d, int* hw, int g0, int G, int tick, int lane, int (&tg)[MS_ROUNDS]) {
#pragma unroll
  for (int r = 0; r < MS_ROUNDS; ++r) {  // all targets are in flight before the first one is used
    int g = g0 + r * 32 + lane;
    tg[r] = g < G ? d.newTarget[g] : -1;
  }
#pragma unroll
  for (int r = 0; r < MS_ROUNDS; ++r)
    if (tg[r] >= 0) atomicAdd(&hw[tg[r] - tick], 1);
}
__global__ void __launch_bounds__(256) k_ms_count(Dev d) {
  extern __shared__ int msHist[];  // [msWarps][ring]
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int G = d.ctl->totalSlots, tick = d.ctl->tick, ring = d.ring;
  const int W = d.msWarps, CH = W * MS_SUB;
  const int nChunks = (G + CH - 1) / CH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int ch = blk; ch < nChunks; ch += nBlk) {
    msZero(msHist, ring, W);
    __syncthreads();
    int tg[MS_ROUNDS];
    msWarpHistogram(d, msHist + warp * ring, ch * CH + warp * MS_SUB, G, tick, lane, tg);
    __syncthreads();
    int* row = d.msCount + (size_t)ch * ring;
    for (int b = threadIdx.x; b < ring; b += blockDim.x) {
      int tot = 0;
      for (int w = 0; w < W; ++w) tot += msHist[w * ring + b];
      row[b] = tot;
    }
    __syncthreads();
  }
}
// per ring bin: running offset over chunks, starting at the bucket's current fill
__global__ void k_ms_scan(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  int G = d.ctl->totalSlots, tick = d.ctl->tick, ring = d.ring;
  const int CH = d.msWarps * MS_SUB;
  int nChunks = (G + CH - 1) / CH;
  if (nChunks == 0) return;
  for (int b = blk * blockDim.x + threadIdx.x; b < ring; b += nBlk * blockDim.x) {
    int slot = (tick + b) & (ring - 1);
    int run = d.bucketCount[slot];
    for (int ch0 = 0; ch0 < nChunks; ch0 += 8) {
      int v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = ch0 + k < nChunks ? d.msCount[(size_t)(ch0 + k) * ring + b] : 0;
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (ch0 + k < nChunks) {
          d.msCount[(size_t)(ch0 + k) * ring + b] = run;
          run += v[k];
        }
    }
    if (run > d.bcap) {
      setError(d, ERR_BUCKET_OVERFLOW, tick + b);
      run = d.bcap;
    }
    d.bucketCount[slot] = run;
  }
}
__global__ void __launch_bounds__(256) k_ms_scatter(Dev d) {
  extern __shared__ int msHist[];
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int G = d.ctl->totalSlots, tick = d.ctl->tick, ring = d.ring;
  const int W = d.msWarps, CH = W * MS_SUB;
  const int nChunks = (G + CH - 1) / CH;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int* base = msHist + warp * ring;
  CoopWarp cw;
  for (int ch = blk; ch < nChunks; ch += nBlk) {
    msZero(msHist, ring, W);
    __syncthreads();
    const int g0 = ch * CH + warp * MS_SUB;
    int tg[MS_ROUNDS];
    msWarpHistogram(d, base, g0, G, tick, lane, tg);
    __syncthreads();
    const int* row = d.msCount + (size_t)ch * ring;  // first position of this chunk in every bin (after the scan)
    for (int b = threadIdx.x; b < ring; b += blockDim.x) {
      int run = row[b];
      for (int w = 0; w < W; ++w) {
        int c = msHist[w * ring + b];
        msHist[w * ring + b] = run;
        run += c;
      }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < MS_ROUNDS; ++r) {
      int g = g0 + r * 32 + lane;
      int t = tg[r];
      int pos = cw.claim(base, t - tick, t >= 0);
      if (t >= 0) {
        if (pos < d.bcap) {
          const int4* src = reinterpret_cast<const int4*>(d.newEv + g);
          int4* dst = reinterpret_cast<int4*>(d.buckets + (size_t)(t & (ring - 1)) * (size_t)d.bcap + pos);
          int4 x = src[0], y = src[1];
          dst[0] = x;
          dst[1] = y;
          if (d.G > 1) d.bucketKey[(size_t)(t & (ring - 1)) * (size_t)d.bcap + pos] = orderKey((unsigned)d.ctl->xseq, (unsigned)g);
        }
        if (d.G > 1) d.newTarget[g] = -1;  // the array is indexed by the global creation index: clean for the next pass
      }
      __syncwarp();
    }
    __syncthreads();
  }
}

__global__ void k_free(Dev d) {
  if (d.ctl->error) return;
  const int blk = blockIdx.x, nBlk = gridDim.x;
  const int per = d.freeCap / ARENA_STRIPES;
  const int stripe = blk & (ARENA_STRIPES - 1);
  int cnt = d.ctl->freeCnt[stripe];
  if (cnt > per) cnt = per;
  const int sub = (blk >> 6) * blockDim.x + threadIdx.x;
  const int nsub = (nBlk >> 6) * blockDim.x;
  for (int j = sub; j < cnt; j += nsub) freeApply(d, stripe * per + j);
}

// ---- init kernels ---------------------------------------------------------------------------
__global__ void k_gsf_init_nodes(Dev d) {
  int n = d.n0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (n < d.n0 + d.nLoc) gsfInitNodeBody(d, n);
}
__global__ void k_rng_candidates(Dev d, u64 s0, u64 count, u64 chunk, int maxBound, u64* out, int* outCount, int cap) {
  u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  u64 start = t * chunk;
  if (start >= count) return;
  u64 len = start + chunk <= count ? chunk : count - start;
  rngCandidateChunk(d, s0, start, len, maxBound, out, outCount, cap);
}
template <class PeerT>
__global__ void k_gsf_shuffle(Dev d, int l, u64 s0, const int* liveRank, const u64* rejOrd, int nRej) {
  int n = d.n0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (n < d.n0 + d.nLoc) gsfShuffleLevel<PeerT>(d, n, l, s0, liveRank, rejOrd, nRej);
}

// ------------------------------------------------------------------------------------------------
class CudaBackend : public Backend {
 public:
  cudaStream_t st = nullptr;
  cudaStream_t side = nullptr;  // second branch of a pass (enqueueTick); joined back into st before the pass goes on
  cudaEvent_t forkEv = nullptr, joinEv = nullptr;
  int devId = 0;  // every entry point binds it: callers may drive different networks from different host threads
  void bind() const { cudaSetDevice(devId); }
  int sms = 132;
  int smemOptin = 0;
  // one graph per pass shape (SHAPE_*): whether the pass runs its own checkSigs, and whether it runs the next pass's
  enum { SHAPE_PLAIN, SHAPE_FIRST, SHAPE_LAST, SHAPE_MIDDLE, NSHAPES };
  cudaGraphExec_t tickGraph[NSHAPES] = {};
  long long shapeKernels[NSHAPES] = {};
  const void* graphFor = nullptr;
  bool useGraph = true;
  long long launches = 0;      // kernels enqueued (graph replays counted kernel by kernel)
  cudaEvent_t tm0 = nullptr, tm1 = nullptr;
  // per-kernel profiling: one slot per timed group of kernels, reported under profNames[slot]
  // The dispatch's scan A has slots of its own; unless the caller asked for them apart (profileEnable(true, true)),
  // profileRead adds them into scan B's k_scan_partial / k_scan_final.
  enum ProfSlot { P_BEGIN, P_COND_SCAN, P_DISPATCH_COUNT, P_SCAN_PARTIAL, P_EXCHANGE, P_SCAN_FINAL, P_DISPATCH_SCATTER, P_NODE,
                  P_EMIT, P_MS_COUNT, P_MS_SCAN, P_MS_SCATTER, P_FREE, P_END, P_COND_SCORE, P_COND_SELECT, P_EMIT_PEERS,
                  P_SCAN_A_PARTIAL, P_SCAN_A_FINAL, NK };
  bool profiling = false;
  bool profSplitScans = false;
  std::vector<cudaEvent_t> evPool;
  std::vector<int> evKernel;  // kernel id of each event pair
  size_t evUsed = 0;
  double profMs[NK] = {};
  long long profCnt[NK] = {};
  const char* profNames[NK] = {"k_begin", "k_cond_scan", "k_dispatch_count", "k_scan_partial", "k_exchange", "k_scan_final",
                               "k_dispatch_scatter", "k_node", "k_emit", "k_ms_count", "k_ms_scan", "k_ms_scatter", "k_free",
                               "k_end", "k_cond_score", "k_cond_select", "k_emit_peers", "k_scan_a_partial", "k_scan_a_final"};

  explicit CudaBackend(int requested = -1) {
    int dev = 0;
    const char* e = std::getenv("LOCAL_RANK");
    int cnt = 0;
    CUDA_OK(cudaGetDeviceCount(&cnt));
    if (cnt == 0) throw std::runtime_error("no CUDA device");
    if (e) dev = std::atoi(e) % cnt;
    const char* e2 = std::getenv("WTG_DEVICE");
    if (e2) dev = std::atoi(e2) % cnt;
    if (requested >= 0) {  // wtg_create_on: the caller places this network itself
      if (requested >= cnt) throw std::invalid_argument("CUDA device " + std::to_string(requested) + " does not exist");
      dev = requested;
    }
    CUDA_OK(cudaSetDevice(dev));
    devId = dev;
    cudaDeviceProp p;
    CUDA_OK(cudaGetDeviceProperties(&p, dev));
    sms = p.multiProcessorCount;
    CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamCreateWithFlags(&side, cudaStreamNonBlocking));
    CUDA_OK(cudaEventCreateWithFlags(&forkEv, cudaEventDisableTiming));
    CUDA_OK(cudaEventCreateWithFlags(&joinEv, cudaEventDisableTiming));
    CUDA_OK(cudaDeviceGetAttribute(&smemOptin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    CUDA_OK(cudaFuncSetAttribute(k_ms_count, cudaFuncAttributeMaxDynamicSharedMemorySize, smemOptin));
    CUDA_OK(cudaFuncSetAttribute(k_ms_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize, smemOptin));
    const char* g = std::getenv("WTG_NO_GRAPH");
    if (g && g[0] == '1') useGraph = false;
  }
  ~CudaBackend() override {
    for (void* q : ipcOpened) cudaIpcCloseMemHandle(q);
    for (cudaGraphExec_t g : tickGraph)
      if (g) cudaGraphExecDestroy(g);
    if (forkEv) cudaEventDestroy(forkEv);
    if (joinEv) cudaEventDestroy(joinEv);
    if (side) cudaStreamDestroy(side);
    if (st) cudaStreamDestroy(st);
  }
  void* alloc(size_t bytes) override {
    bind();
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) throw std::runtime_error("cudaMalloc of " + std::to_string(bytes) + " bytes failed: " + cudaGetErrorString(e));
    CUDA_OK(cudaMemsetAsync(p, 0, bytes, st));
    return p;
  }
  void release(void* p) override { cudaFree(p); }
  int deviceId() const override { return devId; }
  // exchange region of a shard: plain cudaMalloc memory (CUDA IPC cannot export pool allocations)
  void exportShared(void* p, unsigned char* handle) override {
    bind();
    std::memset(handle, 0, 128);
    cudaIpcMemHandle_t ih;
    CUDA_OK(cudaIpcGetMemHandle(&ih, p));
    static_assert(sizeof(ih) == 64, "cudaIpcMemHandle_t");
    std::memcpy(handle, &ih, 64);
    long long pid = (long long)getpid();
    std::memcpy(handle + 64, &pid, 8);
    std::memcpy(handle + 72, &p, sizeof(p));
    std::memcpy(handle + 80, &devId, 4);
  }
  std::vector<void*> ipcOpened;
  void* importShared(const unsigned char* handle) override {
    bind();
    long long pid;
    void* p;
    int dev;
    std::memcpy(&pid, handle + 64, 8);
    std::memcpy(&p, handle + 72, sizeof(p));
    std::memcpy(&dev, handle + 80, 4);
    if (pid == (long long)getpid()) {  // a shard of this process: same address space
      if (dev != devId) {
        int can = 0;
        CUDA_OK(cudaDeviceCanAccessPeer(&can, devId, dev));
        if (!can) throw std::runtime_error("GPU " + std::to_string(devId) + " cannot access GPU " + std::to_string(dev) + " (peer access)");
        cudaError_t e = cudaDeviceEnablePeerAccess(dev, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CUDA_OK(e);
        cudaGetLastError();
      }
      return p;
    }
    cudaIpcMemHandle_t ih;
    std::memcpy(&ih, handle, 64);
    void* q = nullptr;
    CUDA_OK(cudaIpcOpenMemHandle(&q, ih, cudaIpcMemLazyEnablePeerAccess));
    ipcOpened.push_back(q);
    return q;
  }
  void upload(void* dst, const void* src, size_t bytes) override {
    bind();
    CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaStreamSynchronize(st));
  }
  void download(void* dst, const void* src, size_t bytes) override {
    bind();
    CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
  }
  void sync() override {
    bind();
    CUDA_OK(cudaStreamSynchronize(st));
    drainProfile();
  }
  void timerStart() override {
    bind();
    if (!tm0) {
      CUDA_OK(cudaEventCreate(&tm0));
      CUDA_OK(cudaEventCreate(&tm1));
    }
    CUDA_OK(cudaEventRecord(tm0, st));
  }
  double timerStopMs() override {
    bind();
    CUDA_OK(cudaEventRecord(tm1, st));
    CUDA_OK(cudaEventSynchronize(tm1));
    float ms = 0;
    CUDA_OK(cudaEventElapsedTime(&ms, tm0, tm1));
    return (double)ms;
  }
  void profileEnable(bool on, bool splitScans) override {
    sync();
    profiling = on;
    profSplitScans = splitScans;
    if (on) {
      for (int i = 0; i < NK; ++i) {
        profMs[i] = 0;
        profCnt[i] = 0;
      }
    }
  }
  int profileRead(double* ms, long long* cnt, const char** names, int cap) override {
    sync();
    const int shown = profSplitScans ? NK : P_SCAN_A_PARTIAL;
    int k = 0;
    for (int i = 0; i < shown && k < cap; ++i, ++k) {
      ms[k] = profMs[i];
      cnt[k] = profCnt[i];
      names[k] = profNames[i];
      const int a = i == P_SCAN_PARTIAL ? P_SCAN_A_PARTIAL : i == P_SCAN_FINAL ? P_SCAN_A_FINAL : -1;
      if (!profSplitScans && a >= 0) {
        ms[k] += profMs[a];
        cnt[k] += profCnt[a];
      }
    }
    return k;
  }
  void drainProfile() {
    for (size_t i = 0; i < evUsed; ++i) {
      float ms = 0;
      cudaEventElapsedTime(&ms, evPool[2 * i], evPool[2 * i + 1]);
      profMs[evKernel[i]] += ms;
      profCnt[evKernel[i]] += 1;
    }
    evUsed = 0;
  }
  void profBegin(int kid) {
    if (!profiling) return;
    if (evUsed * 2 + 2 > evPool.size()) {
      if (evUsed >= 8192) {  // bound the pool: drain what has completed so far
        CUDA_OK(cudaStreamSynchronize(st));
        drainProfile();
      } else {
        cudaEvent_t a, b;
        CUDA_OK(cudaEventCreate(&a));
        CUDA_OK(cudaEventCreate(&b));
        evPool.push_back(a);
        evPool.push_back(b);
        evKernel.push_back(0);
      }
    }
    evKernel[evUsed] = kid;
    CUDA_OK(cudaEventRecord(evPool[2 * evUsed], st));
  }
  void profEnd() {
    if (!profiling) return;
    CUDA_OK(cudaEventRecord(evPool[2 * evUsed + 1], st));
    ++evUsed;
  }

  // `side` starts at st's current position
  void fork() {
    CUDA_OK(cudaEventRecord(forkEv, st));
    CUDA_OK(cudaStreamWaitEvent(side, forkEv, 0));
  }
  // st waits for everything queued on `side` so far
  void join() {
    CUDA_OK(cudaEventRecord(joinEv, side));
    CUDA_OK(cudaStreamWaitEvent(st, joinEv, 0));
  }
  // checkSigs (C) on stream s: scan, score, select; Handel: draw scan and pick
  void enqueueCond(const Dev& d, cudaStream_t s) {
    const int wide = sms * 8;
    // GSF's select keeps one bit per queue entry per warp in dynamic shared memory; Handel's scratch is static
    const size_t smem8 = d.proto == PROTO_GSF ? (size_t)8 * (size_t)(d.qcap / 32) * sizeof(uint32_t) : 0;
    profBegin(P_COND_SCAN);
    k_cond_mark<<<(d.nLoc + 255) / 256, 256, 0, s>>>(d);
    k_cond_nodes<0><<<ARENA_STRIPES * 19, 256, 0, s>>>(d);
    profEnd();
    profBegin(P_COND_SCORE);
    k_cond_score<<<ARENA_STRIPES * 19, 256, 0, s>>>(d);
    profEnd();
    profBegin(P_COND_SELECT);
    k_cond_nodes<1><<<ARENA_STRIPES * 19, 256, smem8, s>>>(d);
    profEnd();
    launches += 4;
    if (d.proto == PROTO_HANDEL) {  // draw scan and pick
      // the draw scan's tile partials go to their own buffer: scan A may be running on `side` at the same time
      Dev dd = d;
      dd.scanPartial = d.drawScanPartial;
      profBegin(P_SCAN_PARTIAL);
      k_scan_partial<<<wide, SCAN_THREADS, 0, s>>>(dd, 2);
      profEnd();
      profBegin(P_SCAN_FINAL);
      k_scan_final<<<wide, SCAN_THREADS, 0, s>>>(dd, 2);
      profEnd();
      if (d.G > 1) {  // node-sharded: the pick exchange puts the picks of the lower shards first
        profBegin(P_EXCHANGE);
        k_hpick_publish<<<sms, 256, 0, s>>>(d);
        k_x_sync<<<1, 32, 0, s>>>(d, 3);
        profEnd();
        profBegin(P_COND_SELECT);
        k_hpick_xcheck<<<sms, 256, 0, s>>>(d);
        k_hpick_xapply<<<sms, 256, 0, s>>>(d);
        profEnd();
        launches += 5;
      } else {
        profBegin(P_COND_SELECT);
        k_hpick_check<<<sms, 256, 0, s>>>(d);
        k_hpick_apply<<<sms, 256, 0, s>>>(d);
        profEnd();
        launches += 3;
      }
    }
  }
  // ownCond: the pass runs its own checkSigs (false: the previous pass ran it ahead).  nextCond: this pass runs the next
  // pass's checkSigs beside its emission.  Both differ from true / false only for unsharded GSF in mode 1, unprofiled.
  void enqueueTick(const Dev& d, int mode, bool ownCond = true, bool nextCond = false) {
    const int wide = sms * 8;
    const size_t msSmem = (size_t)d.msWarps * d.ring * sizeof(int);
    // Two branches per pass for the protocols with a conditional pass, in mode 1: the delivery dispatch (count, scan A,
    // scatter) runs on `side` beside checkSigs, and k_free beside the multisplit.  Neither branch reads or writes what
    // the other writes (DESIGN.md §4).  The profiled pass keeps the serial order on st, so that every kernel's
    // event time is its own.  Under stream capture the fork and join become edges of the tick graph.
    // Node-sharded engines keep one stream: their exchange kernels spin until every shard has signalled, and shards that
    // share a GPU need a hardware queue each, or a spinning kernel can hold up another shard's publication behind it.
    const bool branches = mode == 1 && !profiling && d.G == 1 && (d.proto == PROTO_GSF || d.proto == PROTO_HANDEL);
    // A pass whose checkSigs ran ahead has only the dispatch left before the handlers: it stays on st.  One that runs the
    // next pass's checkSigs forks after the handlers: k_free, k_cond_begin and C on `side`, the emission on st.
    const bool condBranch = branches && ownCond;
    cudaStream_t sd = condBranch ? side : st;
    // mode 3: the host prepared the control block and the descriptors of sends it injects at the current time
    // (Engine::inject); only the emission half of the pipeline runs
    if (mode != 3) {
      profBegin(P_BEGIN);
      k_begin<<<1, 32, 0, st>>>(d, mode, !ownCond);
      profEnd();
    }
    if (condBranch) fork();
    if ((d.proto == PROTO_GSF || d.proto == PROTO_HANDEL) && mode != 3 && ownCond) enqueueCond(d, st);  // conditional tasks
    if (mode != 2 && mode != 3) {  // dispatch and handlers
      profBegin(P_DISPATCH_COUNT);
      k_dispatch_count<<<wide, 256, 0, sd>>>(d);
      profEnd();
      profBegin(P_SCAN_A_PARTIAL);
      k_scan_partial<<<wide, SCAN_THREADS, 0, sd>>>(d, 0);
      profEnd();
      profBegin(P_SCAN_A_FINAL);
      k_scan_final<<<wide, SCAN_THREADS, 0, sd>>>(d, 0);
      profEnd();
      profBegin(P_DISPATCH_SCATTER);
      k_dispatch_scatter<<<wide, 256, 0, sd>>>(d);
      profEnd();
      if (condBranch) join();  // k_node_msgs appends deliveries to the queues checkSigs has just compacted
      profBegin(P_NODE);
      k_node_msgs<<<(d.nLoc + 255) / 256, 256, 0, st>>>(d);
      k_node_tasks<<<ARENA_STRIPES * 19, 256, 0, st>>>(d);
      if (d.proto == PROTO_CASPER) {
        k_casper_fixups<<<1, 32, 0, st>>>(d);
        launches += 1;
      }
      profEnd();
      launches += 6;
    }
    const bool pooled = d.proto == PROTO_GSF || d.proto == PROTO_HANDEL;  // only these protocols hold pooled payloads
    if (nextCond) {  // every pool allocation and deferred free of the pass is behind us
      fork();
      k_free<<<ARENA_STRIPES * 2, 256, 0, side>>>(d);
      k_cond_begin<<<1, 1, 0, side>>>(d);
      enqueueCond(d, side);
      launches += 2;
    }
    profBegin(P_SCAN_PARTIAL);
    k_scan_partial<<<wide, SCAN_THREADS, 0, st>>>(d, 1);
    profEnd();
    profBegin(P_SCAN_FINAL);
    k_scan_final<<<wide, SCAN_THREADS, 0, st>>>(d, 1);
    profEnd();
    if (d.G > 1) {  // node-sharded: exchange 1 (items -> creation / draw offsets over all shards)
      profBegin(P_EXCHANGE);
      k_x1_publish<<<sms * 2, 256, 0, st>>>(d);
      k_x_sync<<<1, 32, 0, st>>>(d, 0);
      k_x1_totals<<<1, 1, 0, st>>>(d);
      k_x1_offsets<<<sms * 2, 256, 0, st>>>(d);
      profEnd();
      launches += 4;
    }
    profBegin(P_EMIT);
    if (d.shufCap > 0) {
      k_shuffle_check<<<ARENA_STRIPES * 4, 256, 0, st>>>(d);
      k_shuffle_serial<<<1, 1, 0, st>>>(d);
      launches += 2;
    }
    k_emit<<<ARENA_STRIPES * 16, 256, 0, st>>>(d);
    if (d.allCap > 0) {
      if (d.G > 1)
        k_x_all_publish<<<8, 128, 0, st>>>(d);
      else
        k_emit_all<<<d.allWarps / 4, 128, 0, st>>>(d);
      launches += 1;
    }
    profEnd();
    if (d.proto == PROTO_P2PFLOOD) {
      profBegin(P_EMIT_PEERS);
      k_emit_peers<<<sms * 8, 128, 0, st>>>(d);
      profEnd();
      launches += 1;
    }
    if (d.G > 1) {  // exchange 2: the envelopes were stored into their destination shards' arrays by k_emit
      profBegin(P_EXCHANGE);
      k_x_sync<<<1, 32, 0, st>>>(d, 1);
      k_x2_ingest<<<sms * 4, 256, 0, st>>>(d);
      launches += 2;
      if (d.allCap > 0) {
        k_x_all_build<<<d.allWarps / 4, 128, 0, st>>>(d);
        launches += 1;
      }
      profEnd();
    }
    if (branches && !nextCond) fork();  // every pool allocation of the pass (handlers, HiddenByzantine's pick) is behind us
    profBegin(P_MS_COUNT);
    k_ms_count<<<sms * 2, d.msWarps * 32, msSmem, st>>>(d);
    profEnd();
    profBegin(P_MS_SCAN);
    k_ms_scan<<<(d.ring + 127) / 128, 128, 0, st>>>(d);
    profEnd();
    profBegin(P_MS_SCATTER);
    k_ms_scatter<<<sms * 2, d.msWarps * 32, msSmem, st>>>(d);
    profEnd();
    if (pooled && !nextCond) {
      profBegin(P_FREE);
      k_free<<<ARENA_STRIPES * 2, 256, 0, branches ? side : st>>>(d);
      profEnd();
    }
    if (branches) join();
    profBegin(P_END);
    k_end<<<1, 1, 0, st>>>(d, mode, nextCond);
    profEnd();
    launches += pooled && !nextCond ? 9 : 8;  // with nextCond, k_free was counted with k_cond_begin
  }
  // dynamic shared memory of the multisplit kernels: the attribute is per device and shared by every engine on it (several
  // engines may be driven from concurrent host threads), so it is set once, to the device's opt-in maximum
  void configure(const Dev& d) {
    const size_t msSmem = (size_t)d.msWarps * d.ring * sizeof(int);
    if (msSmem > (size_t)smemOptin) throw std::runtime_error("time ring too large for the multisplit's shared-memory histogram");
  }
  void tick(const Dev& d, int mode) override {
    bind();
    configure(d);
    enqueueTick(d, mode);
    CUDA_OK(cudaGetLastError());
  }
  // A window of `count` mode-1 passes.  Unsharded GSF (cond_ahead on) runs the first pass with its own checkSigs and the
  // next pass's, the middle ones with the next pass's only, the last with neither; a single pass keeps the plain shape.
  // No checkSigs runs ahead across a call: between windows the host may change what it reads (stop / start nodes,
  // partitions, injected sends), and the window's end-of-window pass (mode 2) runs its own.
  void ticks(const Dev& d, int count) override {
    bind();
    configure(d);
    const bool ahead = d.condAhead != 0 && d.proto == PROTO_GSF && d.G == 1 && !profiling && count > 1;
    auto shapeOf = [&](int i) { return !ahead ? SHAPE_PLAIN : i == 0 ? SHAPE_FIRST : i == count - 1 ? SHAPE_LAST : SHAPE_MIDDLE; };
    auto enqueueShape = [&](int shape) { enqueueTick(d, 1, shape == SHAPE_PLAIN || shape == SHAPE_FIRST, shape == SHAPE_FIRST || shape == SHAPE_MIDDLE); };
    if (!useGraph || profiling || count < 4) {
      for (int i = 0; i < count; ++i) enqueueShape(shapeOf(i));
      CUDA_OK(cudaGetLastError());
      return;
    }
    if (graphFor != (const void*)d.ctl) {
      for (cudaGraphExec_t& g : tickGraph)
        if (g) {
          cudaGraphExecDestroy(g);
          g = nullptr;
        }
      graphFor = (const void*)d.ctl;
    }
    for (int i = 0; i < count; ++i) {
      const int shape = shapeOf(i);
      if (!tickGraph[shape]) {
        cudaGraph_t g;
        long long before = launches;
        CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        enqueueShape(shape);
        CUDA_OK(cudaStreamEndCapture(st, &g));
        shapeKernels[shape] = launches - before;  // kernels per replay
        launches = before;
        CUDA_OK(cudaGraphInstantiate(&tickGraph[shape], g, 0));
        cudaGraphDestroy(g);
      }
      CUDA_OK(cudaGraphLaunch(tickGraph[shape], st));
      launches += shapeKernels[shape];
    }
  }
  void gsfInitNodes(const Dev& d) override {
    bind();
    k_gsf_init_nodes<<<(d.nLoc + 255) / 256, 256, 0, st>>>(d);
    CUDA_OK(cudaGetLastError());
  }
  void rngCandidates(const Dev& d, unsigned long long s0, unsigned long long count, int maxBound,
                     std::vector<unsigned long long>& out) override {
    bind();
    const u64 chunk = 16384;
    u64 threads = (count + chunk - 1) / chunk;
    int cap = (int)std::min<u64>((u64)1 << 26, count / 1024 + (1 << 16));
    u64* dOut = nullptr;
    int* dCnt = nullptr;
    CUDA_OK(cudaMalloc(&dOut, (size_t)cap * sizeof(u64)));
    CUDA_OK(cudaMalloc(&dCnt, sizeof(int)));
    CUDA_OK(cudaMemsetAsync(dCnt, 0, sizeof(int), st));
    u64 blocks = (threads + 127) / 128;
    k_rng_candidates<<<(unsigned)blocks, 128, 0, st>>>(d, s0, count, chunk, maxBound, dOut, dCnt, cap);
    CUDA_OK(cudaGetLastError());
    int n = 0;
    CUDA_OK(cudaMemcpyAsync(&n, dCnt, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    if (n > cap) {
      cudaFree(dOut);
      cudaFree(dCnt);
      throw std::runtime_error("rng candidate list overflow");
    }
    out.resize((size_t)n);
    if (n) CUDA_OK(cudaMemcpyAsync(out.data(), dOut, (size_t)n * sizeof(u64), cudaMemcpyDeviceToHost, st));
    CUDA_OK(cudaStreamSynchronize(st));
    cudaFree(dOut);
    cudaFree(dCnt);
  }
  void gsfShufflePeers(const Dev& d, unsigned long long s0, const int* liveRank, const unsigned long long* rejOrd, int nRej) override {
    bind();
    for (int l = d.L - 1; l >= 1; --l) {
      if (d.peerBits == 16)
        k_gsf_shuffle<uint16_t><<<(d.nLoc + 127) / 128, 128, 0, st>>>(d, l, s0, liveRank, rejOrd, nRej);
      else
        k_gsf_shuffle<uint32_t><<<(d.nLoc + 127) / 128, 128, 0, st>>>(d, l, s0, liveRank, rejOrd, nRej);
    }
    CUDA_OK(cudaGetLastError());
    CUDA_OK(cudaStreamSynchronize(st));
  }
};

Backend* makeBackend(int device) { return new CudaBackend(device); }
long long backendLaunches(Backend* b) { return static_cast<CudaBackend*>(b)->launches; }

}  // namespace wtg

#define WTG_API(name) wtg_##name
#include "wtg_capi.inl"
