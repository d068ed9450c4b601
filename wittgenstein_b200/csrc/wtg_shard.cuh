// wittgenstein_b200 — node-sharded simulation: one simulation spread over G engines (one GPU each), shard r owning the
// node ids [r * nLoc, (r + 1) * nLoc).  Handlers only touch the destination node's state (SURVEY.md §8e), so a shard runs
// the whole tick pipeline on its own nodes; what has to be global is the reference's *sequential order*:
//   * the creation index g of every new envelope (insertion order of the per-ms lists, Network.java:145-147)
//   * the index of every rd.nextInt() draw (one java.util.Random for the whole network, Network.java:32)
// Both are prefix sums over the tick's events in processing order.  Every bucket entry carries an ordering key
// (creation tick, creation index, position inside a multi-destination record); after the handlers every shard publishes
// its items (key, prefix of slots, prefix of draws) into the other shards' memory, and each shard derives the global
// offsets of its own items by bisection of the other shards' sorted lists (exchange 1).  The emit step then computes
// arrivals with the global draw indices and stores each new envelope straight into the *destination* shard's
// creation-indexed array over NVLink (peer stores; exchange 2), pooled payloads into a staging area of the destination.
// The multisplit of every shard walks the creation-indexed array, so its buckets stay in the reference's order.
// Synchronisation: per pass two flag words per peer (a third for fast-forwarding protocols, another for Handel's pick
// exchange; release / acquire at system scope), waited on by 1-block kernels.
#pragma once
#include "wtg_types.h"

#if !defined(__CUDA_ARCH__)
#include <chrono>
#include <thread>
#endif

namespace wtg {

// `pass` = Ctl.xseq of the pipeline pass that created the envelope (a millisecond can have two passes: the reference's extra
// time++ at the end of a runMs window creates tasks too)
WTG_HD u64 orderKey(unsigned pass, unsigned g) { return ((u64)pass << KEY_PASS_SHIFT) | ((u64)g << KEY_G_SHIFT); }
WTG_HD u64 keySub(int j) { return (u64)(KEY_SUB_MAX - (unsigned)j); }  // position j inside a multi-destination record
WTG_HD int ownerOf(const Dev& d, int n) { return d.G > 1 ? (d.ownShift >= 0 ? (n >> d.ownShift) : n / d.perShard) : 0; }

WTG_HD void xFence() {
#if defined(__CUDA_ARCH__)
  __threadfence_system();
#else
  __atomic_thread_fence(__ATOMIC_SEQ_CST);
#endif
}
WTG_HD int xLoadAcquire(const int* p) {
#if defined(__CUDA_ARCH__)
  int v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#else
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#endif
}
WTG_HD void xStoreRelease(int* p, int v) {
#if defined(__CUDA_ARCH__)
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#else
  __atomic_store_n(p, v, __ATOMIC_RELEASE);
#endif
}

// ---- CasperIMD: block / attestation tables inside the exchange region, one copy per shard (layout from the Dev's sizes) ----
struct CasperTabs {
  CasperG* cg;
  int* cbHeight;
  int* cbParent;
  int* cbProducer;
  int* cbTime;
  int* attHead;
  int* attHeight;
  unsigned long long* cbIncluded;
};
WTG_HD size_t casperTabsBytes(int maxBlocks, int maxAtts, int attWords) {
  return 256 + sizeof(int) * (4 * (size_t)maxBlocks + 2 * (size_t)maxAtts) + 64 + sizeof(unsigned long long) * (size_t)maxBlocks * (size_t)attWords;
}
WTG_HD CasperTabs casperTabsAt(char* base, int maxBlocks, int maxAtts) {
  CasperTabs t;
  t.cg = reinterpret_cast<CasperG*>(base);
  int* p = reinterpret_cast<int*>(base + 256);
  t.cbHeight = p;
  t.cbParent = p + maxBlocks;
  t.cbProducer = p + 2 * (size_t)maxBlocks;
  t.cbTime = p + 3 * (size_t)maxBlocks;
  t.attHead = p + 4 * (size_t)maxBlocks;
  t.attHeight = t.attHead + maxAtts;
  size_t off = 256 + sizeof(int) * (4 * (size_t)maxBlocks + 2 * (size_t)maxAtts);
  off = (off + 63) / 64 * 64;
  t.cbIncluded = reinterpret_cast<unsigned long long*>(base + off);
  return t;
}
WTG_HD CasperTabs casperTabsOf(const Dev& d, int q) { return casperTabsAt(d.peer[q].proto, d.cMaxBlocks, d.cMaxAtts); }

// ---- exchange 1: items -------------------------------------------------------------------------------------------
// local conditional-task totals: the scan over [cond | items] holds them at the first item position
WTG_HD void xLocalCond(const Dev& d, int& condS, int& condD) {
  const Ctl& c = *d.ctl;
  if (c.nItems > 0) {
    condS = d.slotBase[d.nLoc];
    condD = d.drawBase[d.nLoc];
  } else {
    condS = c.totalSlots;
    condD = c.totalDraws;
  }
}
// item i of this shard -> every shard's copy of this shard's list (i == nItems: sentinel with the totals)
WTG_HD void xPublishItem(const Dev& d, int i) {
  const Ctl& c = *d.ctl;
  int condS, condD;
  xLocalCond(d, condS, condD);
  XItem it;
  if (i < c.nItems) {
    it.key = d.itemKey[i];
    it.ps = (uint32_t)(d.slotBase[d.nLoc + i] - condS);
    it.pd = (uint32_t)(d.drawBase[d.nLoc + i] - condD);
  } else {
    it.key = 0;
    it.ps = (uint32_t)(c.totalSlots - condS);
    it.pd = (uint32_t)(c.totalDraws - condD);
  }
  for (int q = 0; q < d.G; ++q) d.peer[q].items[(size_t)d.rank * d.xItemCap + i] = it;
}
WTG_HD void xPublishHeader(const Dev& d) {
  const Ctl& c = *d.ctl;
  int condS, condD;
  xLocalCond(d, condS, condD);
  XHdr h;
  h.seq = c.xseq;
  h.nEv = c.nEv;
  h.nItems = c.nItems;
  h.condSlots = condS;
  h.condDraws = condD;
  h.itemSlots = c.totalSlots - condS;
  h.itemDraws = c.totalDraws - condD;
  h.error = c.error;
  for (int q = 0; q < d.G; ++q) d.peer[q].hdr[d.rank] = h;
}
// after all writes of the phase: sequence number into every shard's flag word of this shard
WTG_HD void xSignal(const Dev& d, int phase) {
  xFence();
  for (int q = 0; q < d.G; ++q) xStoreRelease(&d.peer[q].flags[phase * MAX_SHARDS + d.rank], d.ctl->xseq);
}
// wait until shard q has signalled this pass (bounded: a shard that died must not hang the others)
WTG_HD void xWaitOne(const Dev& d, int phase, int q) {
  const int want = d.ctl->xseq;
  const int* f = &d.peer[d.rank].flags[phase * MAX_SHARDS + q];
#if defined(__CUDA_ARCH__)
  long long t0 = clock64();
  while (xLoadAcquire(f) < want) {
    if (d.ctl->error) return;
    if (clock64() - t0 > 20000000000LL) {  // ~10 s
      setError(d, ERR_PEER_TIMEOUT, q * 2 + phase);
      return;
    }
    __nanosleep(200);
  }
#else
  auto t0 = std::chrono::steady_clock::now();
  while (xLoadAcquire(f) < want) {
    if (d.ctl->error) return;
    if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(60)) {
      setError(d, ERR_PEER_TIMEOUT, q * 2 + phase);
      return;
    }
    std::this_thread::yield();
  }
#endif
}
// global totals of the pass (one thread)
WTG_HD void xTotals(const Dev& d) {
  Ctl& c = *d.ctl;
  const XHdr* h = d.peer[d.rank].hdr;
  int allS = 0, allD = 0, befS = 0, befD = 0, totS = 0, totD = 0, nEv = 0;
  for (int q = 0; q < d.G; ++q) {
    if (h[q].error && !c.error) setError(d, ERR_PEER_ERROR, q);
    if (h[q].seq != c.xseq && !c.error) setError(d, ERR_INTERNAL, 700 + q);
    if (q < d.rank) {
      befS += h[q].condSlots;
      befD += h[q].condDraws;
    }
    allS += h[q].condSlots;
    allD += h[q].condDraws;
    totS += h[q].condSlots + h[q].itemSlots;
    totD += h[q].condDraws + h[q].itemDraws;
    nEv += h[q].nEv;
  }
  c.condXoffS = befS;
  c.condXoffD = befD;
  c.allCondS = allS;
  c.allCondD = allD;
  c.totalSlots = totS;  // from here on: over all shards (length of the creation-indexed arrays, draws of the tick)
  c.totalDraws = totD;
  c.nEvGlobal = nEv;
  if (totS > d.newEvCap) setError(d, ERR_DESC_OVERFLOW, totS);
  if (totS >= (1 << (KEY_PASS_SHIFT - KEY_G_SHIFT)) || (unsigned)c.xseq >= (1u << (64 - KEY_PASS_SHIFT))) setError(d, ERR_INTERNAL, 720);  // ordering-key fields
}
// creation indices / draws of the other shards that precede local item i.  Run after xTotals' inputs are complete but
// independent of its outputs (reads the headers itself).
WTG_HD void xOffsets(const Dev& d, int i) {
  if (d.evSlots[i] == 0 && d.evDraws[i] == 0) return;  // nothing created: nobody asks for the offset
  const XHdr* h = d.peer[d.rank].hdr;
  const u64 key = d.itemKey[i];
  uint32_t xs = 0, xd = 0;
  for (int q = 0; q < d.G; ++q) {
    if (q == d.rank) continue;
    xs += (uint32_t)h[q].condSlots;
    xd += (uint32_t)h[q].condDraws;
    const XItem* a = d.peer[d.rank].items + (size_t)q * d.xItemCap;
    int lo = 0, hi = h[q].nItems;  // first index whose key is smaller than ours = items of q processed before this one
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (a[mid].key > key)
        lo = mid + 1;
      else
        hi = mid;
    }
    xs += a[lo].ps;
    xd += a[lo].pd;
  }
  d.xoffS[i] = xs;
  d.xoffD[i] = xd;
}

// ---- exchange 2: envelopes ---------------------------------------------------------------------------------------
// store a new envelope into the creation-indexed arrays of the shard that owns its destination
WTG_HD void xStoreEnvelope(const Dev& d, int q, int g, const Ev& ev, int target) {
  d.peer[q].newEv[g] = ev;
  d.peer[q].newTarget[g] = target;
}
// copy of a multi-destination record into shard q's sub-arena of this shard; returns the record index on q or -1
WTG_HD int xCopyRecord(const Dev& d, int q, uint32_t from, uint32_t meta, u64 pl, int n, int cur, const uint32_t* dst, const int* arr, uint32_t pad) {
  int ri = WTG_ATOMIC_ADD(&d.ctl->xRecTop[q], 1);
  int off = WTG_ATOMIC_ADD(&d.ctl->xRecDestTop[q], n);
  if (ri >= d.xRecCap || off + n > d.xRecDestCap) {
    setError(d, ERR_REC_OVERFLOW, ri);
    return -1;
  }
  ri += d.rank * d.xRecCap;
  off += d.rank * d.xRecDestCap;
  MultiRec rc;
  rc.from = from;
  rc.meta = meta;
  rc.pl = pl;
  rc.n = (uint32_t)n;
  rc.cur = (uint32_t)cur;
  rc.off = (uint32_t)off;
  rc.pad = pad;  // Envelope.sendTime + 1 (peekMessages)
  d.peer[q].rec[ri] = rc;
  for (int i = 0; i < n; ++i) {
    d.peer[q].recDest[off + i] = dst[i];
    d.peer[q].recArrival[off + i] = arr[i];
  }
  return ri;
}
// A multi-destination envelope whose next arrivals (indices [j0, up) of the sorted list share one arrival) lie on several
// shards gets one bucket entry on every shard that owns one of them, all with the same creation index; each entry
// references a record copy on its shard.  `localRec` >= 0: this shard already holds the record (re-push).
WTG_HD void xPlaceMulti(const Dev& d, int g, uint32_t from, uint32_t meta, u64 pl, int n, int j0, const uint32_t* dst, const int* arr, int localRec, uint32_t pad) {
  int up = j0;
  while (up < n && arr[up] == arr[j0]) ++up;
  uint32_t done = 0;
  for (int j = j0; j < up; ++j) {
    int q = ownerOf(d, (int)dst[j]);
    if (done & (1u << q)) continue;
    done |= 1u << q;
    int ri = (q == d.rank && localRec >= 0) ? localRec : xCopyRecord(d, q, from, meta, pl, n, j0, dst, arr, pad);
    if (ri < 0) return;
    Ev ev;
    ev.kind = EV_MULTI;
    ev.to = dst[j];
    ev.from = from;
    ev.meta = 0;
    ev.pl = 0;
    ev.aux = (uint32_t)ri;
    ev.pad = pad;
    xStoreEnvelope(d, q, g, ev, arr[j0]);
  }
}

// Replicated records (sendAll: every shard built the same sorted record in the same slot `ri`): the bucket entries of the
// group that starts at index j0 — one per shard that owns one of its destinations, all with creation index g; the entry
// carries j0 (Ev.pl) because the shards advance through their copies independently.
WTG_HD void xPlaceReplicated(const Dev& d, int g, int ri, int j0) {
  const MultiRec& rc = d.rec[ri];
  const uint32_t* dst = d.recDest + rc.off;
  const int* arr = d.recArrival + rc.off;
  const int n = (int)rc.n;
  uint32_t done = 0;
  for (int j = j0; j < n && arr[j] == arr[j0]; ++j) {
    int q = ownerOf(d, (int)dst[j]);
    if (done & (1u << q)) continue;
    done |= 1u << q;
    Ev ev;
    ev.kind = EV_MULTI;
    ev.to = dst[j];
    ev.from = rc.from;
    ev.meta = 0;
    ev.pl = (u64)(uint32_t)j0;
    ev.aux = (uint32_t)ri;
    ev.pad = rc.pad;
    xStoreEnvelope(d, q, g, ev, arr[j0]);
    if (done == (1u << d.G) - 1u) break;
  }
}

// ---- begin exchange (fast-forwarding protocols): the next millisecond that holds an event, over all shards ----
// one thread: publish (next, after) of this shard, signal, wait for the others, reduce
WTG_HD void xBeginExchange(const Dev& d, int next, int after, int& gNext, int& gAfter) {
  XBegin b;
  b.seq = d.ctl->xseq;
  b.next = next;
  b.after = after;
  b.error = d.ctl->error;
  for (int q = 0; q < d.G; ++q) d.peer[q].beg[d.rank] = b;
  xSignal(d, 2);
  gNext = next;
  gAfter = after;
  for (int q = 0; q < d.G; ++q) {
    if (q == d.rank) continue;
    xWaitOne(d, 2, q);
    if (d.ctl->error) return;
    const XBegin o = d.peer[d.rank].beg[q];
    if (o.error) {
      setError(d, ERR_PEER_ERROR, q);
      return;
    }
    if (o.seq != d.ctl->xseq) {
      setError(d, ERR_INTERNAL, 710 + q);
      return;
    }
    if (o.next < gNext) gNext = o.next;
    if (o.after < gAfter) gAfter = o.after;
  }
}

// staging slot for a pooled payload addressed to shard q: returns the word offset or -1
WTG_HD int xStageAlloc(const Dev& d, int q, int words) {
  int off = WTG_ATOMIC_ADD(&d.ctl->stageTop[q], words);
  if (off + words > d.stageCapWords) {
    setError(d, ERR_STAGE_OVERFLOW, q);
    return -1;
  }
  return off;
}
WTG_HD u64* xStagePtr(const Dev& d, int onShard, int fromShard, int off) {
  return d.peer[onShard].stage + ((size_t)((d.ctl->xseq & 1) * d.G + fromShard)) * (size_t)d.stageCapWords + (size_t)off;
}

}  // namespace wtg
