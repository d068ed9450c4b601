// TEST INFRASTRUCTURE — the host build of tests/emu (wtg_emu.cpp) with the pass of a node-sharded Handel network, which
// the CUDA backend runs as k_hpick_publish / k_x_sync(3) / k_hpick_xcheck / k_hpick_xapply between the draw scan and the
// handlers (wittgenstein_b200/csrc/wtg_handel.cuh, "the pick exchange").  Every other network runs HostBackend's pass
// unchanged.  It exports wtgemuh_* symbols and is loaded by tests/emu_handel_lib.py only; the package never loads it.
//
// The C ABI is instantiated here first, with this file's backend factory; wtg_emu.cpp then contributes HostBackend (its own
// instantiation of the C ABI is skipped: wtg_capi.inl is included once per translation unit).
#include "../../wittgenstein_b200/csrc/wtg_engine.hpp"

namespace wtg {
Backend* makeHandelShardsBackend(int device);
}
#define makeBackend makeHandelShardsBackend
#define WTG_API(name) wtgemuh_##name
#include "../../wittgenstein_b200/csrc/wtg_capi.inl"
#undef makeBackend
#undef WTG_API

#include "wtg_emu.cpp"

namespace wtg {

class HandelShardsBackend : public HostBackend {
 public:
  void tick(const Dev& d, int mode) override {
    if (d.proto != PROTO_HANDEL || d.G == 1) {
      HostBackend::tick(d, mode);
      return;
    }
    // node-sharded Handel: no far-future calendar and no caller-issued sends (mode 3) on a sharded network
    CoopSerial c;
    const int n1 = d.n0 + d.nLoc;
    tickBegin(d, mode);
    // conditional pass (checkSigs) of the shard's own nodes, then the pick exchange; a shard in error still publishes its
    // pick header (which carries the error) and signals, so that the others stop at once
    HScratch sc;
    for (int n = d.n0; n < n1; ++n)
      if (hCondMark(d, n)) hCondScanQueue(d, c, n);
    int per = d.workCap / ARENA_STRIPES, tot = stripedTotal(d.ctl->workCnt, per);
    for (int t = 0; t < tot; ++t) hScoreItem(d, c, d.workList[stripedIndex(d.ctl->workCnt, per, t)]);
    for (int n = d.n0; n < n1; ++n) hCondSelect(d, c, n, &sc);
    pairScan(d, 2);
    if (!d.ctl->error)
      for (int n = d.n0; n < n1; ++n) hPickPublish(d, n);
    hPickPublishHeader(d);
    xSignal(d, 3);
    for (int q = 0; q < d.G; ++q) xWaitOne(d, 3, q);
    if (!d.ctl->error) {
      hPickHeaders(d);
      const int upTo = hPicksBelow(d, d.rank + 1);
      for (int t = 0; t < upTo && !d.ctl->hReject; ++t)
        if (hPickRejects(d, t)) d.ctl->hReject = 1;
    }
    if (!d.ctl->error) {
      if (!d.ctl->hReject) {
        const u64 below = (u64)hPicksBelow(d, d.rank);
        for (int n = d.n0; n < n1; ++n) hCondPick(d, n, below + (u64)d.hDrawBase[n], true);
      } else {
        hPickSerial(d);
      }
    }
    if (bail(d, 0)) return;
    if (mode != 2) {  // dispatch and handlers
      int nEv = d.ctl->nEv;
      for (int i = 0; i < nEv; ++i) dispatchCount(d, i);
      pairScan(d, 0);
      if (bail(d, 0)) return;
      for (int i = 0; i < nEv; ++i) dispatchScatter(d, i);
      for (int n = d.n0; n < n1; ++n) nodeProcess(d, c, n, 0);
    }
    pairScan(d, 1);
    // exchange 1 (items -> global creation / draw offsets)
    for (int i = 0; i <= d.ctl->nItems; ++i) xPublishItem(d, i);
    xPublishHeader(d);
    xSignal(d, 0);
    for (int q = 0; q < d.G; ++q) xWaitOne(d, 0, q);
    if (!d.ctl->error) {
      for (int i = 0; i < d.ctl->nItems; ++i) xOffsets(d, i);
      xTotals(d);
    }
    if (bail(d, 1)) return;
    for (int n = d.n0; n < n1; ++n) emitCond(d, n);
    per = d.descCap / ARENA_STRIPES;
    tot = stripedTotal(d.ctl->descCnt, per);
    for (int t = 0; t < tot; ++t) emitDesc(d, stripedIndex(d.ctl->descCnt, per, t));
    // exchange 2: every shard has stored its envelopes (and staged pooled payloads) into the destination shards' regions
    xSignal(d, 1);
    for (int q = 0; q < d.G; ++q) xWaitOne(d, 1, q);
    if (d.ctl->error) return;
    for (int g = 0; g < d.ctl->totalSlots; ++g)
      if (xNeedsIngest(d, g)) xIngest(d, c, g);
    if (d.ctl->error) return;
    // multisplit: stable append into the ring in creation order
    for (int g = 0; g < d.ctl->totalSlots; ++g) {
      int t = d.newTarget[g];
      if (t < 0) continue;
      d.newTarget[g] = -1;  // the array is indexed by the global creation index: clean for the next pass
      int slot = t & (d.ring - 1);
      int pos = d.bucketCount[slot];
      if (pos >= d.bcap) {
        setError(d, ERR_BUCKET_OVERFLOW, t);
        continue;
      }
      d.buckets[(size_t)slot * d.bcap + pos] = d.newEv[g];
      d.bucketKey[(size_t)slot * d.bcap + pos] = orderKey((unsigned)d.ctl->xseq, (unsigned)g);
      d.bucketCount[slot] = pos + 1;
    }
    per = d.freeCap / ARENA_STRIPES;
    tot = stripedTotal(d.ctl->freeCnt, per);
    for (int t = 0; t < tot; ++t) freeApply(d, stripedIndex(d.ctl->freeCnt, per, t));
    tickEnd(d, mode);
    launches += 1;
  }
};

Backend* makeHandelShardsBackend(int) { return new HandelShardsBackend(); }

}  // namespace wtg
