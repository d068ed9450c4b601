// TEST INFRASTRUCTURE — the host build of tests/emu (wtg_emu.cpp) with the pass shapes the CUDA backend uses for an
// unsharded GSFSignature network inside a runMs window: the checkSigs of millisecond t+1 runs beside the emission tail of
// millisecond t (CudaBackend::ticks, DESIGN.md §4).  The host runs one order of the two branches, chosen by the tunable
// cond_ahead: 1 runs `k_free -> condBegin -> checkSigs(t+1)` before the tail (scan B, emission, multisplit), 2 after it —
// the two extreme interleavings the device allows.  cond_ahead = 0, windows of one millisecond, and every other network run
// HostBackend's pass unchanged.  It exports wtgemuc_* symbols and is loaded by tests/emu_cond_ahead_lib.py only; the package
// never loads it.
//
// The C ABI is instantiated here first, with this file's backend factory; wtg_emu.cpp then contributes HostBackend (its own
// instantiation of the C ABI is skipped: wtg_capi.inl is included once per translation unit).
#include "../../wittgenstein_b200/csrc/wtg_engine.hpp"

namespace wtg {
Backend* makeCondAheadBackend(int device);
}
#define makeBackend makeCondAheadBackend
#define WTG_API(name) wtgemuc_##name
#include "../../wittgenstein_b200/csrc/wtg_capi.inl"
#undef makeBackend
#undef WTG_API

#include "wtg_emu.cpp"

namespace wtg {

class CondAheadBackend : public HostBackend {
 public:
  void ticks(const Dev& d, int count) override {
    if (d.condAhead == 0 || d.proto != PROTO_GSF || d.G != 1 || count < 2) {
      for (int i = 0; i < count; ++i) tick(d, 1);
      return;
    }
    if (d.shufCap > 0 || d.allCap > 0 || d.ffwd) throw std::logic_error("the GSF pass of this build has no shuffles, sendAll or fast-forward");
    for (int i = 0; i < count; ++i) gsfPass(d, i == 0, i < count - 1);
  }

 private:
  std::vector<uint32_t> keep;
  void gsfCond(const Dev& d, CoopSerial& c) {
    for (int n = d.n0; n < d.n0 + d.nLoc; ++n)
      if (gsfCondMark(d, n)) gsfCondScanQueue(d, c, n);
    int per = d.workCap / ARENA_STRIPES, tot = stripedTotal(d.ctl->workCnt, per);
    for (int t = 0; t < tot; ++t) gsfScoreItem(d, c, d.workList[stripedIndex(d.ctl->workCnt, per, t)]);
    for (int n = d.n0; n < d.n0 + d.nLoc; ++n)
      if (d.condDue[n]) gsfCondSelect(d, c, n, keep.data());
  }
  void freeAll(const Dev& d) {
    int per = d.freeCap / ARENA_STRIPES, tot = stripedTotal(d.ctl->freeCnt, per);
    for (int t = 0; t < tot; ++t) freeApply(d, stripedIndex(d.ctl->freeCnt, per, t));
  }
  // the branch the device forks after the handlers: k_free, k_cond_begin, checkSigs of the next millisecond
  void aheadBranch(const Dev& d, CoopSerial& c) {
    freeAll(d);
    condBegin(d);
    gsfCond(d, c);
  }
  // one mode-1 pass of an unsharded GSF network (GSF has no sendAll, no shuffles and no caller-issued sends in a window)
  void gsfPass(const Dev& d, bool ownCond, bool nextCond) {
    CoopSerial c;
    keep.assign((size_t)std::max(1, d.qcap), 0u);
    if (d.farCap > 0)
      tickBeginFar(d, c, 1, !ownCond);
    else
      tickBegin(d, 1, !ownCond);
    if (d.ctl->error) return;
    if (ownCond) gsfCond(d, c);
    const int nEv = d.ctl->nEv;
    for (int i = 0; i < nEv; ++i) dispatchCount(d, i);
    pairScan(d, 0);
    if (d.ctl->error) return;
    for (int i = 0; i < nEv; ++i) dispatchScatter(d, i);
    for (int n = d.n0; n < d.n0 + d.nLoc; ++n) nodeProcess(d, c, n, 0);
    if (nextCond && d.condAhead == 1) aheadBranch(d, c);
    pairScan(d, 1);
    if (d.ctl->error) return;
    for (int n = d.n0; n < d.n0 + d.nLoc; ++n) emitCond(d, n);
    {
      int per = d.descCap / ARENA_STRIPES, tot = stripedTotal(d.ctl->descCnt, per);
      for (int t = 0; t < tot; ++t) emitDesc(d, stripedIndex(d.ctl->descCnt, per, t));
    }
    if (d.ctl->error) return;
    // multisplit: stable append into the ring in creation order
    const int G = d.ctl->totalSlots;
    for (int g = 0; g < G; ++g) {
      int t = d.newTarget[g];
      if (t < 0) continue;
      int slot = t & (d.ring - 1);
      int pos = d.bucketCount[slot];
      if (pos >= d.bcap) {
        setError(d, ERR_BUCKET_OVERFLOW, t);
        continue;
      }
      d.buckets[(size_t)slot * d.bcap + pos] = d.newEv[g];
      d.bucketCount[slot] = pos + 1;
    }
    if (!nextCond)
      freeAll(d);
    else if (d.condAhead == 2)
      aheadBranch(d, c);
    tickEnd(d, 1, nextCond);
    launches += 1;
  }
};

Backend* makeCondAheadBackend(int) { return new CondAheadBackend(); }

}  // namespace wtg
