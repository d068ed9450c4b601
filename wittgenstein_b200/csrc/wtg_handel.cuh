// wittgenstein_b200 — Handel state-transition bodies (protocols/Handel.java), included by wtg_logic.cuh.
//
//   onNewSig            :753-786   -> hOnNewSig          (one thread per node)
//   dissemination       :331-343, HLevel.doCycle :470-480, getRemainingPeers :482-504 -> hDissemination (lane per level)
//   updateVerifiedSignatures :686-750 -> hUpdate         (warp per node)
//   checkSigs :792-837 + HLevel.bestToVerify :566-630 + createSuicideByzantineSig :538-559 + score :651-664
//                                   -> hCondMark / hCondScanQueue / hScoreItem / hCondSelect / hCondPick
// State layout: six N-bit rows per node (lastAggVerified, totalIncoming, verifiedIndSignatures, toVerifyInd,
// finishedPeers, blacklist); level l of a node is the aligned block of the row, exactly as for GSF.
// totalOutgoing(l) is not stored: it always equals the totalIncoming row restricted to the node's own half of
// level l (it is refreshed from the lower levels' totalIncoming at every improving update, :733-745).
// HiddenByzantine (:840-917) runs inside the pick (hHiddenAttack).
// Node-sharded runs: pooled payloads for a receiver on another shard are staged on that shard at emission (hStageAtEmit),
// and the picks' draw indices are made global by the pick exchange (hPick*, after the local draw scan).
#pragma once

namespace wtg {

constexpr uint32_t HMETA_BAD = 1u << 12;       // SigToVerify.badSig
constexpr uint32_t HMETA_FINISHED = 1u << 13;  // SendSigs.levelFinished

struct HScratch {  // per-coop scratch of the select phase (shared memory on the device)
  int minRank[32];
  unsigned long long bestIn[32];   // (score << 32) | ~index : max = highest score, earliest entry
  unsigned long long bestOut[32];  // (rank << 32) | index   : min = lowest rank, earliest entry
  int removed[32];
  int count[32];
  int hitPeer[32];
  int hitRank[32];
};

// pooled payloads are shared by the queue entry and by every pending updateVerifiedSignatures task that was
// scheduled for it (the reference keeps the SigToVerify object alive); the slab returns to the pool at 0
WTG_HD void hRelease(const Dev& d, int n, int level, uint32_t slot, bool direct) {
  int before = WTG_ATOMIC_ADD(&d.poolRef[level][slot], -1);
  if (before == 1) {
    if (direct)
      freeDirect(d, level, slot);
    else
      freeDeferred(d, n, level, slot);
  }
}
WTG_HD int hMsgSize(int l) { return 1 + ((1 << (l - 1)) / 8) + 96 * 2; }  // Handel.java:256-259
WTG_HD bool rowBit(const u64* row, int i) { return (row[i >> 6] >> (i & 63)) & 1ULL; }
WTG_HD u64* hRow(u64* base, const Dev& d, int n) { return base + (size_t)n * d.W64; }

// sizeIfIncluded (:528-536) and score (:651-664) of a payload against level l of node n
struct HEval {
  int s, score;
};
WTG_HD HEval hEvalFrom(int size, int cLast, int cSig, int cSigIncVer, int cSigVer, bool interInc, bool interLast, int cSigInd) {
  // cSigIncVer = |sig | totInc | verInd|, cSigVer = |sig | verInd|, cSigInd = |verInd | sig| (same as cSigVer)
  HEval e;
  e.s = interInc ? cSigVer : cSigIncVer;
  if (cLast >= size)
    e.score = 0;
  else if (!interLast)
    e.score = cLast + cSig;
  else {
    int v = cSigInd - cLast;
    e.score = v > 0 ? v : 0;
  }
  return e;
}
WTG_HD HEval hEvalScalar(const Dev& d, int n, const HQEntry& e) {
  int l = (int)metaLevel(e.meta);
  int size = 1 << (l - 1);
  int cLast = d.hCntLast[n * d.L + l];
  int kind = (int)metaKind(e.meta);
  if (kind == PK_FULL) {  // the whole level block
    int cInc = d.hCntInc[n * d.L + l];
    return hEvalFrom(size, cLast, size, size, size, cInc > 0, cLast > 0, size);
  }
  Blk b = levelBlock((int)e.from, l);
  u64 sg = e.pl;
  u64 inc = hRow(d.hTotInc, d, n)[b.w0] & b.mask, ind = hRow(d.hVerInd, d, n)[b.w0] & b.mask, la = hRow(d.hLastAgg, d, n)[b.w0] & b.mask;
  return hEvalFrom(size, cLast, WTG_POPC64(sg), WTG_POPC64(sg | inc | ind), WTG_POPC64(sg | ind), (sg & inc) != 0, (sg & la) != 0,
                   WTG_POPC64(sg | ind));
}
template <class C>
WTG_HD HEval hEvalPool(const Dev& d, C& c, int n, uint32_t from, uint32_t meta, u64 pl) {
  int l = (int)metaLevel(meta);
  int size = 1 << (l - 1);
  Blk b = levelBlock((int)from, l);
  const u64* sig = d.pool[l] + (size_t)(uint32_t)pl * (size_t)b.nw;
  const u64* inc = hRow(d.hTotInc, d, n) + b.w0;
  const u64* ind = hRow(d.hVerInd, d, n) + b.w0;
  const u64* la = hRow(d.hLastAgg, d, n) + b.w0;
  int a = 0, v = 0, ii = 0, il = 0;
  for (int w = c.lane(); w < b.nw; w += C::LANES) {
    u64 sg = sig[w], x = inc[w], y = ind[w], z = la[w];
    a += WTG_POPC64(sg | x | y);
    v += WTG_POPC64(sg | y);
    ii |= (sg & x) != 0;
    il |= (sg & z) != 0;
  }
  a = c.sum(a);
  v = c.sum(v);
  bool bi = c.any(ii != 0), bl = c.any(il != 0);
  return hEvalFrom(size, d.hCntLast[n * d.L + l], (int)(pl >> 32), a, v, bi, bl, v);
}

// ---- onNewSig (:753-786): one thread ---------------------------------------------------------------
WTG_HD void hOnNewSig(const Dev& d, int n, uint32_t from, uint32_t meta, u64 pl) {
  const int tick = d.ctl->tick;
  int l = (int)metaLevel(meta);
  bool pooled = metaKind(meta) == PK_POOL;
  if (d.doneAt[n] > 0) {
    d.hMsgFiltered[n] += 1;
    if (pooled) hRelease(d, n, l, (uint32_t)pl, false);
    return;
  }
  if (tick < d.hStartAt[n] || rowBit(hRow(d.hBlack, d, n), (int)from)) {
    if (pooled) hRelease(d, n, l, (uint32_t)pl, false);
    return;
  }
  if (meta & HMETA_FINISHED) hRow(d.hFinPeers, d, n)[from >> 6] |= 1ULL << (from & 63);
  if (!rowBit(hRow(d.hVerInd, d, n), (int)from)) hRow(d.hToVerInd, d, n)[from >> 6] |= 1ULL << (from & 63);
  d.hSigQueueSize[n] += 1;
  int len = d.qLen[n];
  if (len + 1 > d.qcap) {
    setError(d, ERR_QUEUE_OVERFLOW, n);
    if (pooled) hRelease(d, n, l, (uint32_t)pl, false);
    return;
  }
  HQEntry e;
  e.from = from;
  e.meta = meta & ~(HMETA_BAD | HMETA_FINISHED);
  e.pl = pl;
  e.rank = d.hRanks[(size_t)n * d.N + from];
  e.id = (uint32_t)d.hSeq[n]++;
  e.s = 0;
  e.score = 0;
  d.hQueue[(size_t)n * d.qcap + len] = e;
  d.qStamp[(size_t)n * d.qcap + len] = 0;
  d.qLen[n] = len + 1;
  statMax(d, n, ST_MAXQUEUE, (unsigned long long)(len + 1));
}

// getRemainingPeers (:482-504) for one level; executed by one lane.  Returns the number of peers taken.
WTG_HD int hTakePeers(const Dev& d, int n, int l, int want, uint32_t* out) {
  int pos = d.hPos[n * d.L + l];
  bool fin = d.hOutFin[n * d.L + l] != 0;
  const int size = 1 << (l - 1);
  const int start = pos;
  const u64* finRow = hRow(d.hFinPeers, d, n);
  const u64* blRow = hRow(d.hBlack, d, n);
  int cnt = 0;
  while (want > 0 && !fin) {
    int p = (int)peerAt(d, n, l, pos++);
    if (pos >= size) pos = 0;
    if (!rowBit(finRow, p) && !rowBit(blRow, p)) {
      out[cnt++] = (uint32_t)p;
      --want;
    } else if (pos == start) {
      fin = true;
    }
  }
  d.hPos[n * d.L + l] = pos;
  d.hOutFin[n * d.L + l] = fin ? 1 : 0;
  return cnt;
}

// payload of totalOutgoing(l): our own half of level l of the totalIncoming row
template <class C>
WTG_HD bool hMakePayload(const Dev& d, C& c, int n, int l, int card, uint32_t& meta, u64& pl, unsigned long long& words) {
  const int size = 1 << (l - 1);
  if (card == size) {
    meta = metaMake(PK_FULL, (uint32_t)l, (uint32_t)(l - 1));
    pl = 0;
    return true;
  }
  Blk ob = levelBlock(n, l);
  const u64* row = hRow(d.hTotInc, d, n);
  if (l <= INLINE_MAX_LEVEL) {
    meta = metaMake(PK_INLINE, (uint32_t)l, 0);
    pl = row[ob.w0] & ob.mask;
    return true;
  }
  meta = metaMake(PK_POOL, (uint32_t)l, 0);
  uint32_t slot = 0;
  int ok = 1;
  if (c.lane() == 0) ok = poolAlloc(d, l, n, slot) ? 1 : 0;
  slot = (uint32_t)c.bcast((int)slot, 0);
  ok = c.bcast(ok, 0);
  if (ok) {
    if (c.lane() == 0) d.poolRef[l][slot] = 1;
    u64* dst = d.pool[l] + (size_t)slot * (size_t)ob.nw;
    for (int w = c.lane(); w < ob.nw; w += C::LANES) dst[w] = row[ob.w0 + w];
    words += (unsigned long long)(2 * ob.nw);
  }
  pl = (u64)slot | ((u64)(uint32_t)card << 32);
  return ok != 0;
}

// ---- dissemination (:331-343) + periodic re-arm: generic (level loop); all lanes run the scalar part ------
template <class C>
WTG_HD void hDissemination(const Dev& d, C& c, int n, int item, int& outSlots, int& outDraws) {
  const int L = d.L, tick = d.ctl->tick;
  bool active = true;
  if (d.doneAt[n] > 0) {
    int ac = d.hAddedCycle[n];
    c.sync();
    if (ac > 0) {
      if (c.lane() == 0) d.hAddedCycle[n] = ac - 1;
    } else {
      active = false;
    }
  }
  // pass 1 (lane 0 decides; getRemainingPeers mutates the cursor): which levels send, and to whom
  uint32_t dest[MAX_LEVELS];
  uint32_t sendMask = 0;
  int cards[MAX_LEVELS];
  if (active) {
    int prefix = 1;
    for (int l = 1; l < L; ++l) {
      cards[l] = prefix;
      int size = 1 << (l - 1);
      int got = 0;
      uint32_t dd = 0;
      if (c.lane() == 0) {
        bool fin = d.hOutFin[n * L + l] != 0;
        bool open = !fin && (tick >= (l - 1) * d.hLevelWait || prefix == size);  // isOpen :454-468
        if (open) got = hTakePeers(d, n, l, 1, &dd);
      }
      got = c.bcast(got, 0);
      dd = (uint32_t)c.bcast((int)dd, 0);
      if (got) {
        sendMask |= 1u << l;
        dest[l] = dd;
      }
      prefix += d.hCntInc[n * L + l];
    }
  }
  int nSend = WTG_POPC32(sendMask);
  int base = descAlloc(d, c, n, nSend + 1);
  int sub = 0;
  long long bytes = 0;
  unsigned long long words = 0;
  for (int l = 1; l < L; ++l) {
    if (!(sendMask & (1u << l))) continue;
    uint32_t meta;
    u64 pl;
    hMakePayload(d, c, n, l, cards[l], meta, pl, words);
    if (d.hCntInc[n * L + l] == (1 << (l - 1))) meta |= HMETA_FINISHED;  // SendSigs.levelFinished = l.incomingComplete()
    bytes += hMsgSize(l);
    if (base >= 0 && c.lane() == 0) {
      Desc ds;
      ds.dkind = DK_SEND_SINGLE;
      ds.item = (uint32_t)(d.nLoc + item);
      ds.sub = (uint32_t)sub;
      ds.from = (uint32_t)n;
      ds.to = dest[l];
      ds.nDest = 1;
      ds.evKind = EV_MSG;
      ds.meta = meta;
      ds.pl = pl;
      ds.target = 0;
      ds.aux = 0;
      d.desc[base + sub] = ds;
    }
    ++sub;
  }
  if (c.lane() == 0) {
    if (base >= 0) {
      Desc ds;
      ds.dkind = DK_INSERT_AT;
      ds.item = (uint32_t)(d.nLoc + item);
      ds.sub = (uint32_t)sub;
      ds.from = (uint32_t)n;
      ds.to = (uint32_t)n;
      ds.nDest = 0;
      ds.evKind = EV_PERIODIC;
      ds.meta = 0;
      ds.pl = 0;
      ds.target = tick + d.period;
      ds.aux = 0;
      d.desc[base + sub] = ds;
    }
    d.msgSent[n] += nSend;
    d.bytesSent[n] += bytes;
    statAdd(d, n, ST_CYCLES, 1ULL);
    statAdd(d, n, ST_SENDS, (unsigned long long)nSend);
    if (words) statAdd(d, n, ST_SENDWORDS, words);
  }
  c.sync();
  outSlots = nSend + 1;
  outDraws = nSend;
}

// ---- updateVerifiedSignatures (:686-750) -----------------------------------------------------------------
template <class C>
WTG_HD void hUpdate(const Dev& d, C& c, int n, uint32_t from, uint32_t meta, u64 pl, uint32_t id, int item, int& outSlots, int& outDraws) {
  const int L = d.L, tick = d.ctl->tick;
  outSlots = 0;
  outDraws = 0;
  if (c.lane() == 0) statAdd(d, n, ST_UPDATES, 1ULL);
  if (meta & HMETA_BAD) {  // :687-694
    if (c.lane() == 0) {
      hRow(d.hBlack, d, n)[from >> 6] |= 1ULL << (from & 63);
      // a candidate left: the cached minimum rank of the level only changes if it was the one holding it
      int* bm = &d.hBizNoHit[n * L + (int)metaLevel(meta)];
      if (*bm == d.hRanks[(size_t)n * d.N + from]) *bm = -2147483647 - 1;
    }
    c.sync();
    return;
  }
  const int l = (int)metaLevel(meta), kind = (int)metaKind(meta);
  const int size = 1 << (l - 1);
  Blk b = levelBlock((int)from, l);
  u64* rInc = hRow(d.hTotInc, d, n);
  u64* rInd = hRow(d.hVerInd, d, n);
  u64* rLast = hRow(d.hLastAgg, d, n);
  // vsl.toVerifyAgg.remove(vs): drop the queue entry with this id if it is still there (order-preserving)
  {
    int len = d.qLen[n];
    HQEntry* q = d.hQueue + (size_t)n * d.qcap;
    uint32_t* qst = d.qStamp + (size_t)n * d.qcap;
    int found = -1;
    for (int base = 0; base < len && found < 0; base += C::LANES) {
      int i = base + c.lane();
      bool hit = i < len && q[i].id == id;
      uint32_t m = c.ballot(hit);
      if (m) found = base + c.first(m);
    }
    if (found >= 0) {
      for (int base = found; base < len - 1; base += C::LANES) {
        int i = base + c.lane();
        HQEntry e;
        uint32_t st = 0;
        bool ok = i < len - 1;
        if (ok) {
          e = q[i + 1];
          st = qst[i + 1];
        }
        c.sync();
        if (ok) {
          q[i] = e;
          qst[i] = st;
        }
        c.sync();
      }
      if (c.lane() == 0) {
        d.qLen[n] = len - 1;
        if (kind == PK_POOL) hRelease(d, n, l, (uint32_t)pl, false);  // the list's reference
      }
    }
  }
  int cLast = d.hCntLast[n * L + l], cInc = d.hCntInc[n * L + l], cInd = d.hCntInd[n * L + l];
  int total = d.hTotal[n];
  const u64 fbit = 1ULL << (from & 63);
  const int fw = (int)(from >> 6);
  c.sync();
  if (c.lane() == 0) {
    hRow(d.hToVerInd, d, n)[fw] &= ~fbit;  // :701
    d.lvVer[n * L + l] += 1;
  }
  bool hadInd = (rInd[fw] & fbit) != 0, hadInc = (rInc[fw] & fbit) != 0;
  c.sync();
  if (!hadInd) {  // :704
    if (c.lane() == 0) rInd[fw] |= fbit;
    cInd += 1;
  }
  bool improved = false;
  if (!hadInc) {  // :707-710
    if (c.lane() == 0) rInc[fw] |= fbit;
    cInc += 1;
    total += 1;
    improved = true;
  }
  c.sync();
  // all = sig | verifiedInd ; does it add to the individual set?  does sig touch lastAggVerified?
  int cAll = 0;
  bool interLast = false;
  if (kind == PK_FULL) {
    cAll = size;
    interLast = cLast > 0;
  } else if (kind == PK_INLINE) {
    u64 ind = rInd[b.w0] & b.mask;
    cAll = WTG_POPC64(pl | ind);
    interLast = (pl & rLast[b.w0] & b.mask) != 0;
  } else {
    const u64* sig = d.pool[l] + (size_t)(uint32_t)pl * (size_t)b.nw;
    int ca = 0, il = 0;
    for (int w = c.lane(); w < b.nw; w += C::LANES) {
      u64 sg = sig[w];
      ca += WTG_POPC64(sg | rInd[b.w0 + w]);
      il |= (sg & rLast[b.w0 + w]) != 0;
    }
    cAll = c.sum(ca);
    interLast = c.any(il != 0);
  }
  if (cAll > cInd) {  // :714-725
    improved = true;
    int nl = 0, ni = 0;
    if (kind == PK_FULL) {
      for (int w = c.lane(); w < b.nw; w += C::LANES) {
        rLast[b.w0 + w] |= b.mask;
        rInc[b.w0 + w] |= b.mask;
      }
      nl = size;
      ni = size;
    } else if (kind == PK_INLINE) {
      u64 curL = rLast[b.w0], curI = rInc[b.w0], ind = rInd[b.w0] & b.mask;
      u64 newL = (interLast ? 0ULL : (curL & b.mask)) | pl;
      u64 newI = newL | ind;
      c.sync();
      if (c.lane() == 0) {
        rLast[b.w0] = (curL & ~b.mask) | newL;
        rInc[b.w0] = (curI & ~b.mask) | newI;
      }
      nl = WTG_POPC64(newL);
      ni = WTG_POPC64(newI);
    } else {
      const u64* sig = d.pool[l] + (size_t)(uint32_t)pl * (size_t)b.nw;
      int a = 0, bb = 0;
      for (int w = c.lane(); w < b.nw; w += C::LANES) {
        u64 newL = (interLast ? 0ULL : rLast[b.w0 + w]) | sig[w];
        u64 newI = newL | rInd[b.w0 + w];
        rLast[b.w0 + w] = newL;
        rInc[b.w0 + w] = newI;
        a += WTG_POPC64(newL);
        bb += WTG_POPC64(newI);
      }
      nl = c.sum(a);
      ni = c.sum(bb);
    }
    total += ni - cInc;
    cLast = nl;
    cInc = ni;
  }
  if (c.lane() == 0) {
    d.hCntLast[n * L + l] = cLast;
    d.hCntInc[n * L + l] = cInc;
    d.hCntInd[n * L + l] = cInd;
    d.hTotal[n] = total;
    if (kind == PK_POOL) hRelease(d, n, l, (uint32_t)pl, false);  // this task's reference
  }
  c.sync();
  if (!improved) return;
  // :731-745 fast path on the levels above when this level has just been completed
  const bool justCompleted = cInc == size;
  if (justCompleted && d.hFastPath > 0) {
    int prefix = 1;
    for (int j = 1; j <= l; ++j) prefix += d.hCntInc[n * L + j];
    // count the sends (a level sends only if getRemainingPeers finds somebody), allocating one descriptor per send
    int sub = 0;
    long long sentMsgs = 0, sentBytes = 0;
    for (int lv = l + 1; lv < L; ++lv) {
      const int lsz = 1 << (lv - 1);
      if (d.hOutFin[n * L + lv] == 0 && prefix == lsz) {  // !outgoingFinished && outgoingComplete()
        uint32_t dests[MAX_ACC];
        int cnt = 0;
        if (c.lane() == 0) cnt = hTakePeers(d, n, lv, d.hFastPath, dests);
        cnt = c.bcast(cnt, 0);
        if (cnt > 0) {
          int base = descAlloc(d, c, n, 1);
          if (base >= 0 && c.lane() == 0) {
            Desc ds;
            ds.item = (uint32_t)(d.nLoc + item);
            ds.sub = (uint32_t)sub;
            ds.from = (uint32_t)n;
            ds.evKind = EV_MSG;
            ds.meta = metaMake(PK_FULL, (uint32_t)lv, (uint32_t)(lv - 1)) | (d.hCntInc[n * L + lv] == lsz ? HMETA_FINISHED : 0u);
            ds.pl = 0;
            ds.target = 0;
            ds.aux = 0;
            if (cnt == 1) {
              ds.dkind = DK_SEND_SINGLE;
              ds.to = dests[0];
              ds.nDest = 1;
            } else {
              int off = destAlloc(d, n, cnt);
              if (off >= 0)
                for (int i = 0; i < cnt; ++i) d.destScratch[off + i] = dests[i];
              ds.dkind = DK_SEND_MULTI;
              ds.to = (uint32_t)(off < 0 ? 0 : off);
              ds.nDest = (uint32_t)(off < 0 ? 0 : cnt);
            }
            d.desc[base] = ds;
          }
          sentMsgs += cnt;
          sentBytes += (long long)cnt * hMsgSize(lv);
          ++sub;
        }
      }
      prefix += d.hCntInc[n * L + lv];
    }
    if (c.lane() == 0 && sub > 0) {
      d.msgSent[n] += sentMsgs;
      d.bytesSent[n] += sentBytes;
      statAdd(d, n, ST_MULTISENDS, (unsigned long long)sub);
    }
    outSlots = sub;
    outDraws = sub;
  }
  if (c.lane() == 0 && d.doneAt[n] == 0 && total >= d.threshold) d.doneAt[n] = tick;  // :747-749
  c.sync();
}

// ---- checkSigs, phase A: conditional-task bookkeeping (one thread per node) --------------------------------
WTG_HD bool hCondMark(const Dev& d, int n) {
  const Ctl& ctl = *d.ctl;
  bool dueNow = false;
  if (ctl.condMode != 0 && !d.ndown[n]) {
    int ms = d.minStart[n];
    bool due = ctl.condMode == 1 ? (ms <= ctl.tick) : (ms <= ctl.until);
    if (due && d.stamp[n] != ctl.callId) {
      d.stamp[n] = ctl.callId;
      if (d.hSigQueueSize[n] != 0) {  // startIf: hasSigToVerify() :345-347
        dueNow = true;
        d.minStart[n] = ctl.tick + d.pairing[n];
        statAdd(d, n, ST_CONDRUNS, 1ULL);
      }
    }
  }
  d.condDue[n] = dueNow ? 1 : 0;
  d.condFired[n] = 0;
  d.condDraws[n] = 0;
  d.hCandK[n] = 0;
  return dueNow;
}
// phase A, queue part: refresh (sizeIfIncluded, score) of stale entries; pooled ones go to the work list
template <class C>
WTG_HD void hCondScanQueue(const Dev& d, C& c, int n) {
  int len = d.qLen[n];
  HQEntry* q = d.hQueue + (size_t)n * d.qcap;
  uint32_t* qst = d.qStamp + (size_t)n * d.qcap;
  const uint32_t* ver = d.lvVer + (size_t)n * d.L;
  const int st = n & (ARENA_STRIPES - 1);
  const int per = d.workCap / ARENA_STRIPES;
  for (int base = 0; base < len; base += C::LANES) {
    int i = base + c.lane();
    bool stalePool = false;
    if (i < len) {
      HQEntry e = q[i];
      uint32_t v = ver[metaLevel(e.meta)];
      if (qst[i] != v) {
        if (metaKind(e.meta) == PK_POOL) {
          stalePool = true;
        } else {
          HEval r = hEvalScalar(d, n, e);
          q[i].s = r.s;
          q[i].score = r.score;
          qst[i] = v;
        }
      }
    }
    uint32_t pm = c.ballot(stalePool);
    if (pm) {
      int cnt = c.count(pm), off = c.rank(pm);
      int b0 = 0;
      if (c.lane() == 0) b0 = WTG_ATOMIC_ADD(&d.ctl->workCnt[st], cnt);
      b0 = c.bcast(b0, 0);
      if (stalePool) {
        if (b0 + off < per)
          d.workList[(size_t)st * per + b0 + off] = (uint32_t)((size_t)n * d.qcap + i);
        else
          setError(d, ERR_DESC_OVERFLOW, -n);
      }
    }
  }
  if (c.lane() == 0) statAdd(d, n, ST_EVALENTRIES, (unsigned long long)len);
}
template <class C>
WTG_HD void hScoreItem(const Dev& d, C& c, uint32_t item) {
  int n = (int)(item / (uint32_t)d.qcap);
  HQEntry e = d.hQueue[item];
  HEval r = hEvalPool(d, c, n, e.from, e.meta, e.pl);
  if (c.lane() == 0) {
    d.hQueue[item].s = r.s;
    d.hQueue[item].score = r.score;
    d.qStamp[item] = d.lvVer[(size_t)n * d.L + metaLevel(e.meta)];
    statAdd(d, n, ST_EVALWORDS, (unsigned long long)(4 * poolWords((int)metaLevel(e.meta))));
  }
}

// phase C: bestToVerify of every level (:566-630), curation, suicide-Byzantine injection (:538-559).
// Leaves, per node, the candidate of each level (queue index after compaction) in hCand and their count in hCandK.
template <class C>
WTG_HD void hCondSelect(const Dev& d, C& c, int n, HScratch* sc) {
  if (!d.condDue[n]) return;
  const int L = d.L;
  int len = d.qLen[n];
  HQEntry* q = d.hQueue + (size_t)n * d.qcap;
  uint32_t* qst = d.qStamp + (size_t)n * d.qcap;
  const u64* blRow = hRow(d.hBlack, d, n);
  const int window = d.hWindow[n];
  for (int l = c.lane(); l < 32; l += C::LANES) {
    sc->minRank[l] = 0x7fffffff;
    sc->bestIn[l] = 0ULL;
    sc->bestOut[l] = ~0ULL;
    sc->removed[l] = 0;
    sc->count[l] = 0;
    sc->hitPeer[l] = -1;
    sc->hitRank[l] = 0;
  }
  c.sync();
  // 1. window index = lowest rank of the level's list (:574-575)
  for (int base = 0; base < len; base += C::LANES) {
    int i = base + c.lane();
    if (i < len) {
      int l = (int)metaLevel(q[i].meta);
      WTG_ATOMIC_MIN(&sc->minRank[l], (int)q[i].rank);
      WTG_ATOMIC_ADD(&sc->count[l], 1);
    }
  }
  c.sync();
  // 2. createSuicideByzantineSig (:538-559).  All lanes scan the emission list of one level together.
  //    (a) suicideBizAfter = first peer at or after the old index that is down and not blacklisted (or -1);
  //    (b) the injected signature comes from the first such peer whose reception rank is < maxRank.  hBizNoHit
  //        holds the exact minimum rank over the level's candidates (recomputed lazily after a candidate's rank
  //        was bumped or it was blacklisted), so "nobody qualifies" is answered without walking the list.
  // One lane per level first answers the common case from cached state: the peer at the old index is still a
  // candidate (so suicideBizAfter does not move) and the level's cached minimum rank says nobody is below maxRank.
  // Only the levels that need a walk of the emission list take the cooperative path below.
  uint32_t slowLevels = 0;
  for (int k = 0; k < 32 / C::LANES; ++k) {  // levels as lanes (see gsfLastFinishedLevel)
    const int l = k * C::LANES + c.lane();
    bool slow = false;
    if (l >= 1 && l < L && sc->count[l] > 0) {
      int biz = d.hBiz[n * L + l];
      if (biz >= 0) {
        int p = (int)peerAt(d, n, l, biz);
        int bmin = d.hBizNoHit[n * L + l];
        slow = !(d.ndown[p] && !rowBit(blRow, p)) || bmin == (-2147483647 - 1) || sc->minRank[l] + window > bmin;
      }
    }
    slowLevels |= c.ballot(slow) << (k * C::LANES);
  }
  for (int l = 1; l < L; ++l) {
    if (!((slowLevels >> l) & 1u)) continue;
    int biz = d.hBiz[n * L + l];
    if (sc->count[l] <= 0 || biz < 0) continue;
    const int size = 1 << (l - 1);
    const int maxRank = sc->minRank[l] + window;
    int first = -1;
    for (int base = biz; base < size && first < 0; base += C::LANES) {
      int i = base + c.lane();
      bool cand = false;
      if (i < size) {
        int p = (int)peerAt(d, n, l, i);
        cand = d.ndown[p] && !rowBit(blRow, p);
      }
      uint32_t m = c.ballot(cand);
      if (m) first = base + c.first(m);
    }
    int hitP = -1, hitR = 0;
    if (first >= 0) {
      const int HB_DIRTY = -2147483647 - 1;
      int bmin = d.hBizNoHit[n * L + l];  // exact minimum rank over the level's candidates, or HB_DIRTY
      if (bmin == HB_DIRTY) {
        // full pass: minimum rank over all candidates and, on the way, the first one below maxRank
        int lmin = 0x7fffffff;
        constexpr int FU = 4;  // chunks of the emission list in flight per lane (the walk is a chain of dependent loads)
        for (int base = first; base < size; base += C::LANES * FU) {
          int pp[FU], rr[FU];
          bool cc[FU];
#pragma unroll
          for (int u = 0; u < FU; ++u) {
            int i = base + u * C::LANES + c.lane();
            pp[u] = i < size ? (int)peerAt(d, n, l, i) : -1;
          }
#pragma unroll
          for (int u = 0; u < FU; ++u) {
            cc[u] = pp[u] >= 0 && d.ndown[pp[u]] && !rowBit(blRow, pp[u]);
            rr[u] = pp[u] >= 0 ? d.hRanks[(size_t)n * d.N + pp[u]] : 0;
          }
#pragma unroll
          for (int u = 0; u < FU; ++u) {
            bool hit = false;
            if (cc[u]) {
              if (rr[u] < lmin) lmin = rr[u];
              hit = rr[u] < maxRank;
            }
            uint32_t m = c.ballot(hit);
            if (m && hitP < 0) {
              int src = c.first(m);
              hitP = c.bcast(pp[u], src);
              hitR = c.bcast(rr[u], src);
            }
          }
        }
        lmin = c.minv(lmin);
        if (c.lane() == 0) d.hBizNoHit[n * L + l] = lmin;
      } else if (maxRank > bmin) {  // somebody qualifies: find the first one in emission order
        constexpr int FU = 4;
        for (int base = first; base < size && hitP < 0; base += C::LANES * FU) {
          int pp[FU], rr[FU];
          bool cc[FU];
#pragma unroll
          for (int u = 0; u < FU; ++u) {
            int i = base + u * C::LANES + c.lane();
            pp[u] = i < size ? (int)peerAt(d, n, l, i) : -1;
          }
#pragma unroll
          for (int u = 0; u < FU; ++u) {
            cc[u] = pp[u] >= 0 && d.ndown[pp[u]] && !rowBit(blRow, pp[u]);
            rr[u] = pp[u] >= 0 ? d.hRanks[(size_t)n * d.N + pp[u]] : 0;
          }
#pragma unroll
          for (int u = 0; u < FU; ++u) {
            uint32_t m = c.ballot(cc[u] && rr[u] < maxRank);
            if (m && hitP < 0) {
              int src = c.first(m);
              hitP = c.bcast(pp[u], src);
              hitR = c.bcast(rr[u], src);
            }
          }
        }
      }
    }
    if (c.lane() == 0) {
      d.hBiz[n * L + l] = first;  // -1: no Byzantine peer left in this level
      sc->hitPeer[l] = hitP;
      sc->hitRank[l] = hitR;
    }
  }
  c.sync();
  // 3. curation flags of the levels without an injected signature (:591-614) + compaction
  int w = 0;
  for (int base = 0; base < len; base += C::LANES) {
    int i = base + c.lane();
    HQEntry e;
    uint32_t st = 0;
    bool keep = false;
    if (i < len) {
      e = q[i];
      st = qst[i];
      int l = (int)metaLevel(e.meta);
      if (sc->hitPeer[l] >= 0) {
        keep = true;
      } else {
        keep = !rowBit(blRow, (int)e.from) && e.s > d.hCntInc[n * L + l];
        if (!keep) {
          WTG_ATOMIC_ADD(&sc->removed[l], 1);
          if (metaKind(e.meta) == PK_POOL) hRelease(d, n, l, (uint32_t)e.pl, true);
        }
      }
    }
    uint32_t km = c.ballot(keep);
    c.sync();
    int off = c.rank(km), tot = c.count(km);
    if (keep && w + off != i) {
      q[w + off] = e;
      qst[w + off] = st;
    }
    w += tot;
    c.sync();
  }
  len = w;
  // 4. best inside the window by score (first strict max), best outside by rank (first min) (:599-610)
  for (int base = 0; base < len; base += C::LANES) {
    int i = base + c.lane();
    if (i < len) {
      HQEntry e = q[i];
      int l = (int)metaLevel(e.meta);
      if (sc->hitPeer[l] < 0) {
        if ((int)e.rank <= sc->minRank[l] + window) {
          if (e.score > 0) WTG_ATOMIC_MAX(&sc->bestIn[l], ((unsigned long long)(uint32_t)e.score << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)i));
        } else {
          WTG_ATOMIC_MIN(&sc->bestOut[l], ((unsigned long long)e.rank << 32) | (unsigned long long)(uint32_t)i);
        }
      }
    }
  }
  c.sync();
  // 5. append the injected signatures (level order) and publish the per-level candidates
  if (c.lane() == 0) {
    int removedTotal = 0, k = 0;
    int sqs = d.hSigQueueSize[n];
    for (int l = 1; l < L; ++l) {
      int cand = -1;
      if (sc->count[l] == 0) {
        d.hCand[(size_t)n * 32 + l] = -1;
        continue;
      }
      if (sc->hitPeer[l] >= 0) {
        if (len + 1 > d.qcap) {
          setError(d, ERR_QUEUE_OVERFLOW, n);
        } else {
          HQEntry e;
          e.from = (uint32_t)sc->hitPeer[l];
          e.meta = metaMake(PK_FULL, (uint32_t)l, (uint32_t)(l - 1)) | HMETA_BAD;  // sig = waitedSigs, badSig = true
          e.pl = 0;
          e.rank = (uint32_t)sc->hitRank[l];
          e.id = (uint32_t)d.hSeq[n]++;
          e.s = 0;
          e.score = 0;
          q[len] = e;
          qst[len] = 0;
          cand = len;
          ++len;
          ++sqs;  // :580-581
        }
      } else {
        removedTotal += sc->removed[l];
        if (sc->bestIn[l] != 0ULL)
          cand = (int)(0xFFFFFFFFu - (uint32_t)(sc->bestIn[l] & 0xFFFFFFFFULL));
        else if (sc->bestOut[l] != ~0ULL)
          cand = (int)(uint32_t)(sc->bestOut[l] & 0xFFFFFFFFULL);
      }
      d.hCand[(size_t)n * 32 + l] = cand;
      if (cand >= 0) ++k;
    }
    d.hCand[(size_t)n * 32] = -1;
    sqs -= removedTotal;  // replaceToVerifyAgg :632-642
    d.hSigQueueSize[n] = sqs;
    d.qLen[n] = len;
    d.hCandK[n] = k;
    d.condDraws[n] = k > 0 ? 1 : 0;  // chooseBestFromLevels draws rd.nextInt(k) (:788-790), even for k == 1
  }
  c.sync();
}

// HiddenByzantine.attack (:861-916) on the level-(L-1) candidate `ci` of node n; returns the queue index of the
// signature to verify.  Scalar: runs inside the pick, after the level draw.  Nothing changed the node's state since
// the select phase, so every queued entry of the level is still improving and carries a fresh (s, score); only the
// injected signature can be curated away by the second bestToVerify() (:566-630).
WTG_HD int hHiddenAttack(const Dev& d, int n, int ci) {
  const int L = d.L, lvl = L - 1;
  HQEntry* q = d.hQueue + (size_t)n * d.qcap;
  uint32_t* qst = d.qStamp + (size_t)n * d.qcap;
  if (d.hbNoPeers[n]) return ci;
  const HQEntry cur = q[ci];
  if (d.hbLastId[n] >= 0 && (uint32_t)d.hbLastId[n] == cur.id) {  // last == currentBest: a previous attack worked
    d.hbLastId[n] = -1;
    return ci;
  }
  int len = d.qLen[n];
  const u64* incRow = hRow(d.hTotInc, d, n);
  if (d.hbLastId[n] >= 0) {
    for (int i = 0; i < len; ++i)
      if ((int)metaLevel(q[i].meta) == lvl && q[i].id == (uint32_t)d.hbLastId[n]) return ci;  // still queued
    if (!rowBit(incRow, d.hbLastFrom[n])) {  // IllegalStateException("byz signature pruned!")
      setError(d, ERR_PROTO_STATE, 20);
      return ci;
    }
    d.hbLastId[n] = -1;
  }
  // firstByzantine (:844-858): lowest reception rank among the down peers not yet in totalIncoming, first in emission order
  const int size = 1 << (lvl - 1);
  int fb = -1, bestRank = 0x7fffffff;
  for (int i = 0; i < size; ++i) {
    int p = (int)peerAt(d, n, lvl, i);
    if (!d.ndown[p]) continue;
    int rk = d.hRanks[(size_t)n * d.N + p];
    if (rk < bestRank && !rowBit(incRow, p)) {
      bestRank = rk;
      fb = p;
      if (rk == 0) break;
    }
  }
  if (fb < 0) {
    d.hbNoPeers[n] = 1;
    return ci;
  }
  if (bestRank >= (int)cur.rank) return ci;  // we can't improve it
  if (len + 1 > d.qcap) {
    setError(d, ERR_QUEUE_OVERFLOW, n);
    return ci;
  }
  HQEntry bad;
  bad.from = (uint32_t)fb;
  bad.rank = (uint32_t)bestRank;
  HEval r;
  if (lvl <= INLINE_MAX_LEVEL) {  // sig = {firstByzantine}
    bad.meta = metaMake(PK_INLINE, (uint32_t)lvl, 0);
    bad.pl = 1ULL << (fb & 63);
    r = hEvalScalar(d, n, bad);
  } else {
    uint32_t slot = 0;
    if (!poolAlloc(d, lvl, n, slot)) return ci;
    d.poolRef[lvl][slot] = 1;
    Blk fbk = levelBlock(fb, lvl);
    u64* slab = d.pool[lvl] + (size_t)slot * (size_t)fbk.nw;
    for (int w = 0; w < fbk.nw; ++w) slab[w] = 0;
    slab[(fb >> 6) - fbk.w0] = 1ULL << (fb & 63);
    bad.meta = metaMake(PK_POOL, (uint32_t)lvl, 0);
    bad.pl = (u64)slot | (1ULL << 32);
    CoopSerial cs;
    r = hEvalPool(d, cs, n, (uint32_t)fb, bad.meta, bad.pl);
  }
  bad.id = (uint32_t)d.hSeq[n]++;
  bad.s = r.s;
  bad.score = r.score;
  const int bi = len;
  q[bi] = bad;
  qst[bi] = d.lvVer[(size_t)n * L + lvl];
  d.qLen[n] = ++len;
  d.hSigQueueSize[n] += 1;
  // l.bestToVerify() again: the window index is the lowest rank of the whole list, curated entries included (:574-575)
  int minRank = 0x7fffffff;
  for (int i = 0; i < len; ++i)
    if ((int)metaLevel(q[i].meta) == lvl && (int)q[i].rank < minRank) minRank = (int)q[i].rank;
  const bool badKept = !rowBit(hRow(d.hBlack, d, n), fb) && bad.s > d.hCntInc[n * L + lvl];
  if (!badKept) {  // replaceToVerifyAgg (:616-618, 632-642)
    d.qLen[n] = --len;
    d.hSigQueueSize[n] -= 1;
    if (metaKind(bad.meta) == PK_POOL) hRelease(d, n, lvl, (uint32_t)bad.pl, false);
  }
  const int lim = minRank + d.hWindow[n];
  int bestIn = -1, bestInScore = 0, bestOut = -1;
  for (int i = 0; i < len; ++i) {
    if ((int)metaLevel(q[i].meta) != lvl) continue;
    if ((int)q[i].rank <= lim) {
      if (q[i].score > bestInScore) {
        bestInScore = q[i].score;
        bestIn = i;
      }
    } else if (bestOut < 0 || q[i].rank < q[bestOut].rank) {
      bestOut = i;
    }
  }
  int nb = bestIn >= 0 ? bestIn : bestOut;
  if (nb < 0) {  // cannot happen: the list holds at least currentBest
    setError(d, ERR_INTERNAL, 21);
    return ci;
  }
  if (nb != bi || !badKept) {
    d.hbLastId[n] = (int)bad.id;
    d.hbLastFrom[n] = fb;
  }
  return nb;
}

// java.util.Random.nextInt(k) at stream index `drawIdx` after ctl.rng: the value in r, the stream values consumed returned
WTG_HD int hNextInt(const Dev& d, u64 drawIdx, int k, int& r) {
  int used = 0;
  for (;;) {
    u64 st = lcgAdvance(d.jumpA, d.jumpC, d.ctl->rng, drawIdx + (u64)used + 1);
    ++used;
    int32_t u = (int32_t)(uint32_t)(st >> 17);
    if ((k & (k - 1)) == 0) {
      r = (int)(((long long)k * (long long)u) >> 31);
      return used;
    }
    r = u % k;
    if ((int32_t)((uint32_t)u - (uint32_t)r + (uint32_t)(k - 1)) >= 0) return used;
  }
}
// phase D: pick the level with network.rd.nextInt(k) and finish checkSigs (:808-837).  `drawIdx` = index of this
// node's draw in the stream after ctl.rng (exclusive scan of condDraws over nodes).  Returns the number of
// stream values consumed (1, or more when nextInt's rejection loop fires).
WTG_HD int hCondPick(const Dev& d, int n, u64 drawIdx, bool apply) {
  int k = d.hCandK[n];
  if (k <= 0) return 0;
  int r;
  const int used = hNextInt(d, drawIdx, k, r);
  if (!apply) return used;
  int lvl = -1, seen = 0;
  for (int l = 1; l < d.L; ++l)
    if (d.hCand[(size_t)n * 32 + l] >= 0) {
      if (seen == r) {
        lvl = l;
        break;
      }
      ++seen;
    }
  int ci = d.hCand[(size_t)n * 32 + lvl];
  if (d.hHidden && lvl == d.L - 1) ci = hHiddenAttack(d, n, ci);  // :813-817
  HQEntry e = d.hQueue[(size_t)n * d.qcap + ci];
  const bool bad = (e.meta & HMETA_BAD) != 0;
  // window (:821-822): ScoringExp(2,4) ceil(curr*2) / floor(curr/4), clamped to [min,max], then to the level size
  int curr = d.hWindow[n];
  int upd = bad ? curr / 4 : curr * 2;
  if (upd > d.hWinMax) upd = d.hWinMax;
  if (upd < d.hWinMin) upd = d.hWinMin;
  int lsz = 1 << (lvl - 1);
  d.hWindow[n] = upd < lsz ? upd : lsz;
  // :825-828 put the sender at the end of the ranking
  int* rk = &d.hRanks[(size_t)n * d.N + e.from];
  const int oldRank = *rk;
  int nr = (int)((uint32_t)oldRank + (uint32_t)d.N);
  if (nr < 0) nr = 0x7fffffff;
  *rk = nr;
  // a candidate's rank grew: the level's cached minimum only changes if this candidate held it
  if (d.ndown[e.from] && d.hBizNoHit[n * d.L + lvl] == oldRank) d.hBizNoHit[n * d.L + lvl] = -2147483647 - 1;
  d.hSigsChecked[n] += 1;
  if (metaKind(e.meta) == PK_POOL) WTG_ATOMIC_ADD(&d.poolRef[metaLevel(e.meta)][(uint32_t)e.pl], 1);
  Ev ev;
  ev.kind = EV_TASK;
  ev.to = (uint32_t)n;
  ev.from = e.from;
  ev.meta = e.meta;
  ev.pl = e.pl;
  ev.aux = e.id;
  ev.pad = (uint32_t)d.ctl->tick + 1u;  // registerTask at network.time: EnvelopeInfo.sentAt + 1
  d.condEv[n] = ev;
  d.condTarget[n] = d.ctl->tick + d.pairing[n];
  d.condFired[n] = 1;
  d.condDraws[n] = used;
  return used;
}

// node-sharded runs: a pooled dissemination payload (hMakePayload) whose receiver lives on another shard moves at emission
// from its slab into that shard's staging area (the slab held only the envelope's reference); k_x2_ingest puts it into a
// slab there.  Emission never allocates, so the slab goes straight back to its free stack.
WTG_HD void hStageAtEmit(const Dev& d, Ev& ev) {
  const int l = (int)metaLevel(ev.meta), nw = poolWords(l), q = ownerOf(d, (int)ev.to);
  const uint32_t slot = (uint32_t)ev.pl;
  const int off = xStageAlloc(d, q, nw);
  if (off >= 0) {
    const u64* src = d.pool[l] + (size_t)slot * (size_t)nw;
    u64* dst = xStagePtr(d, q, d.rank, off);
    for (int w = 0; w < nw; ++w) dst[w] = src[w];
  }
  freeDirect(d, l, slot);
  ev.meta |= META_STAGED | ((uint32_t)d.rank << META_SRC_SHIFT);
  ev.pl = (ev.pl & 0xFFFFFFFF00000000ULL) | (u64)(uint32_t)(off >= 0 ? off : 0);
}

// ---- node-sharded runs: the pick exchange ---------------------------------------------------------------------------
// The conditional pass runs in node-id order before any message of the millisecond, so the level draw of node n sits at
// (picks of the shards below) + (local exclusive scan of the draws, hDrawBase[n]).  Every pick presumes one draw.  Each shard
// publishes its sequence of k values (one byte per pick, node order) and its pick count to every shard, then signals; after
// the wait every shard replays the picks of the pass up to its own on their presumed positions.  None rejects (the common
// case): the presumed positions are the real ones.  One rejects: one thread walks all picks in order (the first rejection
// is found at its real position, every later one is shifted), exactly like the unsharded serial path.
// the pick exchange's part of a shard's exchange region: XPick [G] (256 bytes), then the k values [G][perShard]
WTG_HD size_t hPickBytes(int G, int perShard) { return 256 + (size_t)G * (size_t)perShard; }
WTG_HD XPick* hPickHdr(const Dev& d, int q) { return reinterpret_cast<XPick*>(d.peer[q].proto); }
WTG_HD unsigned char* hPickK(const Dev& d, int q) { return reinterpret_cast<unsigned char*>(d.peer[q].proto) + 256; }
WTG_HD void hPickPublish(const Dev& d, int n) {
  const int k = d.hCandK[n];
  if (k <= 0) return;
  const size_t at = (size_t)d.rank * (size_t)d.perShard + (size_t)d.hDrawBase[n];
  for (int q = 0; q < d.G; ++q) hPickK(d, q)[at] = (unsigned char)k;
}
WTG_HD void hPickPublishHeader(const Dev& d) {
  XPick h;
  h.seq = d.ctl->xseq;
  h.error = d.ctl->error;
  const int last = d.n0 + d.nLoc - 1;
  h.picks = d.ctl->error ? 0 : d.hDrawBase[last] + d.condDraws[last];
  h.pad = 0;
  for (int q = 0; q < d.G; ++q) hPickHdr(d, q)[d.rank] = h;
}
// after the wait (one thread): errors of the other shards; the test hook takes the serial path
WTG_HD void hPickHeaders(const Dev& d) {
  const XPick* h = hPickHdr(d, d.rank);
  for (int q = 0; q < d.G; ++q) {
    if (h[q].error && !d.ctl->error) setError(d, ERR_PEER_ERROR, q);
    if (h[q].seq != d.ctl->xseq && !d.ctl->error) setError(d, ERR_INTERNAL, 730 + q);
  }
  if (d.forcePickSerial) d.ctl->hReject = 1;
}
// picks of the pass on the shards below shard q
WTG_HD int hPicksBelow(const Dev& d, int q) {
  int s = 0;
  for (int p = 0; p < q; ++p) s += hPickHdr(d, d.rank)[p].picks;
  return s;
}
// does pick t of the pass (counted over the shards up to this one) reject at its presumed position t?
WTG_HD bool hPickRejects(const Dev& d, int t) {
  const XPick* h = hPickHdr(d, d.rank);
  int q = 0, base = 0;
  while (q < d.rank && t >= base + h[q].picks) base += h[q++].picks;
  int r;
  return hNextInt(d, (u64)t, (int)hPickK(d, d.rank)[(size_t)q * (size_t)d.perShard + (size_t)(t - base)], r) > 1;
}
// one thread: the real positions of every pick of the pass, in shard and node order
WTG_HD void hPickSerial(const Dev& d) {
  u64 idx = 0;
  int r;
  for (int q = 0; q < d.rank; ++q) {
    const unsigned char* ks = hPickK(d, d.rank) + (size_t)q * (size_t)d.perShard;
    const int cnt = hPickHdr(d, d.rank)[q].picks;
    for (int j = 0; j < cnt; ++j) idx += (u64)hNextInt(d, idx, (int)ks[j], r);
  }
  for (int n = d.n0; n < d.n0 + d.nLoc; ++n) idx += (u64)hCondPick(d, n, idx, true);
}

}  // namespace wtg
