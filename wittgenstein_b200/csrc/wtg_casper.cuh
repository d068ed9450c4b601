// wittgenstein_b200 — CasperIMD handlers (protocols/CasperIMD.java, core/BlockChainNode.java, core/Block.java),
// the sendAll emission path and the far-future calendar they need.  Included by wtg_logic.cuh.
//
// Device representation (DESIGN.md §9):
//   * blocks are rows of a global table (index == creation order == Block.id; genesis = 0);
//   * an attestation is identified by (attester, k-th vote): index k * attestersCount + attester rank, with its head
//     block and slot in attHead / attHeight; `hs` (CasperIMD.java:108,122-126) is implicit: a block h is attested by a
//     iff h is a proper ancestor of a.head at most cycleLength heights below it;
//   * per node: attestations received (one bitmap over attestation indices = every set of attestationsByHead),
//     blocks received, blocksToReevaluate (bitmaps over block indices), head;
//   * per block: the attestations it newly includes (bitmap) = attestationsByHeight flattened (the height is attHeight).
// blocksToReevaluate is folded in ascending block id (the reference's HashSet order is JVM-dependent, see DESIGN.md).
#pragma once

namespace wtg {

struct CMask {  // a set of blocks
  u64 w[CASPER_MAX_BLKWORDS];
};
WTG_HD void cmaskClear(CMask& m) {
  for (int i = 0; i < CASPER_MAX_BLKWORDS; ++i) m.w[i] = 0;
}
WTG_HD void cmaskSet(CMask& m, int b) { m.w[b >> 6] |= 1ULL << (b & 63); }
WTG_HD bool cmaskHas(const CMask& m, int b) { return (m.w[b >> 6] >> (b & 63)) & 1ULL; }

WTG_HD int casperPeriod(const Dev& d, int kind) {  // CasperIMD.java:481-506
  return kind == CK_ATTESTER ? CASPER_SLOT * d.cCycle : CASPER_SLOT * d.cBpCount;
}

// Block.hasDirectLink (Block.java:87-100)
WTG_HD bool cHasDirectLink(const Dev& d, int a, int b) {
  if (a == b) return true;
  int ha = d.cbHeight[a], hb = d.cbHeight[b];
  if (ha == hb) return false;
  int older = ha > hb ? a : b, young = ha < hb ? a : b;
  int hy = d.cbHeight[young];
  while (d.cbHeight[older] > hy) older = d.cbParent[older];
  return older == young;
}

// Attestation.attests (CasperIMD.java:134-136) with hs as built by the constructor (:122-126)
WTG_HD bool cAttests(const Dev& d, int a, int h) {
  int head = d.attHead[a];
  int lim = d.cbHeight[head] - d.cCycle;
  for (int cur = d.cbParent[head]; cur >= 0 && d.cbHeight[cur] >= lim; cur = d.cbParent[cur])
    if (cur == h) return true;
  return false;
}

// countAttestations (CasperIMD.java:262-288): attestations for h on the branch start -> h, received or included
template <class C>
WTG_HD int cCountAttestations(const Dev& d, C& c, int n, int start, int h) {
  CMask chain;
  cmaskClear(chain);
  for (int cur = start; cur != h && cur >= 0; cur = d.cbParent[cur]) cmaskSet(chain, cur);
  const int hh = d.cbHeight[h];
  const int W = d.cAttWords;
  const u64* recv = d.cAttRecv + (size_t)n * W;
  int cnt = 0;
  for (int w = c.lane(); w < W; w += C::LANES) {
    u64 rw = recv[w];
    u64 cand = rw;
    for (int cur = start; cur != h && cur >= 0; cur = d.cbParent[cur]) cand |= d.cbIncluded[(size_t)cur * W + w];
    while (cand) {
      int b = WTG_CTZ64(cand);
      cand &= cand - 1;
      int a = w * 64 + b;
      bool in = ((rw >> b) & 1ULL) && cmaskHas(chain, d.attHead[a]);  // received, with a head on our branch (:282-284)
      if (!in) {
        int ah = d.attHeight[a];
        for (int cur = start; cur != h && cur >= 0 && !in; cur = d.cbParent[cur])  // contained in a block of the branch (:273-278)
          in = ((d.cbIncluded[(size_t)cur * W + w] >> b) & 1ULL) && ah > hh && ah < d.cbHeight[cur];
      }
      if (in && cAttests(d, a, h)) ++cnt;
    }
  }
  return c.sum(cnt);
}

// network.rd.nextBoolean() on a fork-choice tie (CasperIMD.java:250-253) is a draw from the network's one Random *inside* a
// handler: its index is the number of draws of every event processed before this one in the millisecond, which the parallel
// handler pass cannot know.  Every tie of a handler comes before the handler's first non-idempotent write (reevaluateHead
// folds before it stores the head; onBlock compares before it records the block), so a handler that hits a tie can simply
// stop: the node is suspended at that event, and the tie pass (casperResolveTies: one warp, after the parallel pass) runs the
// suspended events in processing order, each with its exact draw index (all earlier events are complete by then).
struct CTie {
  int resolve;  // 0: parallel pass (a tie suspends the node); 1: tie pass (draws are taken at base + used)
  u64 base;     // draws of all events processed before this one in the pass
  int used;     // ties drawn by this event so far
  bool hit;     // parallel pass: a tie was found, nothing may be written
};
// CasperNode.best (CasperIMD.java:205-257)
template <class C>
WTG_HD int cBest(const Dev& d, C& c, int n, int o1, int o2, CTie& tc) {
  if (o1 == o2) return o1;
  int h1 = d.cbHeight[o1], h2 = d.cbHeight[o2];
  if (h1 == h2) {  // two blocks for the same height: IllegalStateException (:208-212)
    setError(d, ERR_PROTO_STATE, 1);
    return o1;
  }
  if (cHasDirectLink(d, o1, o2)) return h1 < h2 ? o2 : o1;
  int b1 = o1, b2 = o2;
  while (d.cbParent[b1] != d.cbParent[b2]) {
    int p1 = d.cbParent[b1], p2 = d.cbParent[b2];
    if (p1 < 0 || p2 < 0) {
      setError(d, ERR_PROTO_STATE, 5);
      return o1;
    }
    if (d.cbHeight[p1] > d.cbHeight[p2])
      b1 = p1;
    else
      b2 = p2;
  }
  int h = d.cbParent[b1];
  int v1 = cCountAttestations(d, c, n, o1, h);
  int v2 = cCountAttestations(d, c, n, o2, h);
  if (v1 > v2) return o1;
  if (v1 < v2) return o2;
  if (d.cRandomTies) {  // return network.rd.nextBoolean() ? o1 : o2  (:250-253)
    if (d.G > 1) {  // node-sharded runs would need the draw prefix of the other shards' events here
      setError(d, ERR_UNSUPPORTED, 1);
      return o1;
    }
    if (!tc.resolve) {
      tc.hit = true;
      return o1;
    }
    u64 st = lcgAdvance(d.jumpA, d.jumpC, d.ctl->rng, tc.base + (u64)tc.used + 1);
    tc.used += 1;
    return ((st >> 47) & 1ULL) ? o1 : o2;  // Random.nextBoolean() = next(1) != 0
  }
  return b1 >= b2 ? o1 : o2;
}

// reevaluateHead (CasperIMD.java:348-353)
template <class C>
WTG_HD void cReevaluate(const Dev& d, C& c, int n, CTie& tc) {
  u64* tr = d.cToReeval + (size_t)n * d.cBlkWords;
  int head = d.cHead[n];
  for (int w = 0; w < d.cBlkWords && !tc.hit; ++w) {
    u64 bits = tr[w];
    while (bits && !tc.hit) {
      int b = w * 64 + WTG_CTZ64(bits);
      bits &= bits - 1;
      head = cBest(d, c, n, head, b, tc);
    }
  }
  c.sync();
  if (tc.hit) return;  // suspended: nothing written
  if (c.lane() == 0) {
    d.cHead[n] = head;
    for (int w = 0; w < d.cBlkWords; ++w) tr[w] = 0;
  }
  c.sync();
}

// BlockProducer.buildBlock (CasperIMD.java:383-428) + the Block constructor checks (Block.java:38-47).
// Returns the new block's index, -1 on error.
template <class C>
WTG_HD int cBuildBlock(const Dev& d, C& c, int n, int base, int height, int item) {
  const int tick = d.ctl->tick;
  if (height <= 0 || tick < d.cbTime[base] || d.cbHeight[base] >= height) {  // IllegalArgumentException
    setError(d, ERR_PROTO_STATE, 2);
    return -1;
  }
  int nb = 0;
  if (c.lane() == 0) nb = WTG_ATOMIC_ADD(&d.cg->nBlocks, 1);
  nb = c.bcast(nb, 0);
  if (nb >= d.cMaxBlocks) {
    setError(d, ERR_UNSUPPORTED, 2);
    return -1;
  }
  const int lim = height - d.cCycle;
  CMask chain;
  cmaskClear(chain);
  for (int cur = base; cur >= 0 && d.cbHeight[cur] >= lim; cur = d.cbParent[cur]) cmaskSet(chain, cur);  // phase-2 blocks (:410-412)
  const int W = d.cAttWords;
  const u64* recv = d.cAttRecv + (size_t)n * W;
  u64* inc = d.cbIncluded + (size_t)nb * W;
  for (int w = c.lane(); w < W; w += C::LANES) {
    u64 fromBlocks = 0;  // phase 1: already included by our parents (:400-407), genesis excluded
    for (int cur = base; cur > 0 && d.cbHeight[cur] >= lim; cur = d.cbParent[cur]) fromBlocks |= d.cbIncluded[(size_t)cur * W + w];
    u64 cand = recv[w] & ~fromBlocks, out = 0;
    while (cand) {
      int b = WTG_CTZ64(cand);
      cand &= cand - 1;
      int a = w * 64 + b;
      if (cmaskHas(chain, d.attHead[a]) && d.attHeight[a] < height) out |= 1ULL << b;  // :414-423
    }
    inc[w] = out;
    if (d.G > 1)  // the block table is replicated: the creator stores the row into every shard's copy (visible to the
                  // receivers before the block can arrive: the exchange that follows the handlers is a system-scope release)
      for (int q = 0; q < d.G; ++q)
        if (q != d.rank) casperTabsOf(d, q).cbIncluded[(size_t)nb * W + w] = out;
  }
  if (c.lane() == 0) {
    d.cbHeight[nb] = height;
    d.cbParent[nb] = base;
    d.cbProducer[nb] = n;
    d.cbTime[nb] = tick;
    d.cbItem[nb] = item;                        // creating event: ids follow the processing order (casperRenumber)
    WTG_ATOMIC_ADD(&d.cg->createdThisTick, 1);  // see tickEnd
    if (d.G > 1)
      for (int q = 0; q < d.G; ++q)
        if (q != d.rank) {
          CasperTabs t = casperTabsOf(d, q);
          t.cbHeight[nb] = height;
          t.cbParent[nb] = base;
          t.cbProducer[nb] = n;
          t.cbTime[nb] = tick;
          WTG_ATOMIC_ADD(&t.cg->nBlocks, 1);          // the same id everywhere: at most one block per pass (tickEnd checks)
          WTG_ATOMIC_ADD(&t.cg->createdThisTick, 1);
        }
  }
  c.sync();
  return nb;
}

// network.sendAll(msg, sendTime, from): the descriptor; the envelope is built by emitAll
WTG_HD void cWriteSendAll(const Dev& d, int di, int n, int item, int sub, uint32_t meta, u64 pl, int sendTime, int tieDraws = 0) {
  Desc ds;
  ds.dkind = DK_SEND_ALL;
  ds.item = (uint32_t)(d.nLoc + item);
  ds.sub = (uint32_t)sub;
  ds.from = (uint32_t)n;
  ds.to = (uint32_t)tieDraws;  // fork-choice ties drawn by this handler before the send: they come first in the draw order
  ds.nDest = (uint32_t)d.N;
  ds.evKind = EV_MULTI;
  ds.meta = meta;
  ds.pl = pl;
  ds.target = sendTime;
  ds.aux = 0;
  d.desc[di] = ds;
  int ai = WTG_ATOMIC_ADD(&d.ctl->allCnt, 1);
  if (ai < d.allCap)
    d.allList[ai] = di;
  else
    setError(d, ERR_DESC_OVERFLOW, ai);
  d.msgSent[n] += d.N;  // msgSent++ / bytesSent += size() per destination, dropped or not (Network.java:476-477)
  d.bytesSent[n] += d.N;
  statAdd(d, n, ST_MULTISENDS, 1ULL);
}
WTG_HD void cWriteInsert(const Dev& d, int di, int n, int item, int sub, uint32_t evKind, uint32_t meta, u64 pl, int target) {
  Desc ds;
  ds.dkind = DK_INSERT_AT;
  ds.item = (uint32_t)(d.nLoc + item);
  ds.sub = (uint32_t)sub;
  ds.from = (uint32_t)n;
  ds.to = (uint32_t)n;
  ds.nDest = 0;
  ds.evKind = evKind;
  ds.meta = meta;
  ds.pl = pl;
  ds.target = target;
  ds.aux = 0;
  d.desc[di] = ds;
}

// BlockChainNode.onBlock + CasperNode.onBlock + ByzBlockProducerWF.onBlock (BlockChainNode.java:33-49, CasperIMD.java:298-314, 667-701)
template <class C>
WTG_HD void cOnBlock(const Dev& d, C& c, int n, int b, int item, int& slots, int& draws, CTie& tc) {
  const int tick = d.ctl->tick;
  u64* tr = d.cToReeval + (size_t)n * d.cBlkWords;
  u64* br = d.cBlkRecv + (size_t)n * d.cBlkWords;
  const int head = d.cHead[n];
  const bool already = rowBit(br, b);
  c.sync();
  if (c.lane() == 0) {  // delta >= 0 always (:302-306): blocksToReevaluate.add(head); add(b), before the duplicate check
    tr[head >> 6] |= 1ULL << (head & 63);
    tr[b >> 6] |= 1ULL << (b & 63);
  }
  if (already) {
    c.sync();
    return;
  }
  int nh = cBest(d, c, n, head, b, tc);
  if (tc.hit) return;  // suspended (the two marks above are idempotent)
  if (c.lane() == 0) {
    br[b >> 6] |= 1ULL << (b & 63);
    d.cHead[n] = nh;
  }
  c.sync();
  if (d.cKind[n] != CK_BYZ_WF) return;
  const int toSend = d.cg->byzToSend;
  if (d.cbHeight[b] != toSend - 1) return;
  const int perfectDate = CASPER_SLOT * toSend + d.cByzDelay;
  c.sync();
  if (tick >= perfectDate) {  // r.run(); late++ (:689-691)
    int nb = cBuildBlock(d, c, n, b, toSend, item);
    int base = descAlloc(d, c, n, 1);
    if (c.lane() == 0) {
      d.cg->byzToSend = toSend + d.cBpCount;
      d.cg->byzLate += 1;
      if (nb >= 0) d.cHead[n] = nb;
      if (nb >= 0 && base >= 0) cWriteSendAll(d, base, n, item, 0, CM_BLOCK, (u64)(uint32_t)nb, tick + d.cBlockTime, tc.used);
    }
    slots = 1;
    draws = 1;
  } else {  // network.registerTask(r, perfectDate, this); onTime++ (:692-695)
    int base = descAlloc(d, c, n, 1);
    if (c.lane() == 0) {
      d.cg->byzToSend = toSend + d.cBpCount;
      d.cg->byzOnTime += 1;
      if (base >= 0) cWriteInsert(d, base, n, item, 0, EV_TASK, CT_BUILD, (u64)(uint32_t)b | ((u64)(uint32_t)toSend << 32), perfectDate);
    }
    slots = 1;
    draws = 0;
  }
  c.sync();
}

// onAttestation (CasperIMD.java:316-337)
WTG_HD void cOnAttestation(const Dev& d, int n, int a) {
  u64* ar = d.cAttRecv + (size_t)n * d.cAttWords;
  ar[a >> 6] |= 1ULL << (a & 63);
  int hb = d.attHead[a];
  if (rowBit(d.cBlkRecv + (size_t)n * d.cBlkWords, hb)) d.cToReeval[(size_t)n * d.cBlkWords + (hb >> 6)] |= 1ULL << (hb & 63);
}

// blocksReceivedByHeight.get(hh).iterator().next(): the received block of that height with the lowest id, -1 if none
WTG_HD int cFirstAtHeight(const Dev& d, int n, int hh) {
  const u64* br = d.cBlkRecv + (size_t)n * d.cBlkWords;
  for (int w = 0; w < d.cBlkWords; ++w) {
    u64 bits = br[w];
    while (bits) {
      int b = w * 64 + WTG_CTZ64(bits);
      bits &= bits - 1;
      if (b != 0 && d.cbHeight[b] == hh) return b;  // genesis is only in blocksReceivedByBlockId (BlockChainNode.java:26)
    }
  }
  return -1;
}

// periodic tasks: Attester.vote (:455-464), BlockProducer (:376-381, 430-436), ByzBlockProducerWF (:656-665, reevaluateH :529-542)
// followed by the re-arm of PeriodicTask.action (messages/PeriodicTask.java:40-47)
template <class C>
WTG_HD void cPeriodic(const Dev& d, C& c, int n, int item, int& slots, int& draws, CTie& tc) {
  const int tick = d.ctl->tick;
  const int kind = d.cKind[n];
  const int period = casperPeriod(d, kind);
  if (kind == CK_ATTESTER) {
    cReevaluate(d, c, n, tc);
    if (tc.hit) return;
    int k = d.cVotes[n];
    int a = k * d.cAttCount + (n - d.cFirstAtt);
    if (a >= d.cMaxAtts) {
      setError(d, ERR_UNSUPPORTED, 3);
      return;
    }
    int base = descAlloc(d, c, n, 2);
    if (c.lane() == 0 && base >= 0) {
      d.attHead[a] = d.cHead[n];
      d.attHeight[a] = tick / CASPER_SLOT;
      if (d.G > 1)  // replicated attestation table
        for (int q = 0; q < d.G; ++q)
          if (q != d.rank) {
            CasperTabs t = casperTabsOf(d, q);
            t.attHead[a] = d.cHead[n];
            t.attHeight[a] = tick / CASPER_SLOT;
          }
      d.cVotes[n] = k + 1;
      cWriteSendAll(d, base, n, item, 0, CM_ATT, (u64)(uint32_t)a, tick + d.cAttTime, tc.used);
      cWriteInsert(d, base + 1, n, item, 1, EV_PERIODIC, 0, 0, tick + period);
    }
    slots = 2;
    draws = 1;
  } else if (kind == CK_PRODUCER) {
    cReevaluate(d, c, n, tc);
    if (tc.hit) return;
    int nb = cBuildBlock(d, c, n, d.cHead[n], tick / CASPER_SLOT, item);
    int base = descAlloc(d, c, n, 2);
    if (c.lane() == 0 && base >= 0 && nb >= 0) {
      d.cHead[n] = nb;
      cWriteSendAll(d, base, n, item, 0, CM_BLOCK, (u64)(uint32_t)nb, tick + d.cBlockTime, tc.used);
      cWriteInsert(d, base + 1, n, item, 1, EV_PERIODIC, 0, 0, tick + period);
    }
    slots = 2;
    draws = 1;
  } else if (kind == CK_BYZ || kind == CK_BYZ_SF || kind == CK_BYZ_NS) {  // :544-564, 588-603, 617-634
    const int toSend = d.cg->byzToSend;
    cReevaluate(d, c, n, tc);  // reevaluateH (:529-542)
    if (tc.hit) return;
    int head = d.cHead[n];
    while (d.cbHeight[head] >= toSend) head = d.cbParent[head];
    const int h = (tick - d.cByzDelay) / CASPER_SLOT;
    if (h != toSend) {
      setError(d, ERR_PROTO_STATE, 3);
      return;
    }
    int direct = 0, older = 0, notBest = 0, skipped = 0;
    if (kind == CK_BYZ) {
      if (d.cbHeight[head] == h - 1) {
        direct = 1;
      } else {
        older = 1;
        int pf = cFirstAtHeight(d, n, h - 1);
        if (pf < 0) {  // blocksReceivedByHeight.get(h - 1) is null: NullPointerException in the reference
          setError(d, ERR_PROTO_STATE, 6);
          return;
        }
        if (d.cbHeight[d.cbParent[pf]] != h - 1) notBest = 1;
      }
    } else if (kind == CK_BYZ_SF) {
      if (head != 0 && d.cbHeight[head] == h - 1) {
        head = d.cbParent[head];
        direct = 1;
      } else {
        older = 1;
      }
    } else {
      if (head != 0 && d.cbHeight[head] == h - 1 && d.cbHeight[d.cbParent[head]] == h - 3) {
        int b = cFirstAtHeight(d, n, h - 2);
        if (b < 0) {
          setError(d, ERR_PROTO_STATE, 6);
          return;
        }
        head = b;
        skipped = 1;
      }
    }
    c.sync();
    int nb = cBuildBlock(d, c, n, head, toSend, item);
    int base = descAlloc(d, c, n, 2);
    if (c.lane() == 0 && base >= 0 && nb >= 0) {
      d.cg->byzH = h;
      d.cg->byzDirect += direct;
      d.cg->byzOlder += older;
      d.cg->byzNotBest += notBest;
      d.cg->byzSkipped += skipped;
      d.cHead[n] = nb;
      d.cg->byzToSend = toSend + d.cBpCount;
      cWriteSendAll(d, base, n, item, 0, CM_BLOCK, (u64)(uint32_t)nb, tick + d.cBlockTime, tc.used);
      cWriteInsert(d, base + 1, n, item, 1, EV_PERIODIC, 0, 0, tick + period);
    }
    slots = 2;
    draws = 1;
  } else if (kind == CK_BYZ_WF) {
    const int toSend = d.cg->byzToSend;
    if (d.cHead[n] == 0 && toSend == 1) {  // kick off the system (:658-663)
      cReevaluate(d, c, n, tc);
      if (tc.hit) return;
      int head = d.cHead[n];
      while (d.cbHeight[head] >= toSend) head = d.cbParent[head];
      int h = (tick - d.cByzDelay) / CASPER_SLOT;
      if (h != toSend) {  // IllegalStateException (:541)
        setError(d, ERR_PROTO_STATE, 3);
        return;
      }
      c.sync();
      int nb = cBuildBlock(d, c, n, head, h, item);
      int base = descAlloc(d, c, n, 2);
      if (c.lane() == 0 && base >= 0 && nb >= 0) {
        d.cg->byzH = h;
        d.cHead[n] = nb;
        d.cg->byzToSend = toSend + d.cBpCount;
        cWriteSendAll(d, base, n, item, 0, CM_BLOCK, (u64)(uint32_t)nb, tick + d.cBlockTime, tc.used);
        cWriteInsert(d, base + 1, n, item, 1, EV_PERIODIC, 0, 0, tick + period);
      }
      slots = 2;
      draws = 1;
    } else {
      int base = descAlloc(d, c, n, 1);
      if (c.lane() == 0 && base >= 0) cWriteInsert(d, base, n, item, 0, EV_PERIODIC, 0, 0, tick + period);
      slots = 1;
      draws = 0;
    }
  } else {  // the observer has no periodic task
    setError(d, ERR_INTERNAL, 40);
  }
  c.sync();
}

// the Runnable registered by ByzBlockProducerWF.onBlock (:674-686)
template <class C>
WTG_HD void cBuildTask(const Dev& d, C& c, int n, u64 pl, int item, int& slots, int& draws) {
  const int tick = d.ctl->tick;
  int b = (int)(uint32_t)pl, th = (int)(pl >> 32);
  int nb = cBuildBlock(d, c, n, b, th, item);
  int base = descAlloc(d, c, n, 1);
  if (c.lane() == 0 && base >= 0 && nb >= 0) {
    d.cHead[n] = nb;
    cWriteSendAll(d, base, n, item, 0, CM_BLOCK, (u64)(uint32_t)nb, tick + d.cBlockTime);
  }
  slots = 1;
  draws = 1;
  c.sync();
}

// Block.id is a global counter (Block.java:10, 49): two blocks created in the same millisecond get their ids in the order of
// the events that created them.  The parallel handler pass hands the ids out in arbitrary order; this pass (one coop, only when
// more than one block was created) gives the new blocks the ids of the processing order: permutes the new rows of the block
// table and patches what refers to them — the creator's head and the SendBlock descriptors of the pass.
constexpr int CASPER_MAX_NEW = 8;
template <class C>
WTG_HD void casperRenumber(const Dev& d, C& c) {
  const int k = d.cg->createdThisTick;
  if (k <= 1) return;
  if (k > CASPER_MAX_NEW) {
    setError(d, ERR_UNSUPPORTED, 4);
    return;
  }
  const int first = d.cg->nBlocks - k;
  int newId[CASPER_MAX_NEW];
  bool same = true;
  for (int i = 0; i < k; ++i) {
    int r = 0;
    for (int j = 0; j < k; ++j)
      if (d.cbItem[first + j] < d.cbItem[first + i]) ++r;
    newId[i] = first + r;
    same = same && r == i;
  }
  if (same) return;
#if !defined(__CUDA_ARCH__) && defined(WTG_DEBUG_RENUMBER)
  fprintf(stderr, "renumber non-identity k=%d tick=%d\n", k, d.ctl->tick);
#endif
  const int W = d.cAttWords;
  // rows -> scratch (in the new order), then back
  for (int i = 0; i < k; ++i) {
    const int dst = newId[i] - first;
    for (int w = c.lane(); w < W; w += C::LANES) d.cbTmp[(size_t)dst * W + w] = d.cbIncluded[(size_t)(first + i) * W + w];
    if (c.lane() == 0) {
      int* t = d.cbTmpRow + dst * 5;
      t[0] = d.cbHeight[first + i];
      t[1] = d.cbParent[first + i];
      t[2] = d.cbProducer[first + i];
      t[3] = d.cbTime[first + i];
      t[4] = d.cbItem[first + i];
    }
  }
  c.sync();
  for (int i = 0; i < k; ++i) {
    for (int w = c.lane(); w < W; w += C::LANES) d.cbIncluded[(size_t)(first + i) * W + w] = d.cbTmp[(size_t)i * W + w];
    if (c.lane() == 0) {
      const int* t = d.cbTmpRow + i * 5;
      d.cbHeight[first + i] = t[0];
      d.cbParent[first + i] = t[1];
      d.cbProducer[first + i] = t[2];
      d.cbTime[first + i] = t[3];
      d.cbItem[first + i] = t[4];
    }
  }
  c.sync();
  if (c.lane() == 0)
    for (int i = 0; i < k; ++i) {  // the creator adopted its block as head (createAndSendBlock :430-436, ByzBlockProducer* :561, 686)
      const int n = d.cbProducer[newId[i]];
      if (d.cHead[n] == first + i) d.cHead[n] = newId[i];
    }
  // head patches of two creators cannot collide: every creator made exactly one of the new blocks and its head is that block
  const int per = d.descCap / ARENA_STRIPES;
  for (int st = 0; st < ARENA_STRIPES; ++st) {
    int cnt = d.ctl->descCnt[st];
    if (cnt > per) cnt = per;
    for (int j = c.lane(); j < cnt; j += C::LANES) {
      Desc& ds = d.desc[st * per + j];
      if (ds.dkind == DK_SEND_ALL && ds.meta == CM_BLOCK) {
        int b = (int)(uint32_t)ds.pl;
        if (b >= first && b < first + k) ds.pl = (u64)(uint32_t)newId[b - first];
      }
    }
  }
  c.sync();
}

// one event of node n; false: a fork-choice tie was hit in the parallel pass — nothing was written, the node is suspended
template <class C>
WTG_HD bool casperEvent(const Dev& d, C& c, int n, uint32_t evKind, uint32_t meta, u64 pl, int item, int& slots, int& draws, CTie& tc) {
  if (evKind == EV_MSG || evKind == EV_MULTI) {
    if (meta == CM_ATT) {
      if (c.lane() == 0) cOnAttestation(d, n, (int)(uint32_t)pl);
      c.sync();
    } else {
      cOnBlock(d, c, n, (int)(uint32_t)pl, item, slots, draws, tc);
      if (tc.hit) return false;
    }
    if (c.lane() == 0) {
      d.msgReceived[n] += 1;
      d.bytesReceived[n] += 1;  // Message.size() default (messages/Message.java:27-29)
      statAdd(d, n, ST_DELIVERIES, 1ULL);
    }
  } else if (evKind == EV_PERIODIC) {
    cPeriodic(d, c, n, item, slots, draws, tc);
    if (tc.hit) return false;
    if (c.lane() == 0) statAdd(d, n, ST_TASKS, 1ULL);
  } else {
    if (c.lane() == 0) statAdd(d, n, ST_TASKS, 1ULL);
    cBuildTask(d, c, n, pl, item, slots, draws);
  }
  draws += tc.used;
  return true;
}
template <class C>
WTG_HD void casperDeliver(const Dev& d, C& c, int n, uint32_t evKind, uint32_t meta, u64 pl, int item, int& slots, int& draws) {
  if (d.cRandomTies && d.cTieItem[n] >= 0) return;  // suspended earlier in this pass: the tie pass runs the node's later events
  CTie tc;
  tc.resolve = 0;
  tc.base = 0;
  tc.used = 0;
  tc.hit = false;
  if (casperEvent(d, c, n, evKind, meta, pl, item, slots, draws, tc)) return;
  slots = 0;
  draws = 0;
  if (c.lane() == 0) {  // suspend the node at this event
    d.cTieItem[n] = item;
    d.cTieCnt[n] = d.inboxFill[n];
    d.cTieList[WTG_ATOMIC_ADD(&d.ctl->tieCnt, 1)] = n;
  }
  c.sync();
}
// The tie pass (one coop, after the parallel handler pass): repeatedly take the suspended node whose suspended event comes
// first in processing order — every earlier event of the pass is complete, so the number of draws before it is exact — run
// that event with its ties drawn, then the node's later events (a later tie suspends it again, further down the order).
template <class C>
WTG_HD void casperResolveTies(const Dev& d, C& c) {
  Ctl& ctl = *d.ctl;
  const Ev* bucket = d.buckets + (size_t)(ctl.tick & (d.ring - 1)) * (size_t)d.bcap;
  for (;;) {
    const int ns = ctl.tieCnt;
    int bestItem = 0x7fffffff;
    for (int i = c.lane(); i < ns; i += C::LANES) {
      int it = d.cTieItem[d.cTieList[i]];
      if (it >= 0 && it < bestItem) bestItem = it;
    }
    bestItem = c.minv(bestItem);
    if (bestItem == 0x7fffffff) break;
    int n = -1;
    for (int i = c.lane(); i < ns; i += C::LANES)
      if (d.cTieItem[d.cTieList[i]] == bestItem) n = d.cTieList[i];
    n = c.maxv(n);
    int sum = 0;  // draws of every event processed before bestItem
    for (int it = c.lane(); it < bestItem; it += C::LANES) sum += d.evDraws[it];
    const u64 base = (u64)(uint32_t)c.sum(sum);
    const int cnt = d.cTieCnt[n];
    const u64* in = d.inbox + d.inboxOff[n];
    c.sync();
    if (c.lane() == 0) d.cTieItem[n] = -1;
    c.sync();
    int lastItem = bestItem - 1;
    bool first = true;
    for (;;) {  // the node's events from the suspended one on, in processing order
      int nxt = 0x7fffffff;
      u64 w = 0;
      for (int i = 0; i < cnt; ++i) {  // inboxes are tiny
        int it = inboxItem(in[i]);
        if (it > lastItem && it < nxt) {
          nxt = it;
          w = in[i];
        }
      }
      if (nxt == 0x7fffffff) break;
      lastItem = nxt;
      const Ev ev = bucket[inboxEntry(w)];
      uint32_t meta = ev.meta;
      u64 pl = ev.pl;
      if (ev.kind == EV_MULTI) {
        const MultiRec& rc = d.rec[ev.aux];
        meta = rc.meta;
        pl = rc.pl;
      }
      int slots = 0, draws = 0;
      const bool isTask = ev.kind == EV_TASK || ev.kind == EV_PERIODIC;
      const uint32_t envFrom = isTask ? (uint32_t)n : (ev.kind == EV_MULTI ? d.rec[ev.aux].from : ev.from);
      bool done = true;
      if (!d.ndown[n] && d.npart[envFrom] == d.npart[n]) {  // Network.java:606 (as in deliver())
        CTie tc;
        tc.resolve = first ? 1 : 0;
        tc.base = base;
        tc.used = 0;
        tc.hit = false;
        done = casperEvent(d, c, n, ev.kind, meta, pl, nxt, slots, draws, tc);
      }
      if (!done) {  // a later event of the node ties as well: its draw index depends on the events in between
        if (c.lane() == 0) d.cTieItem[n] = nxt;
        c.sync();
        break;
      }
      if (c.lane() == 0) {
        d.evSlots[nxt] = slots;
        d.evDraws[nxt] = draws;
      }
      c.sync();
      first = false;
    }
  }
}

// ------------------------------------------------------------------------------------------
// sendAll emission: one coop per descriptor.  createMessageArrivals (Network.java:449-467): arrival per destination
// in allNodes order, stable sort by arrival; MultipleDestEnvelope over the survivors (:435-446).
//   tmp  [N]        unsorted arrivals (scratch private to the coop)
//   hist [ALL_HIST] counters private to the coop (shared memory on the device)
// ------------------------------------------------------------------------------------------
constexpr int ALL_HIST = 1024;
// `seq` < 0: record slot from the engine's own counter (one engine = the whole network).  `seq` >= 0 (node-sharded run): the
// sendAll's global sequence number — every shard builds the identical record in slot seq % recSlots and keeps the bucket
// entry of the first group only when it owns one of that group's destinations.
template <class C>
WTG_HD void emitAllCore(const Dev& d, C& c, uint32_t fromU, uint32_t meta, u64 pl, int sendTime, int g, u64 drawIdx, int seq, int* tmp, int* hist) {
  const Ctl& ctl = *d.ctl;
  const int N = d.N;
  const bool shard = seq >= 0;
  if (g >= d.newEvCap) {
    setError(d, ERR_DESC_OVERFLOW, g);
    return;
  }
  const int32_t seed = lcgNextIntAt(d, ctl.rng, drawIdx);
  const int from = (int)fromU;
  const bool fromOk = !d.ndown[from];
  int mn = 0x7fffffff, mx = -1, cnt = 0;
  for (int to = c.lane(); to < N; to += C::LANES) {
    int a = -1;
    if (fromOk && d.npart[from] == d.npart[to] && !d.ndown[to]) {  // createMessageArrival :478-484
      int nt = latency(d, from, to, pseudoRandom(to, seed));
      if (nt < d.msgDiscardTime) a = sendTime + nt;
    }
    tmp[to] = a;
    if (a >= 0) {
      mn = a < mn ? a : mn;
      mx = a > mx ? a : mx;
      ++cnt;
    }
  }
  mn = c.minv(mn);
  mx = c.maxv(mx);
  cnt = c.sum(cnt);
  c.sync();
  Ev ev;
  ev.kind = EV_MULTI;
  ev.to = 0;
  ev.from = fromU;
  ev.meta = meta;
  ev.pl = pl;
  ev.aux = 0;
  ev.pad = (uint32_t)sendTime + 1u;  // sendAll(msg, sendTime, from): EnvelopeInfo.sentAt + 1
  int target = -1;
  if (cnt == 1) {  // SingleDestEnvelope
    for (int to = c.lane(); to < N; to += C::LANES)
      if (tmp[to] >= 0 && (!shard || ownerOf(d, to) == d.rank)) {
        ev.kind = EV_MSG;
        ev.to = (uint32_t)to;
        target = tmp[to];
        d.newEv[g] = ev;
        d.newTarget[g] = target - ctl.tick >= d.ring ? -1 : target;
        if (target - ctl.tick >= d.ring) setError(d, ERR_FAR_FUTURE, target);
      }
    return;
  }
  bool keep = true;  // this engine holds the bucket entry of the first group
  if (cnt > 1) {
    int ri = 0, samePass = 0;
    if (shard)
      ri = (int)((unsigned)seq % (unsigned)d.recSlots);
    else if (c.lane() == 0) {
      const unsigned raw = (unsigned)WTG_ATOMIC_ADD(&d.ctl->recTop, 1);
      ri = (int)(raw % (unsigned)d.recSlots);
      // an earlier sendAll of this pass took the slot: the warps emit in parallel, so its record may not be written yet
      samePass = raw - (unsigned)ctl.allRecBase >= (unsigned)d.recSlots;
    }
    ri = c.bcast(ri, 0);
    samePass = c.bcast(samePass, 0);
    MultiRec old = d.rec[ri];
    // the slot still holds a live envelope?  (replicated records: the cursor lives in the bucket entries, so a slot is
    // free once its last arrival has been processed)
    const bool live = samePass || (shard ? (old.n > 0 && d.recArrival[old.off + old.n - 1] > ctl.tick) : (old.cur < old.n));
    if (live) {
      setError(d, ERR_REC_OVERFLOW, ri);
      cnt = 0;
    } else {
      const int off = ri * N;
      int placed = 0;
      for (int base = mn; base <= mx; base += ALL_HIST) {
        for (int b = c.lane(); b < ALL_HIST; b += C::LANES) hist[b] = 0;
        c.sync();
        for (int to = c.lane(); to < N; to += C::LANES) {
          int a = tmp[to];
          if (a >= base && a < base + ALL_HIST) WTG_ATOMIC_ADD(&hist[a - base], 1);
        }
        c.sync();
        int run = placed;  // exclusive prefix over the arrival bins
        for (int b0 = 0; b0 < ALL_HIST; b0 += C::LANES) {
          int total;
          hist[b0 + c.lane()] = run + c.exclusiveScan(hist[b0 + c.lane()], total);
          run += total;
        }
        c.sync();
        for (int to0 = 0; to0 < N; to0 += C::LANES) {  // stable: destinations in id order, LANES at a time
          int to = to0 + c.lane();
          int a = to < N ? tmp[to] : -1;
          bool in = a >= base && a < base + ALL_HIST;
          int pos = c.claim(hist, a - base, in);
          if (in) {
            d.recDest[off + pos] = (uint32_t)to;
            d.recArrival[off + pos] = a;
          }
          c.sync();
        }
        placed = run;
      }
      if (c.lane() == 0) {
        MultiRec rc;
        rc.from = fromU;
        rc.meta = meta;
        rc.pl = pl;
        rc.n = (uint32_t)cnt;
        rc.cur = 0;
        rc.off = (uint32_t)off;
        rc.pad = (uint32_t)sendTime + 1u;
        d.rec[ri] = rc;
      }
      c.sync();
      ev.to = d.recDest[off];
      ev.aux = (uint32_t)ri;
      target = mn;
      if (shard) {  // first destination of the first group that this shard owns (none: another shard holds the entry)
        int first = 0x7fffffff;
        for (int j0 = 0; j0 < cnt; j0 += C::LANES) {
          int j = j0 + c.lane();
          bool inGroup = j < cnt && d.recArrival[off + j] == mn;
          if (inGroup && ownerOf(d, (int)d.recDest[off + j]) == d.rank && j < first) first = j;
          if (!c.any(inGroup)) break;
        }
        first = c.minv(first);
        keep = first != 0x7fffffff;
        if (keep) ev.to = d.recDest[off + first];
        ev.meta = 0;
        ev.pl = 0;  // index of the group's first destination (multiCur)
      }
    }
  }
  if (c.lane() == 0) {
    if (target >= 0 && target - ctl.tick >= d.ring) {
      setError(d, ERR_FAR_FUTURE, target);
      target = -1;
    }
    if (!shard) {
      d.newEv[g] = ev;
      d.newTarget[g] = target;
    } else if (keep && target >= 0) {
      d.newEv[g] = ev;
      d.newTarget[g] = target;
    }
  }
}
template <class C>
WTG_HD void emitAll(const Dev& d, C& c, int di, int* tmp, int* hist) {
  const Desc ds = d.desc[di];
  const int g = d.slotBase[ds.item] + (int)ds.sub;
  const u64 drawIdx = (u64)(d.drawBase[ds.item] + (int)ds.sub) + (u64)ds.to;  // ds.to: fork-choice ties the handler drew first
  emitAllCore(d, c, ds.from, ds.meta, ds.pl, ds.target, g, drawIdx, -1, tmp, hist);
}
// node-sharded: publish this shard's j-th sendAll of the pass (global creation / draw index) into every shard's list ...
WTG_HD void xPublishAll(const Dev& d, int j) {
  const Desc ds = d.desc[d.allList[j]];
  XAll a;
  a.from = ds.from;
  a.meta = ds.meta;
  a.pl = ds.pl;
  a.sendTime = ds.target;
  a.g = d.slotBase[ds.item] + (int)ds.sub + (int)d.xoffS[ds.item - d.nLoc];
  a.draw = (u64)(d.drawBase[ds.item] + (int)ds.sub) + (u64)ds.to + (u64)d.xoffD[ds.item - d.nLoc];
  for (int q = 0; q < d.G; ++q) d.peer[q].all[(size_t)d.rank * d.xAllCap + j] = a;
}
WTG_HD void xPublishAllCount(const Dev& d) {
  int cnt = d.ctl->error ? 0 : d.ctl->allCnt;
  if (cnt > d.xAllCap) {
    setError(d, ERR_DESC_OVERFLOW, cnt);
    cnt = 0;
  }
  for (int q = 0; q < d.G; ++q) d.peer[q].allCnt[d.rank] = cnt;
}
// ... and, after the envelope exchange, build the k-th sendAll of the pass over all shards (shard-major order)
WTG_HD int xAllTotal(const Dev& d) {
  int tot = 0;
  for (int q = 0; q < d.G; ++q) tot += d.peer[d.rank].allCnt[q];
  return tot;
}
template <class C>
WTG_HD void xBuildAll(const Dev& d, C& c, int k, int* tmp, int* hist) {
  int q = 0, i = k;
  while (q < d.G && i >= d.peer[d.rank].allCnt[q]) {
    i -= d.peer[d.rank].allCnt[q];
    ++q;
  }
  if (q >= d.G) return;
  const XAll a = d.peer[d.rank].all[(size_t)q * d.xAllCap + i];
  emitAllCore(d, c, a.from, a.meta, a.pl, a.sendTime, a.g, a.draw, (int)(((unsigned)d.ctl->allSeq + (unsigned)k) & 0x3fffffffu), tmp, hist);
}

// ------------------------------------------------------------------------------------------
// far-future calendar: envelopes that arrive at least ring/2 ms after they were created
// ------------------------------------------------------------------------------------------
WTG_HD int farHorizon(const Dev& d) { return d.ring >> 1; }
WTG_HD bool farAppend(const Dev& d, const Ev& ev, int target, int g) {
  int fi = WTG_ATOMIC_ADD(&d.ctl->farCnt, 1);
  if (fi >= d.farCap) {
    setError(d, ERR_FAR_OVERFLOW, fi);
    return false;
  }
  FarEv f;
  f.ev = ev;
  f.target = target;
  f.pad = 0;
  // insertion order among far envelopes; node-sharded: the ordering key of the bucket entry it becomes (wtg_shard.cuh)
  f.key = d.G > 1 ? orderKey((unsigned)d.ctl->xseq, (unsigned)g) : (((u64)(uint32_t)d.ctl->tick << 32) | (u64)(uint32_t)g);
  d.far[fi] = f;
  WTG_ATOMIC_MIN(&d.ctl->farMin, target);
  return true;
}

// Move the far envelopes that arrive within the horizon of tick `t` to the head of their buckets, in insertion order.
// Every envelope created from now on for those buckets is inserted after them, like in the reference's per-ms lists.
template <class C>
WTG_HD void farMigrate(const Dev& d, C& c, int t) {
  Ctl& ctl = *d.ctl;
  const int limit = t + farHorizon(d) - 1;
  if (ctl.farMin > limit) return;
  // farAppend keeps counting past farCap once the calendar has overflowed (the error is final): read only what it holds
  const int cnt = ctl.farCnt < d.farCap ? ctl.farCnt : d.farCap;
  int nsel = 0;
  for (int i0 = 0; i0 < cnt; i0 += C::LANES) {
    int i = i0 + c.lane();
    bool sel = i < cnt && d.far[i].target <= limit;
    uint32_t m = c.ballot(sel);
    if (sel) d.farSel[nsel + c.rank(m)] = i;
    nsel += c.count(m);
  }
  c.sync();
  for (int s = c.lane(); s < nsel; s += C::LANES) {
    const FarEv e = d.far[d.farSel[s]];
    int rank = 0;
    for (int s2 = 0; s2 < nsel; ++s2) {
      const FarEv& o = d.far[d.farSel[s2]];
      if (o.target == e.target && o.key < e.key) ++rank;
    }
    int slot = e.target & (d.ring - 1);
    int pos = d.bucketCount[slot] + rank;
    if (pos < d.bcap) {
      d.buckets[(size_t)slot * (size_t)d.bcap + pos] = e.ev;
      if (d.G > 1) d.bucketKey[(size_t)slot * (size_t)d.bcap + pos] = e.key;
    } else
      setError(d, ERR_BUCKET_OVERFLOW, e.target);
  }
  c.sync();
  for (int s = c.lane(); s < nsel; s += C::LANES) {
    FarEv& e = d.far[d.farSel[s]];
    WTG_ATOMIC_ADD(&d.bucketCount[e.target & (d.ring - 1)], 1);
    e.target = -1;
  }
  c.sync();
  // compact the list in place (the order of the survivors is irrelevant: the key carries it) and refresh farMin
  int kept = 0, mn = 0x7fffffff;
  for (int i0 = 0; i0 < cnt; i0 += C::LANES) {
    int i = i0 + c.lane();
    FarEv e;
    bool live = false;
    if (i < cnt) {
      e = d.far[i];
      live = e.target >= 0;
    }
    uint32_t m = c.ballot(live);
    c.sync();
    if (live) {
      d.far[kept + c.rank(m)] = e;
      mn = e.target < mn ? e.target : mn;
    }
    kept += c.count(m);
    c.sync();
  }
  mn = c.minv(mn);
  if (c.lane() == 0) {
    ctl.farCnt = kept;
    ctl.farMin = mn;
  }
  c.sync();
}

// first non-empty bucket in (from, from + span], or INT_MAX
template <class C>
WTG_HD int ringNextNonEmpty(const Dev& d, C& c, int from, int span) {
  int best = 0x7fffffff;
  for (int b0 = 1; b0 <= span && best == 0x7fffffff; b0 += C::LANES) {
    int b = b0 + c.lane();
    int v = (b <= span && d.bucketCount[(from + b) & (d.ring - 1)] > 0) ? from + b : 0x7fffffff;
    best = c.minv(v);
  }
  return best;
}

// tickBegin for fast-forwarding protocols (no conditional tasks): the tick is the next millisecond of the window
// that has something to run; when there is none the window goes idle and the clock jumps to `until`.
template <class C>
WTG_HD void tickBeginFfwd(const Dev& d, C& c) {
  Ctl& ctl = *d.ctl;
  const int time = ctl.time, until = ctl.until;
  const int H = farHorizon(d);
  if (c.lane() == 0) {  // per-pass counters first: in a node-sharded run the other shards' handlers of this pass (which start
                        // after the begin exchange below) store into some of them
    for (int t = 0; t < ARENA_STRIPES; ++t) {
      ctl.descCnt[t] = 0;
      ctl.destCnt[t] = 0;
      ctl.workCnt[t] = 0;
      ctl.dueCnt[t] = 0;
      ctl.taskCnt[t] = 0;
    }
    ctl.nItems = 0;
    ctl.totalSlots = 0;
    ctl.totalDraws = 0;
    ctl.hReject = 0;
    ctl.allCnt = 0;
    ctl.allRecBase = ctl.recTop;
    ctl.shufReject = 0;
    ctl.peerCnt = 0;
    if (d.cg) d.cg->createdThisTick = 0;
    ctl.tieCnt = 0;
    if (d.G > 1) {
      ctl.xseq += 1;
      ctl.nEvGlobal = 0;
      for (int q = 0; q < MAX_SHARDS; ++q) ctl.stageTop[q] = 0;
    }
  }
  c.sync();
  int span = until - time;
  if (span > H - 1) span = H - 1;
  int next = 0x7fffffff;
  if (!ctl.idle && span > 0) next = ringNextNonEmpty(d, c, time, span);
  if (!ctl.idle && ctl.farMin <= until && ctl.farMin < next) next = ctl.farMin;
  c.sync();
  int after = 0x7fffffff;
  if (d.G > 1) {  // the next event of the whole network: minimum over the shards (every shard takes the same decision)
    if (!ctl.idle && next > until) {
      after = ringNextNonEmpty(d, c, time, H - 1);
      if (ctl.farMin < after) after = ctl.farMin;
    }
    c.sync();
    if (c.lane() == 0) {
      int gn = next, ga = after;
      xBeginExchange(d, next, after, gn, ga);
      ctl.xNext = gn;
      ctl.xAfter = ga;
    }
    c.sync();
    next = ctl.xNext;
    after = ctl.xAfter;
    if (ctl.error) return;
  }
  if (next > until) {  // nothing before the end of the window
    if (d.G == 1 && !ctl.idle) {
      after = ringNextNonEmpty(d, c, time, H - 1);
      if (ctl.farMin < after) after = ctl.farMin;
    }
    c.sync();
    if (c.lane() == 0) {
      if (!ctl.idle) ctl.nextEvent = after;
      ctl.idle = 1;
      ctl.time = until;
      ctl.tick = until;
      ctl.condMode = 0;
      ctl.nEv = 0;
    }
  } else {
    farMigrate(d, c, next);
    if (c.lane() == 0) {
      ctl.time = next;
      ctl.tick = next;
      ctl.condMode = 0;
      ctl.nEv = d.bucketCount[next & (d.ring - 1)];
      if (ctl.nEv > ctl.maxBucket) ctl.maxBucket = ctl.nEv;
    }
  }
  c.sync();
}

}  // namespace wtg
