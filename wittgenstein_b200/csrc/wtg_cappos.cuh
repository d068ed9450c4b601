// wittgenstein_b200 — SanFerminCappos handlers (protocols/SanFerminCappos.java, SanFerminHelper.java) and the k-element
// Collections.shuffle that precedes its multi-sends.  Included by wtg_logic.cuh.  Scalar like SanFerminSignature: per-node
// state is a few ints, the per-level maximum of signatureCache, and the helper's usedNodes bitmap of the current level.
#pragma once

namespace wtg {

// java.util.Random.nextInt(bound) at stream position `idx` after state `s0` (idx = 0: next draw); `used` counts the values
// consumed (more than one when the rejection loop fires)
WTG_HD int javaNextIntAt(const u64* jumpA, const u64* jumpC, u64 s0, u64 idx, int bound, int& used) {
  u64 st = lcgAdvance(jumpA, jumpC, s0, idx);
  used = 0;
  for (;;) {
    st = (st * 0x5DEECE66DULL + 0xBULL) & LCG_MASK;
    ++used;
    int32_t u = (int32_t)(uint32_t)(st >> 17);  // next(31)
    if ((bound & (bound - 1)) == 0) return (int)(((long long)bound * (long long)u) >> 31);
    int32_t r = u % bound;
    if ((int32_t)((uint32_t)u - (uint32_t)r + (uint32_t)(bound - 1)) >= 0) return r;
  }
}
// Collections.shuffle(list, rnd): for (i = size; i > 1; i--) swap(list, i - 1, rnd.nextInt(i)).  list == nullptr only counts.
// Returns the number of stream values consumed.
WTG_HD int javaShuffleAt(const u64* jumpA, const u64* jumpC, u64 s0, u64 idx, uint32_t* list, int m) {
  int consumed = 0;
  for (int i = m; i > 1; --i) {
    int used = 0;
    int r = javaNextIntAt(jumpA, jumpC, s0, idx + (u64)consumed, i, used);
    consumed += used;
    if (list) {
      uint32_t t = list[i - 1];
      list[i - 1] = list[r];
      list[r] = t;
    }
  }
  return consumed;
}
// nextInt(bound) on the LCG state `st` (advanced in place); `consumed` counts the values drawn
WTG_HD int javaNextIntStep(u64& st, int bound, int& consumed) {
  for (;;) {
    st = (st * 0x5DEECE66DULL + 0xBULL) & LCG_MASK;
    ++consumed;
    int32_t u = (int32_t)(uint32_t)(st >> 17);  // next(31)
    if ((bound & (bound - 1)) == 0) return (int)(((long long)bound * (long long)u) >> 31);
    int32_t r = u % bound;
    if ((int32_t)((uint32_t)u - (uint32_t)r + (uint32_t)(bound - 1)) >= 0) return r;
  }
}
// Slush / Snowflake randomRemotes() (Slush.java:126-137, Snowflake.java:136-147) from stream position `idx` after state `s0`:
// one nextInt(n) per attempt until k distinct ids other than `self` are drawn, kept in draw order in `list`.  With
// list == nullptr it only counts, without scratch memory: an id drawn before that is not the sender's was kept then (or
// repeated a kept one), so ArrayList.contains is "drawn before", found by replaying the attempts.  Returns the number of
// stream values consumed: k when no attempt hits the sender or repeats an id and no nextInt rejects.  The caller
// guarantees 1 <= k <= min(n - 1, SHUFFLE_MAX - 1).
WTG_HD int javaSampleAt(const u64* jumpA, const u64* jumpC, u64 s0, u64 idx, int self, int n, int k, uint32_t* list) {
  const u64 st0 = lcgAdvance(jumpA, jumpC, s0, idx);
  u64 st = st0;
  int consumed = 0, cnt = 0;
  while (cnt < k) {
    const int before = consumed;
    const int r = javaNextIntStep(st, n, consumed);
    if (r == self) continue;
    bool seen = false;  // ArrayList.contains
    if (list) {
      for (int i = 0; i < cnt; ++i) seen |= list[i] == (uint32_t)r;
    } else {
      u64 s2 = st0;
      for (int c2 = 0; c2 < before && !seen;) seen = javaNextIntStep(s2, n, c2) == r;
    }
    if (seen) continue;
    if (list) list[cnt] = (uint32_t)r;
    ++cnt;
  }
  return consumed;
}

// SanFerminHelper.pickNextNodes(level, howMany) :123-157 without the shuffle (the emit step performs it): writes the new
// list to `out` (at most howMany + 1 entries), returns its length.  usedNodes indices are the reference's raw ints: the
// node's own position, then positions in the candidate list *after* the removal of that position.
WTG_HD int cpPickNextNodes(const Dev& d, int n, int level, uint32_t* out) {
  const int shift = d.sfP - 1 - level;
  const int S = 1 << shift;
  const int ownMin = (n >> shift) << shift;
  const int candMin = ownMin ^ S;
  const int idx = n - ownMin;
  u64* used = d.sfUsedBits + (size_t)n * d.sfUsedWords;
  int cnt = 0;
  bool removed = false;
  if (!((used[idx >> 6] >> (idx & 63)) & 1ULL)) {
    out[cnt++] = (uint32_t)(candMin + idx);
    removed = true;
    used[idx >> 6] |= 1ULL << (idx & 63);
  }
  const int size = removed ? S - 1 : S;
  int taken = 0;
  for (int w = 0; w * 64 < size && taken < d.sfCandCount; ++w) {
    u64 freeBits = ~used[w];
    while (freeBits && taken < d.sfCandCount) {
      int b = WTG_CTZ64(freeBits);
      freeBits &= freeBits - 1;
      int i = w * 64 + b;
      if (i >= size) break;
      used[w] |= 1ULL << b;
      out[cnt++] = (uint32_t)(removed ? (i < idx ? candMin + i : candMin + i + 1) : candMin + i);
      ++taken;
    }
  }
  return cnt;
}

struct CpEmit {  // what a handler asks for, in program order: an optional reply, an optional shuffled multi-send, one task
  bool reply;
  uint32_t replyTo, replyMeta;
  u64 replyPl;
  int nSend;      // destinations of the swap request (in `list`)
  uint32_t list[SHUFFLE_MAX];
  u64 sendPl;
  bool task;
  uint32_t taskMeta;
  u64 taskPl;
  int taskAt;
};

WTG_HD int cpTotalSigs(const Dev& d, int n, int level) {  // totalNumberOfSigs :351-358
  uint32_t mask = d.sfCacheMask[n];
  int sum = 0;
  for (int l = level < 0 ? 0 : level; l < 32; ++l)
    if ((mask >> l) & 1u) sum += d.sfCache[(size_t)n * 32 + l];
  return sum + 1;
}
WTG_HD void cpPutCachedSig(const Dev& d, int n, int level, int value) {  // :382-393
  int* c = &d.sfCache[(size_t)n * 32 + level];
  if (!((d.sfCacheMask[n] >> level) & 1u) || value > *c) *c = value;  // only max(list) is ever read
  d.sfCacheMask[n] |= 1u << level;
  if (cpTotalSigs(d, n, d.sfCpl[n]) >= d.sfThreshold && !(d.sfFlags[n] & 4)) {
    d.sfFlags[n] |= 4;
    d.sfThresholdAt[n] = d.ctl->tick + d.sfPairing * 2;
  }
}
WTG_HD void cpTryNextNodes(const Dev& d, int n, int cnt, CpEmit& em) {  // :248-296 (the list is already in em.list)
  if (cnt == 0) return;
  const int cpl = d.sfCpl[n];
  em.nSend = cnt;
  em.sendPl = sfPl(cpl, cpTotalSigs(d, n, cpl + 1));
  em.task = true;
  em.taskMeta = CP_T_TIMEOUT;
  em.taskPl = sfPl(cpl, 0);
  em.taskAt = d.ctl->tick + d.sfTimeout;
}
WTG_HD void cpGoNextLevel(const Dev& d, int n, CpEmit& em) {  // :306-344 (the recursion over cached levels is a loop)
  const int tick = d.ctl->tick;
  for (;;) {
    int fl = d.sfFlags[n];
    if (fl & 2) return;
    int cpl = d.sfCpl[n];
    if (cpTotalSigs(d, n, cpl) >= d.sfThreshold && !(fl & 4)) {
      fl |= 4;
      d.sfThresholdAt[n] = tick + d.sfPairing * 2;
    }
    if (cpl == 0) {
      d.doneAt[n] = tick + d.sfPairing * 2;
      fl |= 2;
      d.sfFlags[n] = fl;
      return;
    }
    --cpl;
    d.sfCpl[n] = cpl;
    fl &= ~1;
    d.sfFlags[n] = fl;
    {  // usedNodes of a level that was never picked from is a fresh BitSet
      u64* used = d.sfUsedBits + (size_t)n * d.sfUsedWords;
      int words = ((1 << (d.sfP - 1 - cpl)) + 63) / 64;
      for (int w = 0; w < words; ++w) used[w] = 0;
    }
    if ((d.sfCacheMask[n] >> cpl) & 1u) continue;  // a value for the new level is already cached: go on directly
    int cnt = cpPickNextNodes(d, n, cpl, em.list);
    cpTryNextNodes(d, n, cnt, em);
    return;
  }
}

WTG_HD void cpHandle(const Dev& d, int n, uint32_t from, uint32_t type, u64 pl, int item, int& outSlots, int& outDraws) {
  CpEmit em;
  em.reply = false;
  em.replyTo = em.replyMeta = 0;
  em.replyPl = 0;
  em.nSend = 0;
  em.sendPl = 0;
  em.task = false;
  em.taskMeta = 0;
  em.taskPl = 0;
  em.taskAt = 0;
  const int level = (int)(uint32_t)pl, val = (int)(uint32_t)(pl >> 32);
  const int msgBytes = 4 + d.sfSigSize;
  const int tick = d.ctl->tick;
  if (type == CP_SWAP || type == CP_SWAP_REPLY) {
    d.msgReceived[n] += 1;
    d.bytesReceived[n] += msgBytes;
    statAdd(d, n, ST_DELIVERIES, 1ULL);
  } else {
    statAdd(d, n, ST_TASKS, 1ULL);
  }
  const int fl = d.sfFlags[n], cpl = d.sfCpl[n];
  switch (type) {
    case CP_SWAP:          // wantReply == true
    case CP_SWAP_REPLY: {  // wantReply == false
      const bool wantReply = type == CP_SWAP;
      if ((fl & 2) || level != cpl) {  // onSwap :203-223
        bool cached = level >= 0 && level < 32 && ((d.sfCacheMask[n] >> level) & 1u);
        if (wantReply && cached) {
          em.reply = true;
          em.replyTo = from;
          em.replyMeta = CP_SWAP_REPLY;
          em.replyPl = sfPl(level, d.sfCache[(size_t)n * 32 + level]);  // getBestCachedSig
        } else if (level >= 0 && level < 32 && sfIsCandidate(d, n, (int)from, level)) {
          cpPutCachedSig(d, n, level, val);
        }
        break;
      }
      if (wantReply) {  // :225-228
        em.reply = true;
        em.replyTo = from;
        em.replyMeta = CP_SWAP_REPLY;
        em.replyPl = sfPl(level, cpTotalSigs(d, n, level));
      }
      if (sfIsCandidate(d, n, (int)from, cpl) && !(fl & 1)) {  // transition :364-374
        d.sfFlags[n] |= 1;
        em.task = true;
        em.taskMeta = CP_T_TRANSITION;
        em.taskPl = sfPl(level, val);
        em.taskAt = tick + d.sfPairing;
      }
      break;
    }
    case CP_T_GO:
      cpGoNextLevel(d, n, em);
      break;
    case CP_T_TIMEOUT:  // :281-295
      if (!(fl & 2) && cpl == level) {
        int cnt = cpPickNextNodes(d, n, cpl, em.list);
        cpTryNextNodes(d, n, cnt, em);
      }
      break;
    case CP_T_TRANSITION:
      cpPutCachedSig(d, n, level, val);
      cpGoNextLevel(d, n, em);
      break;
    default:
      break;
  }
  const int nd = (em.reply ? 1 : 0) + (em.nSend > 0 ? 1 : 0) + (em.task ? 1 : 0);
  outSlots = nd;
  outDraws = (em.reply ? 1 : 0) + (em.nSend > 0 ? em.nSend : 0);  // shuffle: nSend - 1 draws, then the send's seed
  if (nd == 0) return;
  CoopSerial cs;
  int base = descAlloc(d, cs, n, nd);
  if (base < 0) return;
  int sub = 0;
  auto fill = [&](Desc& ds) {
    ds.item = (uint32_t)(d.nLoc + item);
    ds.sub = (uint32_t)sub;
    ds.from = (uint32_t)n;
    ds.target = 0;
    ds.aux = 0;
  };
  if (em.reply) {
    Desc ds;
    fill(ds);
    ds.dkind = DK_SEND_SINGLE;
    ds.to = em.replyTo;
    ds.nDest = 1;
    ds.evKind = EV_MSG;
    ds.meta = em.replyMeta;
    ds.pl = em.replyPl;
    d.desc[base + sub] = ds;
    ++sub;
    d.msgSent[n] += 1;
    d.bytesSent[n] += msgBytes;
  }
  if (em.nSend > 0) {
    Desc ds;
    fill(ds);
    ds.evKind = EV_MSG;
    ds.meta = CP_SWAP;
    ds.pl = em.sendPl;
    if (em.nSend == 1) {
      ds.dkind = DK_SEND_SINGLE;
      ds.to = em.list[0];
      ds.nDest = 1;
    } else {
      int off = destAlloc(d, n, 2 * em.nSend);  // destinations, then room for their arrivals
      if (off >= 0)
        for (int i = 0; i < em.nSend; ++i) d.destScratch[off + i] = em.list[i];
      ds.dkind = DK_SEND_MULTI;
      ds.to = (uint32_t)(off < 0 ? 0 : off);
      ds.nDest = off < 0 ? 0u : (uint32_t)em.nSend;
      ds.aux = DESC_SHUFFLEK;
    }
    d.desc[base + sub] = ds;
    ++sub;
    d.msgSent[n] += em.nSend;
    d.bytesSent[n] += (long long)em.nSend * msgBytes;
    statAdd(d, n, ST_SENDS, (unsigned long long)em.nSend);
  }
  if (em.task) {
    Desc ds;
    fill(ds);
    ds.dkind = DK_INSERT_AT;
    ds.to = (uint32_t)n;
    ds.nDest = 0;
    ds.evKind = EV_TASK;
    ds.meta = em.taskMeta;
    ds.pl = em.taskPl;
    ds.target = em.taskAt;
    d.desc[base + sub] = ds;
    ++sub;
  }
}

// ------------------------------------------------------------------------------------------
// draw bookkeeping of shuffled and sampled sends.  A descriptor's first draw sits at drawBase[item] + (draws of the event's
// earlier descriptors); a shuffle consumes max(nDest, 1) draws with its seed (a send to an empty list still draws its seed,
// Network.java:430), a sample nDest + 1 — unless nextInt's rejection loop fires or an attempt of a sample is discarded
// somewhere in the tick, which shifts every later draw: then shuffleSerial re-derives all draw indices of the tick in
// creation order.
// ------------------------------------------------------------------------------------------
WTG_HD int descDrawsNominal(const Desc& ds) {
  if (ds.dkind == DK_INSERT_AT) return 0;
  if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SHUFFLEK)) return ds.nDest > 0 ? (int)ds.nDest : 1;
  if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SAMPLEK)) return (int)ds.nDest + 1;
  if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SHUFFLE2)) return 2;
  return 1;
}
// first draw index of descriptor di under the no-rejection assumption: the event's earlier descriptors are found by
// their sub index (an event emits at most three descriptors here: reply, shuffled send, task)
WTG_HD u64 descDrawOptimistic(const Dev& d, int di) {
  const Desc& ds = d.desc[di];
  u64 idx = (u64)d.drawBase[ds.item];
  for (int k = 1; k <= (int)ds.sub; ++k) idx += (u64)descDrawsNominal(d.desc[di - k]);  // same event: contiguous, in sub order
  return idx;
}
WTG_HD void shuffleCheck(const Dev& d, int di) {
  const Desc& ds = d.desc[di];
  int g = d.slotBase[ds.item] + (int)ds.sub;
  if (g < d.newEvCap) {
    d.byG[g] = di;
    d.byGTick[g] = d.ctl->tick;
  }
  if (d.forceShufSerial) d.ctl->shufReject = 1;
  if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SHUFFLEK)) {
    int consumed = javaShuffleAt(d.jumpA, d.jumpC, d.ctl->rng, descDrawOptimistic(d, di), nullptr, (int)ds.nDest);
    if (consumed != (ds.nDest > 0 ? (int)ds.nDest - 1 : 0)) d.ctl->shufReject = 1;
  } else if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SAMPLEK)) {
    int consumed = javaSampleAt(d.jumpA, d.jumpC, d.ctl->rng, descDrawOptimistic(d, di), (int)ds.from, d.N, (int)ds.nDest, nullptr);
    if (consumed != (int)ds.nDest) d.ctl->shufReject = 1;
  }
}
WTG_HD void shuffleSerial(const Dev& d) {  // one thread
  Ctl& ctl = *d.ctl;
  if (!ctl.shufReject) return;
  ctl.serialPasses += 1;
  u64 running = 0;
  for (int g = 0; g < ctl.totalSlots && g < d.newEvCap; ++g) {
    if (d.byGTick[g] != ctl.tick) continue;  // a conditional-task insert: no descriptor, no draw
    int di = d.byG[g];
    const Desc& ds = d.desc[di];
    d.descDraw[di] = (int)running;
    if (ds.dkind == DK_INSERT_AT) continue;
    if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SHUFFLEK))
      running += (u64)javaShuffleAt(d.jumpA, d.jumpC, ctl.rng, running, nullptr, (int)ds.nDest);
    else if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SAMPLEK))
      running += (u64)javaSampleAt(d.jumpA, d.jumpC, ctl.rng, running, (int)ds.from, d.N, (int)ds.nDest, nullptr);
    else if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SHUFFLE2))
      running += 1;
    running += 1;  // the send's seed
  }
  ctl.totalDraws = (int)running;
}

// emit of a shuffled or sampled multi-send (up to SHUFFLE_MAX destinations): the list step (Collections.shuffle of the
// handler's list, or randomRemotes filling it), seed, arrivals, stable sort, envelope
WTG_HD void emitShuffled(const Dev& d, int di, int g, u64 drawIdx) {
  const Ctl& ctl = *d.ctl;
  const Desc& ds = d.desc[di];
  const int m = (int)ds.nDest;
  uint32_t* list = d.destScratch + ds.to;
  int* arr = reinterpret_cast<int*>(d.destScratch + ds.to + m);
  int consumed = (ds.aux & DESC_SAMPLEK) ? javaSampleAt(d.jumpA, d.jumpC, ctl.rng, drawIdx, (int)ds.from, d.N, m, list)
                                         : javaShuffleAt(d.jumpA, d.jumpC, ctl.rng, drawIdx, list, m);
  const int32_t seed = lcgNextIntAt(d, ctl.rng, drawIdx + (u64)consumed);
  const int from = (int)ds.from, sendTime = ctl.tick + 1;
  int cnt = 0;
  for (int i = 0; i < m; ++i) {  // createMessageArrivals :449-467 (stable insertion sort by arrival)
    int to = (int)list[i];
    if (d.npart[from] == d.npart[to] && !d.ndown[from] && !d.ndown[to]) {
      int nt = latency(d, from, to, pseudoRandom(to, seed));
      if (nt < d.msgDiscardTime) {
        int a = sendTime + nt;
        int j = cnt++;
        while (j > 0 && arr[j - 1] > a) {
          arr[j] = arr[j - 1];
          list[j] = list[j - 1];
          --j;
        }
        arr[j] = a;
        list[j] = (uint32_t)to;
      }
    }
  }
  Ev ev;
  ev.kind = EV_MSG;
  ev.to = 0;
  ev.from = ds.from;
  ev.meta = ds.meta;
  ev.pl = ds.pl;
  ev.aux = 0;
  ev.pad = (uint32_t)sendTime + 1u;  // EnvelopeInfo.sentAt + 1
  int target = -1;
  if (cnt == 1) {
    ev.to = list[0];
    target = arr[0];
  } else if (cnt > 1) {
    int ri = WTG_ATOMIC_ADD(&d.ctl->recTop, 1);
    int off = WTG_ATOMIC_ADD(&d.ctl->recDestTop, cnt);
    if (ri >= d.recCap || off + cnt > d.recDestCap) {
      setError(d, ERR_REC_OVERFLOW, ri);
    } else {
      MultiRec rc;
      rc.from = ds.from;
      rc.meta = ds.meta;
      rc.pl = ds.pl;
      rc.n = (uint32_t)cnt;
      rc.cur = 0;
      rc.off = (uint32_t)off;
      rc.pad = (uint32_t)sendTime + 1u;
      d.rec[ri] = rc;
      for (int i = 0; i < cnt; ++i) {
        d.recDest[off + i] = list[i];
        d.recArrival[off + i] = arr[i];
      }
      ev.kind = EV_MULTI;
      ev.to = list[0];
      ev.aux = (uint32_t)ri;
      target = arr[0];
    }
  }
  if (target >= 0 && target - ctl.tick >= d.ring) {
    setError(d, ERR_FAR_FUTURE, target);
    target = -1;
  }
  d.newEv[g] = ev;
  d.newTarget[g] = target;
}

}  // namespace wtg
