// wittgenstein_b200 — P2PFlood (protocols/P2PFlood.java) on core/P2PNetwork.java + core/messages/FloodMessage.java, written
// once for both builds.  Included by wtg_logic.cuh.  Scalar: a node holds one bit per originating message and their count
// (P2PNode.received(-1) is a HashSet of message identities of which only the size is read), and its deliveries run in
// reference order on one thread.  The peer graph is CSR (Dev.peerOff / peerIds, every row in P2PNode.peers order).
//
// A forward (FloodMessage.action :48-55: dest = to.peers minus from, Collections.shuffle(dest, rd), then
// send(this, time + 1 + localDelay, to, dest, delayBetweenPeers)) is one DESC_PEERS descriptor: the handler writes no list.
// emitPeers builds it from the CSR row at emission, shuffles it at the descriptor's draw index and places the envelope.
#pragma once

namespace wtg {

// FloodMessage.action on node n for an envelope sent by `from`; pl = index of the originating message
WTG_HD void floodHandle(const Dev& d, int n, uint32_t from, u64 pl, int item, int& outSlots, int& outDraws) {
  d.msgReceived[n] += 1;
  d.bytesReceived[n] += 1;  // FloodMessage.size = 1 (P2PFlood.java:157-158); duplicates count too (Network.java:611-613)
  statAdd(d, n, ST_DELIVERIES, 1ULL);
  outSlots = outDraws = 0;
  const int k = (int)(uint32_t)pl;
  u64& w = d.floodBits[(size_t)n * d.floodWords + (k >> 6)];
  const u64 bit = 1ULL << (k & 63);
  if (w & bit) return;  // addToReceived(to) is false: nothing else happens
  w |= bit;
  const int cnt = d.floodCnt[n] + 1;
  d.floodCnt[n] = cnt;
  if (cnt == d.floodMsgs) d.doneAt[n] = d.ctl->tick;  // P2PFloodNode.onFlood :39-43
  const uint32_t r0 = d.peerOff[n], r1 = d.peerOff[n + 1];
  int m = (int)(r1 - r0);
  for (uint32_t i = r0; i < r1; ++i) m -= d.peerIds[i] == from ? 1 : 0;
  outSlots = 1;
  outDraws = m > 0 ? m : 1;  // m - 1 shuffle values and the seed; an empty list still draws its seed (Network.java:430)
  CoopSerial cs;
  const int base = descAlloc(d, cs, n, 1);
  if (base < 0) return;
  Desc ds;
  ds.dkind = DK_SEND_MULTI;
  ds.item = (uint32_t)(d.nLoc + item);
  ds.sub = 0;
  ds.from = (uint32_t)n;
  ds.to = from;  // DESC_PEERS: the peer left out of the list
  ds.nDest = (uint32_t)m;
  ds.evKind = EV_MSG;
  ds.meta = P2P_FLOOD;
  ds.pl = pl;
  ds.target = d.ctl->tick + 1 + d.floodResend;
  ds.aux = DESC_SHUFFLEK | DESC_SENDTIME | DESC_PEERS | ((uint32_t)d.floodBetween << DESC_DELAY_SHIFT);
  d.desc[base] = ds;
  const int pi = WTG_ATOMIC_ADD(&d.ctl->peerCnt, 1);
  if (pi < d.descCap)
    d.peerList[pi] = base;
  else
    setError(d, ERR_DESC_OVERFLOW, pi);
  d.msgSent[n] += m;  // every destination counts, delivered or not (Network.java:476-477)
  d.bytesSent[n] += m;
  statAdd(d, n, ST_SENDS, (unsigned long long)m);
}

// Emission of DESC_PEERS descriptor di by one lane group.  `list` and `arr` hold PEERS_MAX entries each (shared memory of
// the warp on the device).  Steps: the list (CSR row without Desc.to, compacted in row order); Collections.shuffle's
// nextInt(i) values, lane-parallel at their presumed positions when no shuffle of the pass rejected (Ctl.shufReject == 0,
// so value j sits at draw index + j), else one lane walks javaShuffleAt from the serially derived index; the swaps, in
// order; the seed, and per destination sendTime + i * step + latency with the down / partition filter
// (createMessageArrivals, Network.java:449-467); a stable rank by (arrival, position) places the destinations in the record,
// and the first arrival goes to the ring or the far-future calendar like emitDesc's.
template <class C>
WTG_HD void emitPeers(const Dev& d, C& c, int di, uint32_t* list, int* arr) {
  const Ctl& ctl = *d.ctl;
  const Desc ds = d.desc[di];
  const int g = d.slotBase[ds.item] + (int)ds.sub;
  if (g >= d.newEvCap) {
    if (c.lane() == 0) setError(d, ERR_DESC_OVERFLOW, g);
    return;
  }
  const int from = (int)ds.from;
  const int r0 = (int)d.peerOff[from], deg = (int)d.peerOff[from + 1] - r0;
  int m = 0;
  for (int i0 = 0; i0 < deg; i0 += C::LANES) {
    const int i = i0 + c.lane();
    const uint32_t p = i < deg ? d.peerIds[r0 + i] : ds.to;
    const bool keep = p != ds.to;
    const uint32_t b = c.ballot(keep);
    if (keep) list[m + c.rank(b)] = p;
    m += c.count(b);
  }
  c.sync();
  const u64 drawIdx = ctl.shufReject ? (u64)d.descDraw[di] : descDrawOptimistic(d, di);
  int consumed = 0;
  if (!ctl.shufReject) {
    for (int j = c.lane(); j < m - 1; j += C::LANES) {
      const int i = m - j;
      const u64 st = lcgAdvance(d.jumpA, d.jumpC, ctl.rng, drawIdx + (u64)j + 1);
      const int32_t u = (int32_t)(uint32_t)(st >> 17);  // next(31)
      arr[j] = (i & (i - 1)) == 0 ? (int)(((long long)i * (long long)u) >> 31) : (int)(u % i);
    }
    c.sync();
    if (c.lane() == 0)
      for (int j = 0; j < m - 1; ++j) {  // swap(list, i - 1, nextInt(i)) for i = m .. 2
        const int i = m - j, r = arr[j];
        const uint32_t t = list[i - 1];
        list[i - 1] = list[r];
        list[r] = t;
      }
    consumed = m > 1 ? m - 1 : 0;
  } else {
    if (c.lane() == 0) consumed = javaShuffleAt(d.jumpA, d.jumpC, ctl.rng, drawIdx, list, m);
    consumed = c.bcast(consumed, 0);
  }
  c.sync();
  const int32_t seed = lcgNextIntAt(d, ctl.rng, drawIdx + (u64)consumed);
  const int sendTime = ds.target;
  const int delay = (int)(ds.aux >> DESC_DELAY_SHIFT);
  const int step = delay > 0 ? delay + 1 : 0;
  int cnt = 0;
  for (int i0 = 0; i0 < m; i0 += C::LANES) {
    const int i = i0 + c.lane();
    int a = -1;
    if (i < m) {
      const int to = (int)list[i];
      if (d.npart[from] == d.npart[to] && !d.ndown[from] && !d.ndown[to]) {
        const int nt = latency(d, from, to, pseudoRandom(to, seed));
        if (nt < d.msgDiscardTime) a = sendTime + i * step + nt;
      }
      arr[i] = a;
    }
    cnt += c.count(c.ballot(a >= 0));
  }
  c.sync();
  int ri = 0, off = 0;
  if (cnt > 1 && c.lane() == 0) {
    ri = WTG_ATOMIC_ADD(&d.ctl->recTop, 1);
    off = WTG_ATOMIC_ADD(&d.ctl->recDestTop, cnt);
  }
  ri = c.bcast(ri, 0);
  off = c.bcast(off, 0);
  const bool recOk = cnt <= 1 || (ri < d.recCap && off + cnt <= d.recDestCap);
  bool found = false;
  int firstTo = 0, firstA = 0;
  for (int i0 = 0; i0 < m; i0 += C::LANES) {
    const int i = i0 + c.lane();
    const int a = i < m ? arr[i] : -1;
    if (a < 0) continue;
    int rank = 0;  // stable sort by arrival (Collections.sort)
    for (int j = 0; j < m; ++j) {
      const int aj = arr[j];
      rank += (aj >= 0 && (aj < a || (aj == a && j < i))) ? 1 : 0;
    }
    if (cnt > 1 && recOk) {
      d.recDest[off + rank] = list[i];
      d.recArrival[off + rank] = a;
    }
    if (rank == 0) {
      found = true;
      firstTo = (int)list[i];
      firstA = a;
    }
  }
  const uint32_t fb = c.ballot(found);
  const int src = fb ? c.first(fb) : 0;
  firstTo = c.bcast(firstTo, src);
  firstA = c.bcast(firstA, src);
  if (c.lane() != 0) return;
  Ev ev;
  ev.kind = EV_MSG;
  ev.to = (uint32_t)firstTo;
  ev.from = ds.from;
  ev.meta = ds.meta;
  ev.pl = ds.pl;
  ev.aux = 0;
  ev.pad = (uint32_t)sendTime + 1u;  // EnvelopeInfo.sentAt + 1
  int target = cnt > 0 ? firstA : -1;
  if (cnt > 1) {
    if (!recOk) {
      setError(d, ERR_REC_OVERFLOW, ri);
      target = -1;
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
      ev.kind = EV_MULTI;
      ev.aux = (uint32_t)ri;
    }
  }
  if (target >= 0 && target - ctl.tick >= farHorizon(d)) {  // P2PFlood always keeps the calendar (fast-forward)
    farAppend(d, ev, target, g);
    target = -1;
  }
  d.newEv[g] = ev;
  d.newTarget[g] = target;
}

}  // namespace wtg
