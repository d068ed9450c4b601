// wittgenstein_b200 — Slush and Snowflake handlers (protocols/Slush.java, protocols/Snowflake.java), written once for both.
// Included by wtg_logic.cuh.  Scalar: a node holds a colour, a query nonce, a round (Slush) or success counter (Snowflake)
// and at most one pending query, and its events run in reference order on one thread (onQuery writes the colour that
// onAnswer reads).  The sample of a query (randomRemotes) is drawn by the emit step: the handler declares a DESC_SAMPLEK
// send of K destinations, and javaSampleAt (wtg_cappos.cuh) fills the list at the send's draw index.
#pragma once

namespace wtg {

WTG_HD u64 avPl(int queryId, int color) { return (u64)(uint32_t)queryId | ((u64)(uint32_t)color << 32); }

struct AvEmit {  // what a handler asks for, in program order: an optional query (sendQuery), an optional answer
  bool query, answer;
  u64 queryPl, answerPl;
  uint32_t answerTo;
};

// sendQuery :178-182 / :190-194 — ++myQueryNonce, the pending Answer, then send(q, this, randomRemotes())
WTG_HD void avSendQuery(const Dev& d, int n, AvEmit& em) {
  const int nonce = d.avNonce[n] + 1;
  d.avNonce[n] = nonce;
  d.avPend[n] = 1;
  d.avFound[2 * (size_t)n] = 0;
  d.avFound[2 * (size_t)n + 1] = 0;
  em.query = true;
  em.queryPl = avPl(nonce, d.avColor[n]);
}

WTG_HD void avHandle(const Dev& d, int n, uint32_t from, uint32_t type, u64 pl, int item, int& outSlots, int& outDraws) {
  AvEmit em;
  em.query = em.answer = false;
  em.queryPl = em.answerPl = 0;
  em.answerTo = 0;
  const int qid = (int)(uint32_t)pl, color = (int)(uint32_t)(pl >> 32);
  d.msgReceived[n] += 1;
  d.bytesReceived[n] += 1;  // Message.size() default (messages/Message.java:27-29)
  statAdd(d, n, ST_DELIVERIES, 1ULL);
  if (type == AV_QUERY) {  // onQuery :148-154 / :153-159
    if (d.avColor[n] == 0) {
      d.avColor[n] = (uint8_t)color;
      avSendQuery(d, n, em);
    }
    em.answer = true;
    em.answerTo = from;
    em.answerPl = avPl(qid, d.avColor[n]);
  } else if (type == AV_ANSWER) {  // onAnswer :161-176 / :170-188
    if (!d.avPend[n] || qid != d.avNonce[n] || color < 1 || color > 2) {  // answerIP.get(queryId) is null in the reference
      setError(d, ERR_PROTO_STATE, n);
      outSlots = outDraws = 0;
      return;
    }
    uint8_t* found = d.avFound + 2 * (size_t)n;
    found[color - 1] += 1;
    if ((int)found[0] + (int)found[1] == d.sampleK) {
      d.avPend[n] = 0;  // answerIP.remove(queryId)
      const int mine = d.avColor[n], other = mine == 1 ? 2 : 1;
      const bool flip = (double)found[other - 1] > d.sampleAK;
      if (d.sampleB < 0) {  // Slush
        if (flip) d.avColor[n] = (uint8_t)other;
        if (d.avRound[n] < d.sampleM) {
          d.avRound[n] += 1;
          avSendQuery(d, n, em);
        }
      } else {  // Snowflake
        if (flip) {
          d.avColor[n] = (uint8_t)other;
          d.avRound[n] = 0;
        } else if ((double)found[mine - 1] > d.sampleAK) {
          d.avRound[n] += 1;
        }
        if (d.avRound[n] <= d.sampleB) avSendQuery(d, n, em);
      }
    }
  }
  const int nd = (em.query ? 1 : 0) + (em.answer ? 1 : 0);
  outSlots = nd;
  outDraws = (em.query ? d.sampleK + 1 : 0) + (em.answer ? 1 : 0);  // the sample's K attempts and its seed; the answer's seed
  if (nd == 0) return;
  CoopSerial cs;
  int base = descAlloc(d, cs, n, nd);
  if (base < 0) return;
  int sub = 0;
  if (em.query) {
    const int K = d.sampleK;
    int off = destAlloc(d, n, 2 * K);  // the sampled destinations, then their arrivals: filled by the emit step
    Desc ds;
    ds.dkind = DK_SEND_MULTI;
    ds.item = (uint32_t)(d.nLoc + item);
    ds.sub = (uint32_t)sub;
    ds.from = (uint32_t)n;
    ds.to = (uint32_t)(off < 0 ? 0 : off);
    ds.nDest = off < 0 ? 0u : (uint32_t)K;
    ds.evKind = EV_MSG;
    ds.meta = AV_QUERY;
    ds.pl = em.queryPl;
    ds.target = 0;
    ds.aux = DESC_SAMPLEK;
    d.desc[base + sub] = ds;
    ++sub;
    d.msgSent[n] += K;
    d.bytesSent[n] += K;
    statAdd(d, n, ST_SENDS, (unsigned long long)K);
  }
  if (em.answer) {  // send(new AnswerQuery(q, myColor), this, from)
    Desc ds;
    ds.dkind = DK_SEND_SINGLE;
    ds.item = (uint32_t)(d.nLoc + item);
    ds.sub = (uint32_t)sub;
    ds.from = (uint32_t)n;
    ds.to = em.answerTo;
    ds.nDest = 1;
    ds.evKind = EV_MSG;
    ds.meta = AV_ANSWER;
    ds.pl = em.answerPl;
    ds.target = 0;
    ds.aux = 0;
    d.desc[base + sub] = ds;
    ++sub;
    d.msgSent[n] += 1;
    d.bytesSent[n] += 1;
    statAdd(d, n, ST_SENDS, 1ULL);
  }
}

}  // namespace wtg
