// wittgenstein_b200 — state-transition bodies of the tick engine.
//
// Every function here is the body of one CUDA kernel work item.  Work items that touch
// bitmaps are executed by one warp ("coop" = 32 lanes: lane-strided 64-bit loads over the
// level block + warp reductions); scalar control flow is warp-uniform.  The same bodies are
// instantiated with a 1-lane coop by the host-side unit tests (tests/emu) to debug the
// exact-order logic without a GPU; the product library only ever runs the CUDA instantiation.
//
// Reference semantics restated here (file:line are under /root/reference):
//   core/Network.java:493-503   getPseudoRandom / hash                  -> pseudoRandom
//   core/NetworkLatency.java:27-34 getLatency                            -> latency
//   core/Network.java:533-570   conditional-task polling                 -> gsfCond
//   protocols/GSFSignature.java:482-534 evaluateSig                      -> gsfScore*
//   protocols/GSFSignature.java:557-583 checkSigs                        -> gsfCheckSigs
//   protocols/GSFSignature.java:537-555 onNewSig                         -> gsfOnNewSig
//   protocols/GSFSignature.java:384-460 updateVerifiedSignatures         -> gsfUpdate
//   protocols/GSFSignature.java:212-224, 313-349 doCycle/getRemainingPeers -> gsfDoCycle
//   protocols/PingPong.java:60-87                                        -> ppDeliver
#pragma once
#include "wtg_types.h"

// host stand-ins (single-threaded debugging build / nvcc host pass of __host__ __device__ bodies)
template <class T, class U>
static inline T wtg_host_fetch_add(T* p, U v) {
  T o = *p;
  *p = (T)(o + (T)v);
  return o;
}
template <class T>
static inline T wtg_host_fetch_max(T* p, T v) {
  T o = *p;
  if (v > o) *p = v;
  return o;
}
template <class T>
static inline T wtg_host_fetch_min(T* p, T v) {
  T o = *p;
  if (v < o) *p = v;
  return o;
}
template <class T>
static inline T wtg_host_cas(T* p, T a, T b) {
  T o = *p;
  if (o == a) *p = b;
  return o;
}
#if defined(__CUDA_ARCH__)
#define WTG_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#define WTG_ATOMIC_MAX(p, v) atomicMax((p), (v))
#define WTG_ATOMIC_MIN(p, v) atomicMin((p), (v))
#define WTG_ATOMIC_CAS(p, a, b) atomicCAS((p), (a), (b))
#define WTG_POPC64(x) __popcll(x)
#define WTG_POPC32(x) __popc(x)
#define WTG_CTZ32(x) (__ffs((int)(x)) - 1)
#define WTG_CTZ64(x) (__ffsll((long long)(x)) - 1)
#else
#define WTG_ATOMIC_ADD(p, v) wtg_host_fetch_add((p), (v))
#define WTG_ATOMIC_MAX(p, v) wtg_host_fetch_max((p), (v))
#define WTG_ATOMIC_MIN(p, v) wtg_host_fetch_min((p), (v))
#define WTG_ATOMIC_CAS(p, a, b) wtg_host_cas((p), (a), (b))
#define WTG_POPC64(x) __builtin_popcountll(x)
#define WTG_POPC32(x) __builtin_popcount(x)
#define WTG_CTZ32(x) __builtin_ctz(x)
#define WTG_CTZ64(x) __builtin_ctzll(x)
#endif

namespace wtg {

typedef unsigned long long u64;

// ------------------------------------------------------------------------------------------
// coop: the group of lanes that executes one work item
// ------------------------------------------------------------------------------------------
struct CoopSerial {
  static constexpr int LANES = 1;
  WTG_HD int lane() const { return 0; }
  WTG_HD uint32_t ballot(bool p) const { return p ? 1u : 0u; }
  WTG_HD int sum(int v) const { return v; }
  WTG_HD int maxv(int v) const { return v; }
  WTG_HD int minv(int v) const { return v; }
  WTG_HD bool any(bool p) const { return p; }
  WTG_HD int bcast(int v, int) const { return v; }
  WTG_HD u64 bcast64(u64 v, int) const { return v; }
  WTG_HD void sync() const {}
  // value held by lane `src` of a per-lane table (serial: read the table itself)
  WTG_HD int gather(int, int src, const int* table) const { return table[src]; }
  // of a ballot m: lanes set, lanes set below this one, lowest lane set (m != 0)
  WTG_HD int count(uint32_t m) const { return (int)(m & 1u); }
  WTG_HD int rank(uint32_t) const { return 0; }
  WTG_HD int first(uint32_t) const { return 0; }
  // sum of v over the lanes below this one; total = sum over all lanes
  WTG_HD int exclusiveScan(int v, int& total) const {
    total = v;
    return 0;
  }
  // next slot of bins[bin] for every active lane, in lane order
  WTG_HD int claim(int* bins, int bin, bool active) const { return active ? bins[bin]++ : 0; }
  // copy a level block of nw words (nw even, both sides 16-byte aligned)
  WTG_HD void copyWords(u64* dst, const u64* src, int nw) const {
    for (int w = 0; w < nw; ++w) dst[w] = src[w];
  }
};
#if defined(__CUDACC__)
struct CoopWarp {
  static constexpr int LANES = 32;
  __device__ __forceinline__ int lane() const { return threadIdx.x & 31; }
  __device__ __forceinline__ uint32_t ballot(bool p) const { return __ballot_sync(0xffffffffu, p); }
  __device__ __forceinline__ int count(uint32_t m) const { return __popc(m); }
  __device__ __forceinline__ int rank(uint32_t m) const { return __popc(m & ((1u << lane()) - 1u)); }
  __device__ __forceinline__ int first(uint32_t m) const { return __ffs(m) - 1; }
  __device__ __forceinline__ int exclusiveScan(int v, int& total) const {
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane() >= o) inc += t;
    }
    total = __shfl_sync(0xffffffffu, inc, 31);
    return inc - v;
  }
  __device__ __forceinline__ int claim(int* bins, int bin, bool active) const {
    const unsigned peers = __match_any_sync(0xffffffffu, active ? bin : -1 - lane());  // inactive lanes: a key of their own
    const int leader = __ffs(peers) - 1;
    int b0 = 0;
    if (active && lane() == leader) {
      b0 = bins[bin];
      bins[bin] = b0 + __popc(peers);
    }
    return __shfl_sync(0xffffffffu, b0, leader) + rank(peers);
  }
  __device__ __forceinline__ void copyWords(u64* __restrict__ dst, const u64* __restrict__ src, int nw) const {
    const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(src);
    ulonglong2* d2 = reinterpret_cast<ulonglong2*>(dst);
    const int n2 = nw >> 1;
    int w = lane();
    for (; w + 96 < n2; w += 128) {  // 4 independent 16-byte loads in flight per lane
      ulonglong2 a = s2[w], b = s2[w + 32], c = s2[w + 64], e = s2[w + 96];
      d2[w] = a;
      d2[w + 32] = b;
      d2[w + 64] = c;
      d2[w + 96] = e;
    }
    for (; w < n2; w += 32) d2[w] = s2[w];
  }
  __device__ __forceinline__ int sum(int v) const { return __reduce_add_sync(0xffffffffu, v); }
  __device__ __forceinline__ int maxv(int v) const { return __reduce_max_sync(0xffffffffu, v); }
  __device__ __forceinline__ int minv(int v) const { return __reduce_min_sync(0xffffffffu, v); }
  __device__ __forceinline__ bool any(bool p) const { return __any_sync(0xffffffffu, p); }
  __device__ __forceinline__ int bcast(int v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
  __device__ __forceinline__ u64 bcast64(u64 v, int src) const { return __shfl_sync(0xffffffffu, v, src); }
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  __device__ __forceinline__ int gather(int mine, int src, const int*) const { return __shfl_sync(0xffffffffu, mine, src); }
};
#endif

WTG_HD void statAdd(const Dev& d, int n, int idx, unsigned long long v) {
  WTG_ATOMIC_ADD(&d.stats[(size_t)(n & (STAT_SLOTS - 1)) * ST_COUNT + idx], v);
}
WTG_HD void statMax(const Dev& d, int n, int idx, unsigned long long v) {
  unsigned long long* p = &d.stats[(size_t)(n & (STAT_SLOTS - 1)) * ST_COUNT + idx];
  WTG_ATOMIC_MAX(p, v);  // result unused: compiles to a reduction, no round trip
}
WTG_HD void setError(const Dev& d, int code, int detail) {
  if (WTG_ATOMIC_CAS(&d.ctl->error, 0, code) == 0) d.ctl->errorDetail = detail;
}

// ------------------------------------------------------------------------------------------
// java.util.Random stream addressing: state after n steps, from 48 (a,c) power tables
// ------------------------------------------------------------------------------------------
constexpr u64 LCG_MASK = (1ULL << 48) - 1;
WTG_HD u64 lcgAdvance(const u64* jumpA, const u64* jumpC, u64 s, u64 n) {
  for (int i = 0; n != 0; ++i, n >>= 1)
    if (n & 1) s = (s * jumpA[i] + jumpC[i]) & LCG_MASK;
  return s;
}
// value of the (k+1)-th rd.nextInt() after state s (k = 0 -> next draw)
WTG_HD int32_t lcgNextIntAt(const Dev& d, u64 s, u64 k) {
  u64 st = lcgAdvance(d.jumpA, d.jumpC, s, k + 1);
  return (int32_t)(uint32_t)(st >> 16);
}

// core/Network.java:493-503
WTG_HD int32_t javaHash(int32_t a0) {
  uint32_t a = (uint32_t)a0;
  a ^= (a << 13);
  a ^= (a >> 17);
  a ^= (a << 5);
  return (int32_t)a;
}
WTG_HD int pseudoRandom(int nodeId, int32_t seed) {
  int32_t x = javaHash(nodeId) ^ seed;
  int32_t r = x % 100;
  return r < 0 ? -r : r;
}

// core/Node.java:278-282 — (int) Math.sqrt(dx*dx + dy*dy), toroidal
WTG_HD int nodeDist(const Dev& d, int a, int b) {
  int ax = d.nx[a], ay = d.ny[a], bx = d.nx[b], by = d.ny[b];
  int ddx = ax > bx ? ax - bx : bx - ax;
  int ddy = ay > by ? ay - by : by - ay;
  int dx = ddx < 2000 - ddx ? ddx : 2000 - ddx;
  int dy = ddy < 1112 - ddy ? ddy : 1112 - ddy;
  int v = dx * dx + dy * dy;
  int r = (int)sqrt((double)v);
  while (r * r > v) --r;  // exact integer floor, independent of the sqrt implementation
  while ((r + 1) * (r + 1) <= v) ++r;
  return r;
}

// core/NetworkLatency.java:27-34 with the samplers folded into integer tables
WTG_HD int latency(const Dev& d, int from, int to, int delta) {
  if (from == to) return 1;
  int extra = (int)d.nextra[from] + (int)d.nextra[to];
  int ext;
  switch (d.latKind) {
    case LAT_DIST_DELTA:
      ext = d.latTab[nodeDist(d, from, to) * 100 + delta];
      break;
    case LAT_CITY: {
      int cf = d.ncity[from], ct = d.ncity[to];
      if (cf == ct)
        ext = 1;
      else {
        ext = (int)d.latBase[cf * 11 + ct] + (int)d.latJit[delta];
        if (ext < 1) ext = 1;
      }
      break;
    }
    case LAT_CONST:
      ext = d.latParam;
      break;
    case LAT_DELTA:
      ext = d.latTab[delta];
      break;
    case LAT_DELTA_2X: {
      int inner = extra + (int)d.latTab[delta];
      ext = inner < 1 ? 1 : inner;
      break;
    }
    case LAT_CITY_MAT: {
      const int K = d.latParam & 0xffff;
      const int cell = (int)d.ncity[from] * K + (int)d.ncity[to];
      ext = (d.latParam >> 16) ? d.latTab[cell * 100 + delta] : d.latTab[cell];
      break;
    }
    default:  // LAT_DIST
      ext = d.latTab[nodeDist(d, from, to)];
      break;
  }
  int base = extra + ext;
  return base < 1 ? 1 : base;
}

// ------------------------------------------------------------------------------------------
// level geometry: level l of a node = the aligned block of 2^(l-1) ids that contains `id`
// ------------------------------------------------------------------------------------------
struct Blk {
  int base;  // first id
  int size;  // ids in the block
  int w0;    // first 64-bit word of the row
  int nw;    // words
  u64 mask;  // valid bits of the (single) word when size < 64
};
WTG_HD Blk levelBlock(int id, int l) {
  Blk b;
  int sh = l - 1;
  b.size = 1 << sh;
  b.base = (id >> sh) << sh;
  b.w0 = b.base >> 6;
  if (b.size >= 64) {
    b.nw = b.size >> 6;
    b.mask = ~0ULL;
  } else {
    b.nw = 1;
    b.mask = ((1ULL << b.size) - 1ULL) << (b.base & 63);
  }
  return b;
}
WTG_HD int poolWords(int l) { return 1 << (l - 1 - 6); }  // l > INLINE_MAX_LEVEL

WTG_HD int msgSize(int l) { return 1 + ((1 << (l - 1)) / 8) + 96; }  // GSFSignature.java:150

WTG_HD uint32_t peerAt(const Dev& d, int n, int l, int idx) {
  size_t off = (size_t)n * (size_t)(d.N - 1) + (size_t)((1 << (l - 1)) - 1) + (size_t)idx;
  if (d.peerBits == 16) {
    int sib = levelBlock(n ^ (1 << (l - 1)), l).base;
    return (uint32_t)sib + (uint32_t)((const uint16_t*)d.peers)[off];
  }
  return ((const uint32_t*)d.peers)[off];
}

// return a payload slab to its pool.  Kernels that never allocate (k_cond, k_emit) push straight onto the
// stripe's free stack; the handler kernel (which allocates) defers the push to k_free.
WTG_HD void freeDirect(const Dev& d, int level, uint32_t slot) {
  const int per = d.poolCap[level] / POOL_STRIPES;
  int sidx = (int)(slot / (uint32_t)per);
  int k = WTG_ATOMIC_ADD(&d.ctl->poolFreeCnt[level][sidx], 1);
  d.poolFree[level][(size_t)sidx * per + k] = slot;
}
WTG_HD void freeDeferred(const Dev& d, int n, int level, uint32_t slot) {
  int st = n & (ARENA_STRIPES - 1);
  int per = d.freeCap / ARENA_STRIPES;
  int i = WTG_ATOMIC_ADD(&d.ctl->freeCnt[st], 1);
  if (i < per)
    d.freeList[(size_t)st * per + i] = ((uint32_t)level << 27) | slot;
  else
    setError(d, ERR_FREE_OVERFLOW, i);
}
// striped free stacks: stripe s of level l owns slots [s*cap/S, (s+1)*cap/S); a node allocates from the
// stripe of its id and falls over to the next stripes when it is empty
WTG_HD bool poolAlloc(const Dev& d, int level, int n, uint32_t& slot) {
  const int per = d.poolCap[level] / POOL_STRIPES;
  for (int t = 0; t < POOL_STRIPES; ++t) {
    int sidx = (n + t) & (POOL_STRIPES - 1);
    int* cnt = &d.ctl->poolFreeCnt[level][sidx];
    if (*cnt <= 0) continue;
    int i = WTG_ATOMIC_ADD(cnt, -1) - 1;
    if (i >= 0) {
      slot = d.poolFree[level][(size_t)sidx * per + i];
      return true;
    }
    WTG_ATOMIC_ADD(cnt, 1);  // lost the race for the last slot of this stripe
  }
  setError(d, ERR_POOL_EXHAUSTED, level);
  slot = 0;
  return false;
}

}  // namespace wtg
#include "wtg_shard.cuh"
namespace wtg {

// node-sharded runs: a pooled payload that arrived from another shard sits in this shard's staging area; move it
// into a pool slab of this shard and make the envelope an ordinary PK_POOL one (one coop per envelope)
template <class C>
WTG_HD void xIngest(const Dev& d, C& c, int g) {
  Ev* ev = &d.newEv[g];
  const uint32_t meta = ev->meta;
  const int l = (int)metaLevel(meta);
  const int src = (int)((meta >> META_SRC_SHIFT) & 7u);
  const int nw = poolWords(l);
  const u64 pl = ev->pl;
  uint32_t slot = 0;
  int ok = 1;
  if (c.lane() == 0) ok = poolAlloc(d, l, (int)ev->to, slot) ? 1 : 0;
  slot = (uint32_t)c.bcast((int)slot, 0);
  ok = c.bcast(ok, 0);
  if (ok) {
    const u64* from = xStagePtr(d, d.rank, src, (int)(uint32_t)pl);
    u64* dst = d.pool[l] + (size_t)slot * (size_t)nw;
    for (int w = c.lane(); w < nw; w += C::LANES) dst[w] = from[w];
    if (d.proto == PROTO_HANDEL && c.lane() == 0) d.poolRef[l][slot] = 1;  // the reference the queue entry will hold
  }
  c.sync();
  if (c.lane() == 0) {
    ev->meta = meta & ~(META_STAGED | (7u << META_SRC_SHIFT));
    ev->pl = (pl & 0xFFFFFFFF00000000ULL) | (u64)slot;
    if (!ok) d.newTarget[g] = -1;
  }
  c.sync();
}
WTG_HD bool xNeedsIngest(const Dev& d, int g) {
  return (d.proto == PROTO_GSF || d.proto == PROTO_HANDEL) && d.newTarget[g] >= 0 && d.newEv[g].kind == EV_MSG && (d.newEv[g].meta & META_STAGED) != 0;
}

// ------------------------------------------------------------------------------------------
// evaluateSig  (GSFSignature.java:482-534) on range-compressed operands
// ------------------------------------------------------------------------------------------
WTG_HD int gsfScoreFrom(int l, int size, int cV, int cSig, bool inter, int cWI, int cWIV, bool interIndiv) {
  int newTotal, added;
  if (cV == 0) {
    newTotal = cSig;
    added = cSig;
  } else if (inter) {
    newTotal = cWI;
    added = cWI - cV;
  } else {
    newTotal = cWIV;
    added = cWIV - cV;
  }
  if (added <= 0) return (cSig == 1 && !interIndiv) ? 1 : 0;
  if (newTotal == size) return 1000000 - l * 10;
  return 100000 - l * 100 + added;
}

// O(1) kinds: evaluated by a single lane
WTG_HD int gsfScoreScalarC(const Dev& d, int n, const QEntry& e, int cV, int cI, int cU);
WTG_HD int gsfScoreScalar(const Dev& d, int n, const QEntry& e) {
  int l = (int)metaLevel(e.meta);
  return gsfScoreScalarC(d, n, e, d.cntVer[n * d.L + l], d.cntIndiv[n * d.L + l], d.cntUnion[n * d.L + l]);
}
// same with the level's cardinalities (|verified|, |indivVerified|, |verified ∪ indivVerified|) supplied by the caller
WTG_HD int gsfScoreScalarC(const Dev& d, int n, const QEntry& e, int cV, int cI, int cU) {
  int l = (int)metaLevel(e.meta);
  int kind = (int)metaKind(e.meta);
  int size = 1 << (l - 1);
  if (cV >= size) return 0;
  const u64* rowV = d.verified + (size_t)n * d.W64;
  const u64* rowI = d.indivVer + (size_t)n * d.W64;
  if (kind == PK_FULL) {
    int k = (int)metaK(e.meta);
    int c = 1 << k;
    bool interIndiv = cI > 0;
    return gsfScoreFrom(l, size, cV, c, cV > 0, c, c, interIndiv);
  }
  if (kind == PK_INDIV) {
    int f = (int)e.from;
    bool inV = (rowV[f >> 6] >> (f & 63)) & 1ULL;
    bool inI = (rowI[f >> 6] >> (f & 63)) & 1ULL;
    return gsfScoreFrom(l, size, cV, 1, inV, cI + (inI ? 0 : 1), cU + ((inI || inV) ? 0 : 1), inI);
  }
  // PK_INLINE
  Blk b = levelBlock((int)e.from, l);
  u64 s = e.pl, v = rowV[b.w0] & b.mask, i = rowI[b.w0] & b.mask;
  return gsfScoreFrom(l, size, cV, WTG_POPC64(s), (s & v) != 0, WTG_POPC64(i | s), WTG_POPC64(i | s | v), (s & i) != 0);
}

// this lane's share of |indiv ∪ sig|, |indiv ∪ sig ∪ verified| and of the two intersections, over nw words
template <class C>
WTG_HD void poolCounts(C& c, const u64* sig, const u64* rowV, const u64* rowI, int nw, int& cWI, int& cWIV, int& inter, int& interI) {
  for (int w = c.lane(); w < nw; w += C::LANES) {
    u64 s = sig[w], v = rowV[w], i = rowI[w];
    cWI += WTG_POPC64(i | s);
    cWIV += WTG_POPC64(i | s | v);
    inter |= (s & v) != 0;
    interI |= (s & i) != 0;
  }
}
#if defined(__CUDACC__)
// the warp streams 128-bit loads, four independent triples in flight per lane (nw is even for pooled levels)
__device__ __forceinline__ void poolCounts(CoopWarp& c, const u64* sig, const u64* rowV, const u64* rowI, int nw, int& cWI, int& cWIV,
                                           int& inter, int& interI) {
  const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(sig);
  const ulonglong2* v2 = reinterpret_cast<const ulonglong2*>(rowV);
  const ulonglong2* i2 = reinterpret_cast<const ulonglong2*>(rowI);
  const int n2 = nw >> 1;
  for (int w0 = c.lane(); w0 < n2; w0 += 128) {
    ulonglong2 sv[4], vv[4], iv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      int w = w0 + 32 * u;
      if (w < n2) {
        sv[u] = s2[w];
        vv[u] = v2[w];
        iv[u] = i2[w];
      } else {
        sv[u] = make_ulonglong2(0, 0);
        vv[u] = sv[u];
        iv[u] = sv[u];
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      cWI += __popcll(iv[u].x | sv[u].x) + __popcll(iv[u].y | sv[u].y);
      cWIV += __popcll(iv[u].x | sv[u].x | vv[u].x) + __popcll(iv[u].y | sv[u].y | vv[u].y);
      inter |= ((sv[u].x & vv[u].x) | (sv[u].y & vv[u].y)) != 0;
      interI |= ((sv[u].x & iv[u].x) | (sv[u].y & iv[u].y)) != 0;
    }
  }
}
#endif

// PK_POOL: the whole coop scans the level block
template <class C>
WTG_HD int gsfScorePool(const Dev& d, C& c, int n, uint32_t from, uint32_t meta, u64 pl) {
  int l = (int)metaLevel(meta);
  int size = 1 << (l - 1);
  int cV = d.cntVer[n * d.L + l];
  if (cV >= size) return 0;
  Blk b = levelBlock((int)from, l);
  const u64* rowV = d.verified + (size_t)n * d.W64 + b.w0;
  const u64* rowI = d.indivVer + (size_t)n * d.W64 + b.w0;
  const u64* sig = d.pool[l] + (size_t)(uint32_t)pl * (size_t)b.nw;
  int cWI = 0, cWIV = 0, inter = 0, interI = 0;
  poolCounts(c, sig, rowV, rowI, b.nw, cWI, cWIV, inter, interI);
  cWI = c.sum(cWI);
  cWIV = c.sum(cWIV);
  bool bi = c.any(inter != 0), bii = c.any(interI != 0);
  return gsfScoreFrom(l, size, cV, (int)(pl >> 32), bi, cWI, cWIV, bii);
}

// ------------------------------------------------------------------------------------------
// checkSigs  (GSFSignature.java:557-583) in three device phases:
//   A  gsfCondScan   (warp / node)   conditional-task bookkeeping (Network.java:543-565 restated per node, see
//                                    DESIGN.md §2.3); re-scores stale O(1) entries in place and lists the stale
//                                    pooled entries (those whose level changed since they were last scored)
//   B  gsfScoreItem  (warp / entry)  evaluateSig of one listed pooled entry: all lanes stream the level block
//   C  gsfCondSelect (warp / node)   first max score, evict score 0, order-preserving compaction, schedule
//                                    updateVerifiedSignatures at time + nodePairingTime
//   condMode 1: the clock has just ticked to `tick` inside a runMs window ending at `until`
//   condMode 2: the reference's extra time++ past `until` at the end of the window
// ------------------------------------------------------------------------------------------
// Where the per-node outputs of the checkSigs pass of `tick` are: condFired / condEv / condTarget have two halves by tick
// parity (GSF), so that the emission of one pass reads its own while the next pass's checkSigs writes the other half.
WTG_HD size_t condHalf(const Dev& d, int tick) { return (size_t)(tick & 1) * (size_t)d.condStride; }
// phase A, scalar part (one thread per node): is the conditional task examined now and is startIf true?
// GSF's phases read the pass clock from condTick / condCall (see Ctl), not from tick / callId.
WTG_HD bool gsfCondMark(const Dev& d, int n) {
  const Ctl& ctl = *d.ctl;
  bool dueNow = false;
  if (ctl.condMode != 0 && !d.ndown[n]) {
    int ms = d.minStart[n];
    bool due = ctl.condMode == 1 ? (ms <= ctl.condTick) : (ms <= ctl.until);
    if (due && d.stamp[n] != ctl.condCall) {
      d.stamp[n] = ctl.condCall;
      if (d.qLen[n] > 0) {  // startIf: !toVerify.isEmpty()
        dueNow = true;
        d.minStart[n] = ctl.condTick + d.pairing[n];
        statAdd(d, n, ST_CONDRUNS, 1ULL);
      }
    }
  }
  d.condDue[n] = dueNow ? 1 : 0;
  if (!dueNow) d.condFired[condHalf(d, ctl.condTick) + n] = 0;
  return dueNow;
}

// phase A, queue part (one coop per due node).  COND_UNROLL chunks of LANES entries are loaded before any is
// used so that a lane keeps several independent 16-byte loads in flight (the scan is latency-bound otherwise).
constexpr int COND_UNROLL = 4;
template <class C>
WTG_HD void gsfCondScanQueue(const Dev& d, C& c, int n) {
  int len = d.qLen[n];
  QEntry* q = d.queue + (size_t)n * d.qcap;
  int* qsc = d.qScore + (size_t)n * d.qcap;
  uint32_t* qst = d.qStamp + (size_t)n * d.qcap;
  const uint32_t* ver = d.lvVer + (size_t)n * d.L;
  const int st = n & (ARENA_STRIPES - 1);
  const int per = d.workCap / ARENA_STRIPES;
  int reeval = 0;
  // lane l keeps level l's version and cardinalities: per entry they come from a shuffle instead of a dependent load
  const int myL = c.lane() < d.L ? c.lane() : 0;
  const int verMine = (int)ver[myL];
  const int cvMine = d.cntVer[n * d.L + myL], ciMine = d.cntIndiv[n * d.L + myL], cuMine = d.cntUnion[n * d.L + myL];
  for (int base0 = 0; base0 < len; base0 += C::LANES * COND_UNROLL) {
    QEntry e[COND_UNROLL];
    uint32_t es[COND_UNROLL];
#pragma unroll
    for (int u = 0; u < COND_UNROLL; ++u) {
      int i = base0 + u * C::LANES + c.lane();
      if (i < len) {
        e[u] = q[i];
        es[u] = qst[i];
      } else {
        e[u].from = 0;
        e[u].meta = 0;
        e[u].pl = 0;
        es[u] = 0;
      }
    }
#pragma unroll
    for (int u = 0; u < COND_UNROLL; ++u) {
      int i = base0 + u * C::LANES + c.lane();
      bool stalePool = false;
      const int lv = (int)metaLevel(e[u].meta);
      const uint32_t v = (uint32_t)c.gather(verMine, lv, reinterpret_cast<const int*>(ver));
      const int cV = c.gather(cvMine, lv, d.cntVer + n * d.L), cI = c.gather(ciMine, lv, d.cntIndiv + n * d.L),
                cU = c.gather(cuMine, lv, d.cntUnion + n * d.L);
      if (i < len) {
        if (es[u] != v) {
          ++reeval;
          if (metaKind(e[u].meta) == PK_POOL) {
            stalePool = true;
          } else {
            qsc[i] = gsfScoreScalarC(d, n, e[u], cV, cI, cU);
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
  }
  reeval = c.sum(reeval);
  if (c.lane() == 0) {
    statAdd(d, n, ST_EVALENTRIES, (unsigned long long)len);
    statAdd(d, n, ST_EVALPOOL, (unsigned long long)reeval);
  }
}

template <class C>
WTG_HD void gsfScoreItem(const Dev& d, C& c, uint32_t item) {
  int n = (int)(item / (uint32_t)d.qcap);
  QEntry e = d.queue[item];
  int s = gsfScorePool(d, c, n, e.from, e.meta, e.pl);
  if (c.lane() == 0) {
    d.qScore[item] = s;
    d.qStamp[item] = d.lvVer[(size_t)n * d.L + metaLevel(e.meta)];
    statAdd(d, n, ST_EVALWORDS, (unsigned long long)(3 * poolWords((int)metaLevel(e.meta))));
  }
}

// keepBits: scratch of qcap/LANES words private to this coop
template <class C>
WTG_HD void gsfCondSelect(const Dev& d, C& c, int n, uint32_t* keepBits) {  // n is due (callers walk the due list)
  const Ctl& ctl = *d.ctl;
  int len = d.qLen[n];
  const int pairing = d.pairing[n];
  QEntry* q = d.queue + (size_t)n * d.qcap;
  int* qsc = d.qScore + (size_t)n * d.qcap;
  uint32_t* qst = d.qStamp + (size_t)n * d.qcap;
  int bestScore = 0, bestIdx = 0x7fffffff;
  for (int base0 = 0; base0 < len; base0 += C::LANES * COND_UNROLL) {
    int sc[COND_UNROLL];
#pragma unroll
    for (int u = 0; u < COND_UNROLL; ++u) {
      int i = base0 + u * C::LANES + c.lane();
      sc[u] = i < len ? qsc[i] : 0;
    }
#pragma unroll
    for (int u = 0; u < COND_UNROLL; ++u) {
      int base = base0 + u * C::LANES;
      if (base >= len) break;
      int i = base + c.lane();
      uint32_t km = c.ballot(sc[u] > 0);
      if (c.lane() == 0) keepBits[base / C::LANES] = km;
      if (sc[u] > bestScore) {  // strict >: keeps this lane's earliest max (checkSigs :565-567)
        bestScore = sc[u];
        bestIdx = i;
      }
    }
  }
  int mx = c.maxv(bestScore);
  int bi = c.minv(bestScore == mx ? bestIdx : 0x7fffffff);
  bool found = mx > 0;
  c.sync();
  // order-preserving compaction: drop score-0 entries (it.remove() :568-570) and the best one (:574).
  // Chunks before the first removal do not move; from there on COND_UNROLL chunks are loaded, then stored.
  QEntry best;
  best.from = 0;
  best.meta = 0;
  best.pl = 0;
  int w = 0;
  int base0 = 0;
  for (; base0 < len; base0 += C::LANES) {  // skip the static prefix
    uint32_t kw = keepBits[base0 / C::LANES];
    int inChunk = len - base0 < C::LANES ? len - base0 : C::LANES;
    int tot = c.count(kw);
    bool hasBest = found && bi >= base0 && bi < base0 + C::LANES;
    if (tot != inChunk || hasBest) break;
    w += tot;
  }
  for (; base0 < len; base0 += C::LANES * COND_UNROLL) {
    QEntry e[COND_UNROLL];
    int es[COND_UNROLL];
    uint32_t et[COND_UNROLL];
#pragma unroll
    for (int u = 0; u < COND_UNROLL; ++u) {
      int i = base0 + u * C::LANES + c.lane();
      if (i < len) {
        e[u] = q[i];
        es[u] = qsc[i];
        et[u] = qst[i];
      } else {
        e[u].from = 0;
        e[u].meta = 0;
        e[u].pl = 0;
        es[u] = 0;
        et[u] = 0;
      }
    }
    c.sync();  // every lane has loaded its entries before anyone overwrites these chunks
#pragma unroll
    for (int u = 0; u < COND_UNROLL; ++u) {
      int base = base0 + u * C::LANES;
      if (base >= len) break;
      int i = base + c.lane();
      bool keep = false, evict = false;
      uint32_t kw = keepBits[base / C::LANES];
      if (i < len) {
        bool k0 = (kw >> c.lane()) & 1u;
        keep = k0 && !(found && i == bi);
        evict = !k0;
      }
      uint32_t km = c.ballot(keep);
      int off = c.rank(km);
      int tot = c.count(km);
      if (keep && w + off != i) {
        q[w + off] = e[u];
        qsc[w + off] = es[u];
        qst[w + off] = et[u];
      }
      if (evict && metaKind(e[u].meta) == PK_POOL) freeDirect(d, (int)metaLevel(e[u].meta), (uint32_t)e[u].pl);
      if (found && i == bi) best = e[u];
      w += tot;
    }
    c.sync();
  }
  if (found) {
    int srcLane = bi % C::LANES;
    best.from = (uint32_t)c.bcast((int)best.from, srcLane);
    best.meta = (uint32_t)c.bcast((int)best.meta, srcLane);
    best.pl = c.bcast64(best.pl, srcLane);
  }
  if (c.lane() == 0) {
    d.qLen[n] = w;
    if (found) {  // registerTask(updateVerifiedSignatures, time + nodePairingTime, this)  :575-581
      WTG_ATOMIC_ADD(&d.sigChecked[n], 1);
      d.sigQueueSize[n] = w;
      Ev ev;
      ev.kind = EV_TASK;
      ev.to = (uint32_t)n;
      ev.from = best.from;
      ev.meta = best.meta;
      ev.pl = best.pl;
      ev.aux = 0;
      ev.pad = (uint32_t)ctl.condTick + 1u;  // Envelope.sendTime + 1 (EnvelopeInfo.sentAt for peekMessages; 0 = not recorded)
      d.condEv[condHalf(d, ctl.condTick) + n] = ev;
      d.condTarget[condHalf(d, ctl.condTick) + n] = ctl.condTick + pairing;
    }
    d.condFired[condHalf(d, ctl.condTick) + n] = found ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------------
// descriptor helpers
// ------------------------------------------------------------------------------------------
template <class C>
WTG_HD int descAlloc(const Dev& d, C& c, int n, int cnt) {
  int base = 0;
  if (c.lane() == 0) {
    int st = n & (ARENA_STRIPES - 1);
    int per = d.descCap / ARENA_STRIPES;
    int i = WTG_ATOMIC_ADD(&d.ctl->descCnt[st], cnt);
    if (i + cnt > per) {
      setError(d, ERR_DESC_OVERFLOW, i + cnt);
      base = -1;
    } else {
      base = st * per + i;
    }
  }
  return c.bcast(base, 0);
}
// scratch for the destination list of a multi-send (same striping)
WTG_HD int destAlloc(const Dev& d, int n, int cnt) {
  int st = n & (ARENA_STRIPES - 1);
  int per = d.destScratchCap / ARENA_STRIPES;
  int i = WTG_ATOMIC_ADD(&d.ctl->destCnt[st], cnt);
  if (i + cnt > per) {
    setError(d, ERR_DESC_OVERFLOW, i + cnt);
    return -1;
  }
  return st * per + i;
}

WTG_HD void gsfLevelCounters(const Dev& d, int n, int l, int& cV, int& cI, int& cU) {
  cV = d.cntVer[n * d.L + l];
  cI = d.cntIndiv[n * d.L + l];
  cU = d.cntUnion[n * d.L + l];
}

// Per-level scalars of a node are handled "levels as lanes": lane i owns the levels k * LANES + i for k < 32 / LANES
// (a warp: one level per lane; one lane: every level in turn), and level masks are built from per-round ballots.

// number of consecutive complete levels: levels 0..k complete (getLastFinishedLevel :193-210)
template <class C>
WTG_HD int gsfLastFinishedLevel(const Dev& d, C& c, int n) {
  uint32_t comp = 0;
  for (int k = 0; k < 32 / C::LANES; ++k) {
    const int l = k * C::LANES + c.lane();
    comp |= c.ballot(l >= 1 && l < d.L && d.cntVer[n * d.L + l] == (1 << (l - 1))) << (k * C::LANES);
  }
  return WTG_CTZ32(~(comp >> 1));
}

// onNewSig (GSFSignature.java:537-555) — executed by lane 0 only
WTG_HD void gsfOnNewSig(const Dev& d, int n, uint32_t from, uint32_t meta, u64 pl) {
  int l = (int)metaLevel(meta);
  int len = d.qLen[n];
  QEntry* q = d.queue + (size_t)n * d.qcap;
  if (len + 2 > d.qcap) {
    setError(d, ERR_QUEUE_OVERFLOW, n);
    if (metaKind(meta) == PK_POOL) freeDeferred(d, n, l, (uint32_t)pl);
    return;
  }
  QEntry e;
  e.from = from;
  e.meta = meta;
  e.pl = pl;
  uint32_t* qs = d.qStamp + (size_t)n * d.qcap;
  qs[len] = 0;  // score not evaluated yet
  q[len++] = e;
  u64* rowS = d.indivSeen + (size_t)n * d.W64;
  u64 bit = 1ULL << (from & 63);
  if (!(rowS[from >> 6] & bit)) {
    rowS[from >> 6] |= bit;
    QEntry ie;
    ie.from = from;
    ie.meta = metaMake(PK_INDIV, (uint32_t)l, 0);
    ie.pl = 0;
    qs[len] = 0;
    q[len++] = ie;
  }
  d.qLen[n] = len;
  d.sigQueueSize[n] = len;
  statMax(d, n, ST_MAXQUEUE, (unsigned long long)len);
}

// take up to `want` peers of level l (getRemainingPeers :325-349); returns the count, writes ids
template <class C>
WTG_HD int gsfTakePeers(const Dev& d, C& c, int n, int l, int want, uint32_t* out) {
  int rem = d.remaining[n * d.L + l];
  int p = d.pos[n * d.L + l];
  int sz = 1 << (l - 1);
  int cnt = want < rem ? want : rem;
  for (int i = 0; i < cnt; ++i) {
    out[i] = peerAt(d, n, l, p);
    if (++p >= sz) p = 0;
  }
  c.sync();
  if (c.lane() == 0) {
    d.remaining[n * d.L + l] = rem - cnt;
    d.pos[n * d.L + l] = p;
  }
  c.sync();
  return cnt;
}

// ------------------------------------------------------------------------------------------
// updateVerifiedSignatures  (GSFSignature.java:384-460)
// item: scan item of this event; returns via evSlots/evDraws/desc
// ------------------------------------------------------------------------------------------
template <class C>
WTG_HD void gsfUpdate(const Dev& d, C& c, int n, uint32_t from, uint32_t meta, u64 pl, int item, int& outSlots, int& outDraws) {
  const int L = d.L;
  const int tick = d.ctl->tick;
  int l = (int)metaLevel(meta);
  int kind = (int)metaKind(meta);
  int k = (int)metaK(meta);
  int size = 1 << (l - 1);
  Blk b = levelBlock((int)from, l);
  u64* rowV = d.verified + (size_t)n * d.W64;
  u64* rowI = d.indivVer + (size_t)n * d.W64;
  int cV, cI, cU;
  gsfLevelCounters(d, n, l, cV, cI, cU);
  int total = d.totalCard[n];
  int cSig = kind == PK_INDIV ? 1 : kind == PK_FULL ? (1 << k) : kind == PK_INLINE ? WTG_POPC64(pl) : (int)(pl >> 32);
  if (c.lane() == 0) {
    statAdd(d, n, ST_UPDATES, 1ULL);
    WTG_ATOMIC_ADD(&d.lvVer[n * L + l], 1u);  // cached scores of this level's queue entries are stale from here on (no read-back)
  }

  // :387-389  if (sigs.cardinality() == 1) sfl.indivVerifiedSig.set(from.nodeId);
  if (cSig == 1) {
    u64 bit = 1ULL << (from & 63);
    u64 wI = rowI[from >> 6], wV = rowV[from >> 6];
    c.sync();
    if (!(wI & bit)) {
      if (c.lane() == 0) rowI[from >> 6] = wI | bit;
      cI += 1;
      if (!(wV & bit)) cU += 1;
    }
    c.sync();
  }

  bool changed = false;  // the `if (sigs.cardinality() > sfl.verified.cardinality() || resetRemaining)` branch
  bool superset = (kind == PK_FULL && k >= l);  // :397  sigs.cardinality() > sfl.expectedSigs()
  if (superset) {
    bool resetRemaining = false;
    for (int i = 1; i < L && i <= k; ++i) {  // :401  include(sigs, levels[i].waitedSigs)  <=>  i <= k
      int ci = d.cntVer[n * L + i];
      int si = 1 << (i - 1);
      if (ci != si) {  // :403-407
        Blk wb = levelBlock(n ^ (1 << (i - 1)), i);
        for (int w = c.lane(); w < wb.nw; w += C::LANES) rowV[wb.w0 + w] |= wb.mask;
        total += si - ci;
        if (c.lane() == 0) {
          d.cntVer[n * L + i] = si;
          d.cntUnion[n * L + i] = si;
          d.lvVer[n * L + i] += 1;
        }
        if (i == l) {
          cV = si;
          cU = si;
        }
        resetRemaining = true;
      }
      if (resetRemaining && c.lane() == 0) d.remaining[n * L + i] = si;  // :408-410
    }
    c.sync();
    // sigs = clone(waitedSigs): full block; level l is complete (l <= k) so no merge and |sigs| == |verified|
    changed = resetRemaining;
  } else {
    // sig' = sigs | indivVerifiedSig (both inside the level block); count and test against verified
    int cA = 0;
    bool inter = false;
    if (kind == PK_FULL) {  // k == l-1: the whole block
      cA = size;
      inter = cV > 0;
    } else if (kind == PK_INDIV) {  // {from} | indiv == indiv (from was just added)
      cA = cI;
      inter = (cI + cV - cU) > 0;
    } else if (kind == PK_INLINE) {
      u64 a = pl | (rowI[b.w0] & b.mask);
      cA = WTG_POPC64(a);
      inter = (a & rowV[b.w0] & b.mask) != 0;
    } else {
      const u64* sig = d.pool[l] + (size_t)(uint32_t)pl * (size_t)b.nw;
      int ca = 0, it = 0;
      for (int w = c.lane(); w < b.nw; w += C::LANES) {
        u64 a = sig[w] | rowI[b.w0 + w];
        ca += WTG_POPC64(a);
        it |= (a & rowV[b.w0 + w]) != 0;
      }
      cA = c.sum(ca);
      inter = c.any(it != 0);
    }
    bool merge = (cV > 0 && !inter);  // :415-420
    int cM = merge ? cA + cV : cA;
    if (cM > cV) {  // :422
      changed = true;
      // :432-436 replace the level block (and the same bits of the node-wide set) by sig' [| verified]
      c.sync();
      if (kind == PK_FULL) {
        for (int w = c.lane(); w < b.nw; w += C::LANES) rowV[b.w0 + w] |= b.mask;
      } else if (kind == PK_INDIV) {
        for (int w = c.lane(); w < b.nw; w += C::LANES) {
          u64 cur = rowV[b.w0 + w];
          u64 nv = (rowI[b.w0 + w] & b.mask) | (merge ? (cur & b.mask) : 0ULL);
          rowV[b.w0 + w] = (cur & ~b.mask) | nv;
        }
      } else if (kind == PK_INLINE) {
        if (c.lane() == 0) {
          u64 cur = rowV[b.w0];
          u64 nv = pl | (rowI[b.w0] & b.mask) | (merge ? (cur & b.mask) : 0ULL);
          rowV[b.w0] = (cur & ~b.mask) | nv;
        }
      } else {
        const u64* sig = d.pool[l] + (size_t)(uint32_t)pl * (size_t)b.nw;
        for (int w = c.lane(); w < b.nw; w += C::LANES) {
          u64 nv = sig[w] | rowI[b.w0 + w];
          if (merge) nv |= rowV[b.w0 + w];
          rowV[b.w0 + w] = nv;
        }
      }
      total += cM - cV;
      cV = cM;
      cU = cM;  // the new verified set contains indivVerifiedSig
      if (c.lane() == 0) d.cntVer[n * L + l] = cV;
      c.sync();
    }
  }
  if (c.lane() == 0) {
    d.cntIndiv[n * L + l] = cI;
    d.cntUnion[n * L + l] = cU;
    d.totalCard[n] = total;
  }
  if (kind == PK_POOL && c.lane() == 0) {
    freeDeferred(d, n, l, (uint32_t)pl);
    statAdd(d, n, ST_UPDATEWORDS, (unsigned long long)((changed ? 4 : 3) * b.nw));  // read payload ∥ indiv ∥ verified, write verified
  }
  c.sync();

  outSlots = 0;
  outDraws = 0;
  if (!changed) return;

  // :424-428 new signatures: reset remainingCalls of this level and all levels above
  for (int i = l + c.lane(); i < L; i += C::LANES) d.remaining[n * L + i] = 1 << (i - 1);
  c.sync();

  if (d.accel > 0) {  // :438-451
    int kf = gsfLastFinishedLevel(d, c, n);
    // count the sends first so the descriptor block can be allocated in one go
    int nSend = 0;
    for (int cur = l; cur <= kf && cur < L - 1;) {
      ++cur;
      if (d.remaining[n * L + cur] > 0) ++nSend;
    }
    if (nSend > 0) {
      int base = descAlloc(d, c, n, nSend);
      int sub = 0;
      long long sentMsgs = 0, sentBytes = 0;
      for (int cur = l; cur <= kf && cur < L - 1;) {
        ++cur;
        uint32_t dests[MAX_ACC];
        int cnt = gsfTakePeers(d, c, n, cur, d.accel, dests);
        if (cnt == 0) continue;
        sentMsgs += cnt;
        sentBytes += (long long)cnt * msgSize(cur);
        if (base >= 0 && c.lane() == 0) {
          Desc ds;
          ds.item = (uint32_t)(d.nLoc + item);
          ds.sub = (uint32_t)sub;
          ds.from = (uint32_t)n;
          ds.evKind = EV_MSG;
          ds.meta = metaMake(PK_FULL, (uint32_t)cur, (uint32_t)kf);
          ds.pl = 0;
          ds.target = 0;
          ds.aux = 0;
          if (cnt == 1) {  // Network.send(m, from, dests) with one dest -> single-destination path (:357-358)
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
          d.desc[base + sub] = ds;
        }
        ++sub;
      }
      if (c.lane() == 0) {
        d.msgSent[n] += sentMsgs;
        d.bytesSent[n] += sentBytes;
        statAdd(d, n, ST_MULTISENDS, (unsigned long long)sub);
      }
      outSlots = sub;
      outDraws = sub;
    }
  }
  // :452-453
  if (c.lane() == 0 && d.doneAt[n] == 0 && total >= d.threshold) d.doneAt[n] = tick;
  c.sync();
}

// ------------------------------------------------------------------------------------------
// doCycle  (GSFSignature.java:212-224 + SFLevel.doCycle :313-323) and the periodic re-arm
// (messages/PeriodicTask.java:40-47)
// ------------------------------------------------------------------------------------------
// Levels as lanes: the per-level scalars (cardinality, remainingCalls, cursor, next peer) are loaded and decided by the
// level's lane; only the payload snapshots are copied by the whole coop.  The send pass reloads what it needs instead of
// keeping it per level, so the one-lane form holds no per-level arrays.
template <class C>
WTG_HD void gsfDoCycle(const Dev& d, C& c, int n, int item, int& outSlots, int& outDraws) {
  constexpr int K = 32 / C::LANES;
  const int L = d.L;
  const int tick = d.ctl->tick;
  const u64* rowV = d.verified + (size_t)n * d.W64;
  const int kf = gsfLastFinishedLevel(d, c, n);
  uint32_t sendMask = 0;
  int carry = 0;
  for (int k = 0; k < K; ++k) {
    const int l = k * C::LANES + c.lane();
    const bool valid = l >= 1 && l < L;
    const int cv = l < L ? d.cntVer[n * L + l] : 0;
    const int rem = valid ? d.remaining[n * L + l] : 0;
    int total;
    const int prefix = carry + c.exclusiveScan(cv, total);  // sum of the cardinalities of levels 0..l-1
    carry += total;
    const int size = valid ? (1 << (l - 1)) : 0;
    const int card = (kf >= l - 1) ? (1 << kf) : prefix;
    const bool started = tick >= l * d.timeoutPerLevel || card >= size;  // hasStarted :291-311
    sendMask |= c.ballot(valid && rem > 0 && started) << (k * C::LANES);
  }
  const int nSend = WTG_POPC32(sendMask);
  const int base = descAlloc(d, c, n, nSend + 1);
  unsigned long long words = 0;
  int bytes = 0;
  carry = 0;
  for (int k = 0; k < K; ++k) {
    const int l = k * C::LANES + c.lane();
    const bool snd = (sendMask >> l) & 1u;
    const int size = l >= 1 && l < L ? (1 << (l - 1)) : 0;
    int total;
    const int prefix = carry + c.exclusiveScan(l < L ? d.cntVer[n * L + l] : 0, total);
    carry += total;
    uint32_t dest = 0, meta = 0, slot = 0;
    u64 pl = 0;
    bool pooled = false;
    int stagedOn = -1;
    if (snd) {
      const int p = d.pos[n * L + l];
      dest = peerAt(d, n, l, p);  // getRemainingPeers(1) :325-349
      d.pos[n * L + l] = p + 1 >= size ? 0 : p + 1;
      d.remaining[n * L + l] -= 1;
      if (kf >= l - 1) {
        meta = metaMake(PK_FULL, (uint32_t)l, (uint32_t)kf);
      } else if (l <= INLINE_MAX_LEVEL) {
        Blk ob = levelBlock(n, l);  // our own half: what the receiver waits for at its level l
        meta = metaMake(PK_INLINE, (uint32_t)l, 0);
        pl = rowV[ob.w0] & ob.mask;
      } else {
        meta = metaMake(PK_POOL, (uint32_t)l, 0);
        const int q = ownerOf(d, (int)dest);
        if (q != d.rank) {  // the receiver lives on another shard: the snapshot goes into its staging area
          int off = xStageAlloc(d, q, poolWords(l));
          pooled = off >= 0;
          slot = (uint32_t)(pooled ? off : 0);
          meta |= META_STAGED | ((uint32_t)d.rank << META_SRC_SHIFT);
          stagedOn = q;
        } else {
          pooled = poolAlloc(d, l, n, slot);
        }
        pl = (u64)slot | ((u64)(uint32_t)prefix << 32);
      }
    }
    uint32_t pm = c.ballot(pooled);
    while (pm) {
      const int src = c.first(pm);
      pm &= pm - 1;
      const int ls = k * C::LANES + src;
      const uint32_t sl = (uint32_t)c.bcast((int)slot, src);
      const int so = c.bcast(stagedOn, src);
      Blk ob = levelBlock(n, ls);
      u64* dstp = so >= 0 ? xStagePtr(d, so, d.rank, (int)sl) : d.pool[ls] + (size_t)sl * (size_t)ob.nw;
      c.copyWords(dstp, rowV + ob.w0, ob.nw);
      words += (unsigned long long)(2 * ob.nw);
    }
    if (snd && base >= 0) {
      const int sub = WTG_POPC32(sendMask & ((1u << l) - 1u));
      Desc ds;
      ds.dkind = DK_SEND_SINGLE;
      ds.item = (uint32_t)(d.nLoc + item);
      ds.sub = (uint32_t)sub;
      ds.from = (uint32_t)n;
      ds.to = dest;
      ds.nDest = 1;
      ds.evKind = EV_MSG;
      ds.meta = meta;
      ds.pl = pl;
      ds.target = 0;
      ds.aux = 0;
      d.desc[base + sub] = ds;
    }
    bytes += snd ? msgSize(l) : 0;
  }
  bytes = c.sum(bytes);
  if (c.lane() == 0) {
    if (base >= 0) {  // re-arm: network.sendArriveAt(this, time + period, sender, sender)
      Desc ds;
      ds.dkind = DK_INSERT_AT;
      ds.item = (uint32_t)(d.nLoc + item);
      ds.sub = (uint32_t)nSend;
      ds.from = (uint32_t)n;
      ds.to = (uint32_t)n;
      ds.nDest = 0;
      ds.evKind = EV_PERIODIC;
      ds.meta = 0;
      ds.pl = 0;
      ds.target = tick + d.period;
      ds.aux = 0;
      d.desc[base + nSend] = ds;
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

// ------------------------------------------------------------------------------------------
// SanFerminSignature handlers (protocols/SanFerminSignature.java, SanFerminHelper.java) — scalar: per-node
// state is a handful of ints, so every event of a node is handled by one thread, in reference order.
// Power-of-two node counts; candidateCount up to SHUFFLE_MAX - 1 (the shipped scenario uses 1, SanFerminSignature.java:568-571).
// ------------------------------------------------------------------------------------------
struct SfEmit {  // what a handler asks the engine to do, in program order: at most one send, then one task
  int nSend;     // 0, 1 (single destination) or more (shuffled before the send)
  uint32_t dst[SHUFFLE_MAX];
  uint32_t sendMeta;
  u64 sendPl;
  bool task;
  uint32_t taskMeta;
  u64 taskPl;
  int taskAt;
};
WTG_HD u64 sfPl(int level, int value) { return (u64)(uint32_t)level | ((u64)(uint32_t)value << 32); }
WTG_HD bool sfIsCandidate(const Dev& d, int n, int node, int level) {  // SanFerminHelper.getCandidateSet :70-96 (N = 2^P)
  int shift = d.sfP - 1 - level;
  if (shift < 0) return false;
  return (node >> shift) == ((n >> shift) ^ 1);
}
// SanFerminHelper.pickNextNodes(level, candidateCount) :123-157 without the shuffle (the emit step performs it); the
// helper's usedNodes of the current level is a bitmap (wtg_cappos.cuh)
WTG_HD int cpPickNextNodes(const Dev& d, int n, int level, uint32_t* out);
WTG_HD int sfPickNextNodes(const Dev& d, int n, int level, uint32_t* out) { return cpPickNextNodes(d, n, level, out); }
// pendingNodes (:189) holds candidates of the current level only: a bitmap over positions in the candidate block
WTG_HD bool sfPendingHas(const Dev& d, int n, int node) {
  int shift = d.sfP - 1 - d.sfCpl[n];
  if (shift < 0 || !sfIsCandidate(d, n, node, d.sfCpl[n])) return false;
  int pos = node & ((1 << shift) - 1);
  return (d.sfPendBits[(size_t)n * d.sfUsedWords + (pos >> 6)] >> (pos & 63)) & 1ULL;
}
WTG_HD void sfSendToNodes(const Dev& d, int n, const uint32_t* list, int cnt, SfEmit& em) {  // :329-373
  if (cnt == 0) return;
  int cpl = d.sfCpl[n];
  {
    const int shift = d.sfP - 1 - cpl;
    u64* pend = d.sfPendBits + (size_t)n * d.sfUsedWords;
    for (int i = 0; i < cnt; ++i) {  // every picked node is a candidate of the current level
      int pos = (int)list[i] & ((1 << shift) - 1);
      pend[pos >> 6] |= 1ULL << (pos & 63);
    }
  }
  d.sfSentReq[n] += cnt;
  em.nSend = cnt;
  for (int i = 0; i < cnt; ++i) em.dst[i] = list[i];
  em.sendMeta = SF_REQ;
  em.sendPl = sfPl(cpl, d.sfAgg[n]);
  em.task = true;
  em.taskMeta = SF_T_TIMEOUT;
  em.taskPl = sfPl(cpl, 0);
  em.taskAt = d.ctl->tick + d.sfReplyTimeout;
}
WTG_HD void sfGoNextLevel(const Dev& d, int n, SfEmit& em) {  // :383-423
  int fl = d.sfFlags[n];
  if (fl & 2) return;
  int cpl = d.sfCpl[n];
  int agg = d.sfAgg[n];
  const int tick = d.ctl->tick;
  if (agg >= d.sfThreshold && !(fl & 4)) {
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
  d.sfCache[(size_t)n * 32 + cpl] = agg;
  d.sfCacheMask[n] |= 1u << cpl;
  fl &= ~1;
  d.sfFlags[n] = fl;
  {  // pendingNodes.clear(); usedNodes of a level that was never picked from is a fresh BitSet
    int words = ((1 << (d.sfP - 1 - cpl)) + 63) / 64;
    u64* used = d.sfUsedBits + (size_t)n * d.sfUsedWords;
    u64* pend = d.sfPendBits + (size_t)n * d.sfUsedWords;
    for (int w = 0; w < words; ++w) {
      used[w] = 0;
      pend[w] = 0;
    }
  }
  uint32_t list[SHUFFLE_MAX];
  int cnt = sfPickNextNodes(d, n, cpl, list);
  sfSendToNodes(d, n, list, cnt, em);
}
WTG_HD void sfReply(const Dev& d, int n, uint32_t to, uint32_t status, int level, int value, SfEmit& em) {  // :425-432
  (void)d;
  (void)n;
  em.nSend = 1;
  em.dst[0] = to;
  em.sendMeta = status;
  em.sendPl = sfPl(level, value);
}
WTG_HD void sfTransition(const Dev& d, int n, int toAggregate, SfEmit& em) {  // :438-455
  d.sfFlags[n] |= 1;
  em.task = true;
  em.taskMeta = SF_T_TRANSITION;
  em.taskPl = sfPl(0, toAggregate);
  em.taskAt = d.ctl->tick + d.sfPairing;
}
WTG_HD void sfHandle(const Dev& d, int n, uint32_t from, uint32_t type, u64 pl, int item, int& outSlots, int& outDraws) {
  SfEmit em;
  em.nSend = 0;
  em.task = false;
  em.dst[0] = em.dst[1] = 0;
  em.sendMeta = 0;
  em.sendPl = 0;
  em.taskMeta = 0;
  em.taskPl = 0;
  em.taskAt = 0;
  const int level = (int)(uint32_t)pl, val = (int)(uint32_t)(pl >> 32);
  const int msgBytes = 4 + d.sfSigSize;
  if (type == SF_REQ || type == SF_REPLY_OK || type == SF_REPLY_NO) {
    d.msgReceived[n] += 1;
    d.bytesReceived[n] += msgBytes;
    statAdd(d, n, ST_DELIVERIES, 1ULL);
  } else {
    statAdd(d, n, ST_TASKS, 1ULL);
  }
  int fl = d.sfFlags[n], cpl = d.sfCpl[n];
  switch (type) {
    case SF_REQ: {  // onSwapRequest :229-268
      d.sfRecvReq[n] += 1;
      if ((fl & 2) || level != cpl) {
        if (level >= 0 && level < 32 && (d.sfCacheMask[n] >> level) & 1u) {
          sfReply(d, n, from, SF_REPLY_OK, level, d.sfCache[(size_t)n * 32 + level], em);
        } else {
          sfReply(d, n, from, SF_REPLY_NO, cpl, 0, em);
          if (level >= 0 && level < 32 && sfIsCandidate(d, n, (int)from, level)) {
            d.sfCache[(size_t)n * 32 + level] = val;
            d.sfCacheMask[n] |= 1u << level;
          }
        }
      } else if (fl & 1) {
        sfReply(d, n, from, SF_REPLY_OK, level, d.sfAgg[n], em);
      } else if (sfIsCandidate(d, n, (int)from, cpl)) {
        sfTransition(d, n, val, em);
      }
      break;
    }
    case SF_REPLY_OK:
    case SF_REPLY_NO: {  // onSwapReply :270-323
      if (level != cpl || (fl & 2)) break;
      if (fl & 1) break;
      bool pending = sfPendingHas(d, n, (int)from);
      if (type == SF_REPLY_OK) {
        if (pending || sfIsCandidate(d, n, (int)from, cpl)) sfTransition(d, n, val, em);
      } else if (pending) {
        uint32_t list[SHUFFLE_MAX];
        int cnt = sfPickNextNodes(d, n, cpl, list);
        sfSendToNodes(d, n, list, cnt, em);
      }
      break;
    }
    case SF_T_GO:
      sfGoNextLevel(d, n, em);
      break;
    case SF_T_TIMEOUT:  // :356-369
      if (!(fl & 2) && cpl == level) {
        uint32_t list[SHUFFLE_MAX];
        int cnt = sfPickNextNodes(d, n, cpl, list);
        sfSendToNodes(d, n, list, cnt, em);
      }
      break;
    case SF_T_TRANSITION:  // :441-452
      d.sfAgg[n] += val;
      sfGoNextLevel(d, n, em);
      break;
    default:
      break;
  }
  int nd = (em.nSend > 0 ? 1 : 0) + (em.task ? 1 : 0);
  outSlots = nd;
  outDraws = em.nSend;  // nSend - 1 shuffle draws, then the send's seed
  if (nd == 0) return;
  CoopSerial cs;
  int base = descAlloc(d, cs, n, nd);
  if (base < 0) return;
  int sub = 0;
  if (em.nSend > 0) {
    Desc ds;
    ds.item = (uint32_t)(d.nLoc + item);
    ds.sub = 0;
    ds.from = (uint32_t)n;
    ds.evKind = EV_MSG;
    ds.meta = em.sendMeta;
    ds.pl = em.sendPl;
    ds.target = 0;
    ds.aux = 0;
    if (em.nSend == 1) {
      ds.dkind = DK_SEND_SINGLE;
      ds.to = em.dst[0];
      ds.nDest = 1;
    } else {
      int off = destAlloc(d, n, 2 * em.nSend);  // destinations, then room for their arrivals
      if (off >= 0)
        for (int i = 0; i < em.nSend; ++i) d.destScratch[off + i] = em.dst[i];
      ds.dkind = DK_SEND_MULTI;
      ds.to = (uint32_t)(off < 0 ? 0 : off);
      ds.nDest = off < 0 ? 0u : (uint32_t)em.nSend;
      ds.aux = DESC_SHUFFLEK;
    }
    d.desc[base + sub] = ds;
    ++sub;
    d.msgSent[n] += em.nSend;
    d.bytesSent[n] += (long long)em.nSend * msgBytes;
  }
  if (em.task) {
    Desc ds;
    ds.dkind = DK_INSERT_AT;
    ds.item = (uint32_t)(d.nLoc + item);
    ds.sub = (uint32_t)sub;
    ds.from = (uint32_t)n;
    ds.to = (uint32_t)n;
    ds.nDest = 0;
    ds.evKind = EV_TASK;
    ds.meta = em.taskMeta;
    ds.pl = em.taskPl;
    ds.target = em.taskAt;
    ds.aux = 0;
    d.desc[base + sub] = ds;
  }
}

// inbox word of a node: (scan item << 32) | index of the bucket entry
WTG_HD u64 inboxMake(int item, int entry) { return ((u64)(uint32_t)item << 32) | (u64)(uint32_t)entry; }
WTG_HD int inboxItem(u64 w) { return (int)(w >> 32); }
WTG_HD int inboxEntry(u64 w) { return (int)(w & 0xFFFFFFFFULL); }

}  // namespace wtg
#include "wtg_handel.cuh"
#include "wtg_casper.cuh"
#include "wtg_cappos.cuh"
#include "wtg_avalanche.cuh"
#include "wtg_p2p.cuh"
namespace wtg {

// ------------------------------------------------------------------------------------------
// one delivery at node n (Network.receiveUntil :603-627 + the protocol's Message.action)
// `ev` is the envelope, item its scan item.  Writes evSlots/evDraws[item].
// ------------------------------------------------------------------------------------------
template <class C>
WTG_HD void deliver(const Dev& d, C& c, int n, const Ev& ev, uint32_t from, uint32_t meta, u64 pl, int item) {
  int slots = 0, draws = 0;
  bool isTask = (ev.kind == EV_TASK || ev.kind == EV_PERIODIC);
  uint32_t envFrom = isTask ? (uint32_t)n : from;  // tasks are self-addressed envelopes (Network.java:505-519)
  bool ok = !d.ndown[n] && d.npart[envFrom] == d.npart[n];  // :606
  if (!ok) {
    // dropped: a pooled payload dies with the envelope
    if (d.proto == PROTO_GSF && (ev.kind == EV_MSG || ev.kind == EV_TASK) && metaKind(meta) == PK_POOL && c.lane() == 0)
      freeDeferred(d, n, (int)metaLevel(meta), (uint32_t)pl);
    if (d.proto == PROTO_HANDEL && (ev.kind == EV_MSG || ev.kind == EV_TASK) && metaKind(meta) == PK_POOL && c.lane() == 0)
      hRelease(d, n, (int)metaLevel(meta), (uint32_t)pl, false);
  } else if (d.proto == PROTO_HANDEL) {
    if (ev.kind == EV_MSG || ev.kind == EV_MULTI) {
      if (c.lane() == 0) {
        d.msgReceived[n] += 1;
        d.bytesReceived[n] += hMsgSize((int)metaLevel(meta));
        statAdd(d, n, ST_DELIVERIES, 1ULL);
        hOnNewSig(d, n, from, meta, pl);
      }
      c.sync();
    } else if (ev.kind == EV_TASK) {
      if (c.lane() == 0) statAdd(d, n, ST_TASKS, 1ULL);
      hUpdate(d, c, n, from, meta, pl, ev.aux, item, slots, draws);
    } else {
      if (c.lane() == 0) statAdd(d, n, ST_TASKS, 1ULL);
      hDissemination(d, c, n, item, slots, draws);
    }
  } else if (d.proto == PROTO_GSF) {
    if (ev.kind == EV_MSG || ev.kind == EV_MULTI) {
      if (c.lane() == 0) {
        d.msgReceived[n] += 1;
        d.bytesReceived[n] += msgSize((int)metaLevel(meta));
        statAdd(d, n, ST_DELIVERIES, 1ULL);
        gsfOnNewSig(d, n, from, meta, pl);
      }
      c.sync();
    } else if (ev.kind == EV_TASK) {
      if (c.lane() == 0) statAdd(d, n, ST_TASKS, 1ULL);
      gsfUpdate(d, c, n, from, meta, pl, item, slots, draws);
    } else {
      if (c.lane() == 0) statAdd(d, n, ST_TASKS, 1ULL);
      gsfDoCycle(d, c, n, item, slots, draws);
    }
  } else if (d.proto == PROTO_CASPER) {
    casperDeliver(d, c, n, ev.kind, meta, pl, item, slots, draws);
  } else if (d.proto == PROTO_CAPPOS) {
    if (c.lane() == 0) cpHandle(d, n, from, meta, pl, item, slots, draws);
    slots = c.bcast(slots, 0);
    draws = c.bcast(draws, 0);
  } else if (d.proto == PROTO_SANFERMIN) {
    if (c.lane() == 0) sfHandle(d, n, from, meta, pl, item, slots, draws);
    slots = c.bcast(slots, 0);
    draws = c.bcast(draws, 0);
  } else if (d.proto == PROTO_SLUSH || d.proto == PROTO_SNOWFLAKE) {
    if (c.lane() == 0) avHandle(d, n, from, meta, pl, item, slots, draws);
    slots = c.bcast(slots, 0);
    draws = c.bcast(draws, 0);
  } else if (d.proto == PROTO_P2PFLOOD) {
    if (c.lane() == 0) floodHandle(d, n, from, pl, item, slots, draws);
    slots = c.bcast(slots, 0);
    draws = c.bcast(draws, 0);
  } else if (d.proto == PROTO_PINGPONG) {
    if (c.lane() == 0) {
      d.msgReceived[n] += 1;
      d.bytesReceived[n] += 1;  // Message.size() default (messages/Message.java:27-29)
      statAdd(d, n, ST_DELIVERIES, 1ULL);
    }
    if (meta == PP_PING) {  // PingPong.java:73-75  onPing: network.send(new Pong(), this, from)
      int base = descAlloc(d, c, n, 1);
      if (c.lane() == 0) {
        if (base >= 0) {
          Desc ds;
          ds.dkind = DK_SEND_SINGLE;
          ds.item = (uint32_t)(d.nLoc + item);
          ds.sub = 0;
          ds.from = (uint32_t)n;
          ds.to = from;
          ds.nDest = 1;
          ds.evKind = EV_MSG;
          ds.meta = PP_PONG;
          ds.pl = 0;
          ds.target = 0;
          ds.aux = 0;
          d.desc[base] = ds;
        }
        d.msgSent[n] += 1;
        d.bytesSent[n] += 1;
      }
      slots = 1;
      draws = 1;
    } else {  // :77-79 onPong
      if (c.lane() == 0) d.pong[n] += 1;
    }
    c.sync();
  }
  if (c.lane() == 0) {
    d.evSlots[item] = slots;
    d.evDraws[item] = draws;
  }
}

// ------------------------------------------------------------------------------------------
// node work item: process this tick's inbox of node n in reference order
// inbox word: (item << 32) | (entry index << 8 ... see below)
// ------------------------------------------------------------------------------------------

// filter 0: every item in reference order (generic).  filter 1: messages only; filter 2: tasks only — used by the
// CUDA handler kernel for GSF / PingPong, where a message delivery (onNewSig: queue, individual-seen row, receive
// counters) and a task (updateVerifiedSignatures / doCycle: verified rows, level scalars, send counters) touch
// disjoint state of the node, so deliveries can run one thread per node and only tasks need a whole warp.
// Returns the number of items skipped by the filter.
template <class C>
WTG_HD int nodeProcess(const Dev& d, C& c, int n, int filter, u64* skippedWord = nullptr) {
  int cnt = d.inboxFill[n];
  if (cnt == 0) return 0;
  const u64* in = d.inbox + d.inboxOff[n];
  const Ev* bucket = d.buckets + (size_t)(d.ctl->tick & (d.ring - 1)) * (size_t)d.bcap;
  int lastItem = -1;
  int skipped = 0;
  for (int r = 0; r < cnt; ++r) {
    // next delivery in reference order = smallest item index not yet processed (inboxes are tiny)
    int bestItem = 0x7fffffff;
    u64 bestW = 0;
    for (int i = c.lane(); i < cnt; i += C::LANES) {
      u64 w = in[i];
      int it = inboxItem(w);
      if (it > lastItem && it < bestItem) {
        bestItem = it;
        bestW = w;
      }
    }
    int mn = c.minv(bestItem);
    uint32_t who = c.ballot(bestItem == mn);
    int src = c.first(who);
    u64 w = c.bcast64(bestW, src);
    lastItem = mn;
    int item = inboxItem(w), entry = inboxEntry(w);
    Ev ev = bucket[entry];
    bool isTask = ev.kind == EV_TASK || ev.kind == EV_PERIODIC;
    if ((filter == 1 && isTask) || (filter == 2 && !isTask)) {
      ++skipped;
      if (skippedWord) *skippedWord = w;
      continue;
    }
    uint32_t from = ev.from, meta = ev.meta;
    u64 pl = ev.pl;
    if (ev.kind == EV_MULTI) {
      const MultiRec& rc = d.rec[ev.aux];
      from = rc.from;
      meta = rc.meta;
      pl = rc.pl;
    }
    deliver(d, c, n, ev, from, meta, pl, item);
  }
  if (c.lane() == 0) {
    if (filter != 2) statMax(d, n, ST_MAXINBOX, (unsigned long long)cnt);
    if (filter == 0 || filter == 2 || skipped == 0) d.inboxFill[n] = 0;  // ready for the next tick
  }
  return skipped;
}
// the only task of node n this tick, handed over by the message pass (saves re-reading the inbox)
template <class C>
WTG_HD void nodeSingleTask(const Dev& d, C& c, int n, u64 w) {
  const Ev* bucket = d.buckets + (size_t)(d.ctl->tick & (d.ring - 1)) * (size_t)d.bcap;
  Ev ev = bucket[inboxEntry(w)];
  deliver(d, c, n, ev, ev.from, ev.meta, ev.pl, inboxItem(w));
  if (c.lane() == 0) d.inboxFill[n] = 0;
}

// ------------------------------------------------------------------------------------------
// dispatch: expand the bucket of this tick into per-node deliveries (thread per event)
// pass 0 counts (subCount, inboxCnt); pass 1 scatters (after itemBase / inboxOff scans)
// ------------------------------------------------------------------------------------------
WTG_HD void dispatchCount(const Dev& d, int i) {
  const Ctl& ctl = *d.ctl;
  int p = ctl.nEv - 1 - i;  // LIFO: processing position (Network.java:145-147)
  const Ev& ev = d.buckets[(size_t)(ctl.tick & (d.ring - 1)) * (size_t)d.bcap + i];
  int m = 1, rep = 0;
  if (ev.kind == EV_MULTI) {
    const MultiRec& rc = d.rec[ev.aux];
    int j = (int)rc.cur;
    m = 0;
    int lastOwner = d.rank;
    while (j < (int)rc.n && d.recArrival[rc.off + j] == ctl.tick) {
      const int to = (int)d.recDest[rc.off + j];
      lastOwner = ownerOf(d, to);
      if (lastOwner == d.rank) {  // node-sharded: the other shards holding this envelope deliver their own destinations
        WTG_ATOMIC_ADD(&d.inboxCnt[to], 1);
        ++m;
      }
      ++j;
    }
    rep = (j < (int)rc.n && lastOwner == d.rank) ? 1 : 0;  // the shard of the group's last destination re-pushes
  } else {
    WTG_ATOMIC_ADD(&d.inboxCnt[ev.to], 1);
  }
  d.subCount[p] = m + rep;
}

// itemBase[p] = exclusive scan of subCount over processing positions
WTG_HD void dispatchScatter(const Dev& d, int i) {
  const Ctl& ctl = *d.ctl;
  int p = ctl.nEv - 1 - i;
  const size_t be = (size_t)(ctl.tick & (d.ring - 1)) * (size_t)d.bcap + i;
  const Ev& ev = d.buckets[be];
  int item0 = d.itemBase[p];
  const u64 bkey = d.G > 1 ? d.bucketKey[be] : 0;
  if (ev.kind == EV_MULTI) {
    MultiRec& rc = d.rec[ev.aux];
    int j = (int)rc.cur, m = 0;
    int lastOwner = d.rank;
    while (j < (int)rc.n && d.recArrival[rc.off + j] == ctl.tick) {
      int to = (int)d.recDest[rc.off + j];
      lastOwner = ownerOf(d, to);
      if (lastOwner == d.rank) {
        int s = d.inboxOff[to] + WTG_ATOMIC_ADD(&d.inboxFill[to], 1);
        d.inbox[s] = inboxMake(item0 + m, i);
        if (d.G > 1) d.itemKey[item0 + m] = bkey | keySub(j);
        ++m;
      }
      ++j;
    }
    if (j < (int)rc.n && lastOwner == d.rank) {  // Network.java:629-632: re-push for the next destination, after the handler ran
      int dst_ = i & (ARENA_STRIPES - 1), dper_ = d.descCap / ARENA_STRIPES;
      int di = WTG_ATOMIC_ADD(&d.ctl->descCnt[dst_], 1);
      bool dok_ = di < dper_;
      di += dst_ * dper_;
      if (dok_) {
        Desc ds;
        ds.dkind = DK_INSERT_AT;
        ds.item = (uint32_t)(d.nLoc + item0 + m);
        ds.sub = 0;
        ds.from = rc.from;
        ds.to = d.recDest[rc.off + j];
        ds.nDest = 0;
        ds.evKind = EV_MULTI;
        ds.meta = 0;
        ds.pl = 0;
        ds.target = d.recArrival[rc.off + j];
        ds.aux = ev.aux;
        d.desc[di] = ds;
      } else {
        setError(d, ERR_DESC_OVERFLOW, di);
      }
      d.evSlots[item0 + m] = 1;
      d.evDraws[item0 + m] = 0;
      if (d.G > 1) d.itemKey[item0 + m] = bkey | keySub(j);
    }
    rc.cur = (uint32_t)j;
  } else {
    int to = (int)ev.to;
    int s = d.inboxOff[to] + WTG_ATOMIC_ADD(&d.inboxFill[to], 1);
    d.inbox[s] = inboxMake(item0, i);
    if (d.G > 1) d.itemKey[item0] = bkey | keySub(0);
  }
}

// Cooperative variants for protocols whose envelopes fan out to thousands of destinations (sendAll): one coop per
// bucket entry; the destinations that arrive in this tick are found by bisection of the sorted arrivals and
// handled a lane each.  Same results as dispatchCount / dispatchScatter.
WTG_HD int multiUpper(const Dev& d, const MultiRec& rc, int tick) {  // first index >= cur whose arrival is after `tick`
  int lo = (int)rc.cur, hi = (int)rc.n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (d.recArrival[rc.off + mid] <= tick)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}
// first destination index of the group a bucket entry stands for: the record's own cursor, or — replicated sendAll records
// of a node-sharded run, where every shard walks its own copy — the index carried by the entry
WTG_HD int multiCur(const Dev& d, const Ev& ev, const MultiRec& rc) { return d.G > 1 ? (int)(uint32_t)ev.pl : (int)rc.cur; }
WTG_HD int multiUpperFrom(const Dev& d, const MultiRec& rc, int cur, int tick) {
  int lo = cur, hi = (int)rc.n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (d.recArrival[rc.off + mid] <= tick)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}
template <class C>
WTG_HD void dispatchCountCoop(const Dev& d, C& c, int i) {
  const Ctl& ctl = *d.ctl;
  int p = ctl.nEv - 1 - i;
  const Ev& ev = d.buckets[(size_t)(ctl.tick & (d.ring - 1)) * (size_t)d.bcap + i];
  if (ev.kind == EV_MULTI) {
    const MultiRec& rc = d.rec[ev.aux];
    if (d.G > 1) {  // node-sharded: this shard delivers its own destinations of the group; the shard of the last one re-pushes
      const int cur = multiCur(d, ev, rc), up = multiUpperFrom(d, rc, cur, ctl.tick);
      int m = 0;
      for (int j0 = cur; j0 < up; j0 += C::LANES) {
        int j = j0 + c.lane();
        bool mine = j < up && ownerOf(d, (int)d.recDest[rc.off + j]) == d.rank;
        if (mine) WTG_ATOMIC_ADD(&d.inboxCnt[d.recDest[rc.off + j]], 1);
        m += c.count(c.ballot(mine));
      }
      const bool rep = up < (int)rc.n && up > cur && ownerOf(d, (int)d.recDest[rc.off + up - 1]) == d.rank;
      if (c.lane() == 0) d.subCount[p] = m + (rep ? 1 : 0);
      return;
    }
    int cur = (int)rc.cur, up = multiUpper(d, rc, ctl.tick);
    for (int j = cur + c.lane(); j < up; j += C::LANES) WTG_ATOMIC_ADD(&d.inboxCnt[d.recDest[rc.off + j]], 1);
    if (c.lane() == 0) d.subCount[p] = (up - cur) + (up < (int)rc.n ? 1 : 0);
  } else if (c.lane() == 0) {
    WTG_ATOMIC_ADD(&d.inboxCnt[ev.to], 1);
    d.subCount[p] = 1;
  }
}
// re-push descriptor of a multi-destination envelope whose next group starts at index `up` (Network.java:629-632)
WTG_HD void writeRepush(const Dev& d, int i, int item, const MultiRec& rc, uint32_t rec, int up) {
  int dst_ = i & (ARENA_STRIPES - 1), dper_ = d.descCap / ARENA_STRIPES;
  int di = WTG_ATOMIC_ADD(&d.ctl->descCnt[dst_], 1);
  if (di < dper_) {
    Desc ds;
    ds.dkind = DK_INSERT_AT;
    ds.item = (uint32_t)(d.nLoc + item);
    ds.sub = 0;
    ds.from = rc.from;
    ds.to = d.recDest[rc.off + up];
    ds.nDest = 0;
    ds.evKind = EV_MULTI;
    ds.meta = 0;
    ds.pl = (u64)(uint32_t)up;  // replicated records: the index the next group starts at
    ds.target = d.recArrival[rc.off + up];
    ds.aux = rec;
    d.desc[dst_ * dper_ + di] = ds;
  } else {
    setError(d, ERR_DESC_OVERFLOW, di);
  }
  d.evSlots[item] = 1;
  d.evDraws[item] = 0;
}
template <class C>
WTG_HD void dispatchScatterCoop(const Dev& d, C& c, int i) {
  const Ctl& ctl = *d.ctl;
  int p = ctl.nEv - 1 - i;
  const size_t be = (size_t)(ctl.tick & (d.ring - 1)) * (size_t)d.bcap + i;
  const Ev& ev = d.buckets[be];
  int item0 = d.itemBase[p];
  const u64 bkey = d.G > 1 ? d.bucketKey[be] : 0;
  if (ev.kind != EV_MULTI) {
    if (c.lane() == 0) {
      int to = (int)ev.to;
      int s = d.inboxOff[to] + WTG_ATOMIC_ADD(&d.inboxFill[to], 1);
      d.inbox[s] = inboxMake(item0, i);
      if (d.G > 1) d.itemKey[item0] = bkey | keySub(0);
    }
    return;
  }
  MultiRec& rc = d.rec[ev.aux];
  if (d.G > 1) {
    const int cur = multiCur(d, ev, rc), up = multiUpperFrom(d, rc, cur, ctl.tick);
    int m = 0;
    for (int j0 = cur; j0 < up; j0 += C::LANES) {
      int j = j0 + c.lane();
      int to = j < up ? (int)d.recDest[rc.off + j] : -1;
      bool mine = j < up && ownerOf(d, to) == d.rank;
      const uint32_t mm = c.ballot(mine);
      const int r = c.rank(mm);
      if (mine) {
        int s = d.inboxOff[to] + WTG_ATOMIC_ADD(&d.inboxFill[to], 1);
        d.inbox[s] = inboxMake(item0 + m + r, i);
        d.itemKey[item0 + m + r] = bkey | keySub(j);
      }
      m += c.count(mm);
    }
    c.sync();
    if (c.lane() == 0 && up < (int)rc.n && up > cur && ownerOf(d, (int)d.recDest[rc.off + up - 1]) == d.rank) {
      writeRepush(d, i, item0 + m, rc, ev.aux, up);
      d.itemKey[item0 + m] = bkey | keySub(up);
    }
    c.sync();
    return;
  }
  const int cur = (int)rc.cur, up = multiUpper(d, rc, ctl.tick), m = up - cur;
  for (int j = cur + c.lane(); j < up; j += C::LANES) {
    int to = (int)d.recDest[rc.off + j];
    int s = d.inboxOff[to] + WTG_ATOMIC_ADD(&d.inboxFill[to], 1);
    d.inbox[s] = inboxMake(item0 + (j - cur), i);
  }
  c.sync();
  if (c.lane() == 0) {
    if (up < (int)rc.n) writeRepush(d, i, item0 + m, rc, ev.aux, up);
    rc.cur = (uint32_t)up;
  }
  c.sync();
}

// ------------------------------------------------------------------------------------------
// emit: turn one descriptor into a new envelope (seed -> latency -> arrival), in creation order
// ------------------------------------------------------------------------------------------
// A multi-destination send with more destinations than MAX_ACC (only the caller issues those: network.send(msg, from, dests),
// Network.java:352-362): the arrivals live next to the destination list in destScratch ([nDest] ids, then [nDest] arrivals) and
// are sorted there (createMessageArrivals :449-467, stable); the envelope choice is the same (:435-446).  Unsharded only.
WTG_HD void emitBigMulti(const Dev& d, const Desc& ds, int g, int32_t seed, int sendTime, int step, Ev ev) {
  const Ctl& ctl = *d.ctl;
  const int m = (int)ds.nDest, from = (int)ds.from;
  uint32_t* list = d.destScratch + ds.to;
  int* arr = reinterpret_cast<int*>(d.destScratch + ds.to + m);
  int cnt = 0;
  for (int i = 0; i < m; ++i) {
    int to = (int)list[i];
    if (d.npart[from] == d.npart[to] && !d.ndown[from] && !d.ndown[to]) {
      int nt = latency(d, from, to, pseudoRandom(to, seed));
      if (nt < d.msgDiscardTime) {
        int a = sendTime + i * step + nt;
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
  if (target >= 0 && cnt > 0 && arr[cnt - 1] - ctl.tick >= d.ring) {  // a record's arrivals must all lie inside the ring
    setError(d, ERR_FAR_FUTURE, arr[cnt - 1]);
    target = -1;
  }
  d.newEv[g] = ev;
  d.newTarget[g] = target;
}

WTG_HD void emitDesc(const Dev& d, int di) {
  const Ctl& ctl = *d.ctl;
  const Desc& ds = d.desc[di];
  if (ds.dkind == DK_SEND_ALL) return;  // built by emitAll
  const bool shard = d.G > 1;
  int g = d.slotBase[ds.item] + (int)ds.sub;
  if (shard) g += (int)d.xoffS[ds.item - d.nLoc];  // creation indices of the other shards that come first
  if (g >= d.newEvCap) {
    setError(d, ERR_DESC_OVERFLOW, g);
    return;
  }
  Ev ev;
  ev.kind = ds.evKind;
  ev.to = ds.to;
  ev.from = ds.from;
  ev.meta = ds.meta;
  ev.pl = ds.pl;
  ev.aux = ds.dkind == DK_INSERT_AT ? ds.aux : 0;
  ev.pad = (uint32_t)ctl.tick + 1u;  // sendTime + 1 of sendArriveAt / registerTask (Network.java:390, 509): EnvelopeInfo.sentAt
  int target = -1;
  int sendTime = ctl.tick + 1;  // send(m, from, to) == send(m, time + 1, from, to)   Network.java:364-366
  if (ds.dkind == DK_INSERT_AT) {
    target = ds.target;
    if (shard && ds.evKind == EV_MULTI && d.allCap > 0) {  // sendAll record, replicated on every shard: entries only
      xPlaceReplicated(d, g, (int)ds.aux, (int)(uint32_t)ds.pl);
      return;
    }
    if (shard && ds.evKind == EV_MULTI) {  // re-push of a multi-destination envelope: its next arrivals may lie on other shards
      const MultiRec& rc = d.rec[ds.aux];
      xPlaceMulti(d, g, rc.from, rc.meta, rc.pl, (int)rc.n, (int)rc.cur, d.recDest + rc.off, d.recArrival + rc.off, (int)ds.aux, rc.pad);
      return;
    }
  } else {
    u64 drawIdx = (u64)(d.drawBase[ds.item] + (int)ds.sub);
    if (shard) drawIdx += (u64)d.xoffD[ds.item - d.nLoc];
    if (d.shufCap > 0) {  // protocols with k-element shuffles or samples: draws per descriptor vary (wtg_cappos.cuh)
      drawIdx = ctl.shufReject ? (u64)d.descDraw[di] : descDrawOptimistic(d, di);
      if (ds.aux & DESC_PEERS) {  // built by emitPeers (wtg_p2p.cuh): on the device by k_emit_peers, a warp per forward
#if !defined(__CUDA_ARCH__)
        // the host build of these bodies has no separate warp pass: it runs the same body here with a one-lane group
        CoopSerial cs;
        uint32_t list[PEERS_MAX];
        int arr[PEERS_MAX];
        emitPeers(d, cs, di, list, arr);
#endif
        return;
      }
      if (ds.dkind == DK_SEND_MULTI && (ds.aux & (DESC_SHUFFLEK | DESC_SAMPLEK))) {
        emitShuffled(d, di, g, drawIdx);
        return;
      }
    }
    bool swap01 = false;
    if (ds.dkind == DK_SEND_MULTI && (ds.aux & DESC_SHUFFLE2)) {
      // Collections.shuffle of a 2-element list: swap(list, 1, rnd.nextInt(2))  (SanFerminHelper.java:155)
      u64 st = lcgAdvance(d.jumpA, d.jumpC, ctl.rng, drawIdx + 1);
      int32_t r31 = (int32_t)(uint32_t)(st >> 17);
      swap01 = (int)(((long long)2 * (long long)r31) >> 31) == 0;
      drawIdx += 1;
    }
    int32_t seed = lcgNextIntAt(d, ctl.rng, drawIdx);
    int from = (int)ds.from;
    if (ds.aux & DESC_SENDTIME) sendTime = ds.target;
    ev.pad = (uint32_t)sendTime + 1u;
    const int delay = (int)(ds.aux >> DESC_DELAY_SHIFT);
    const int step = delay > 0 ? delay + 1 : 0;  // sendTime += delaysBetweenMessage + 1 after every destination (:455-459)
    if (ds.dkind == DK_SEND_MULTI && (int)ds.nDest > MAX_ACC) {
      if (shard)
        setError(d, ERR_UNSUPPORTED, 8);
      else
        emitBigMulti(d, ds, g, seed, sendTime, step, ev);
      return;
    }
    if (ds.dkind == DK_SEND_SINGLE) {
      int to = (int)ds.to;
      // createMessageArrival :478-484
      if (d.npart[from] == d.npart[to] && !d.ndown[from] && !d.ndown[to]) {
        int nt = latency(d, from, to, pseudoRandom(to, seed));
        if (nt < d.msgDiscardTime) target = sendTime + nt;
      }
    } else {
      // createMessageArrivals :449-467 + envelope choice :435-446
      uint32_t dst[MAX_ACC];
      int arr[MAX_ACC];
      int cnt = 0;
      for (int i = 0; i < (int)ds.nDest; ++i) {
        int to = (int)d.destScratch[ds.to + ((swap01 && i < 2) ? 1 - i : i)];
        if (d.npart[from] == d.npart[to] && !d.ndown[from] && !d.ndown[to]) {
          int nt = latency(d, from, to, pseudoRandom(to, seed));
          if (nt < d.msgDiscardTime) {
            int a = sendTime + i * step + nt;
            int j = cnt++;  // stable insertion sort by arrival (Collections.sort is stable)
            while (j > 0 && arr[j - 1] > a) {
              arr[j] = arr[j - 1];
              dst[j] = dst[j - 1];
              --j;
            }
            arr[j] = a;
            dst[j] = (uint32_t)to;
          }
        }
      }
      if (cnt == 1) {
        ev.to = dst[0];
        target = arr[0];
      } else if (cnt > 1 && shard) {
        if (arr[cnt - 1] - ctl.tick >= d.ring) {
          setError(d, ERR_FAR_FUTURE, arr[cnt - 1]);
          return;
        }
        xPlaceMulti(d, g, ds.from, ds.meta, ds.pl, cnt, 0, dst, arr, -1, (uint32_t)sendTime + 1u);
        return;
      } else if (cnt > 1) {
        ev.aux = 0;
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
            d.recDest[off + i] = dst[i];
            d.recArrival[off + i] = arr[i];
          }
          ev.kind = EV_MULTI;
          ev.to = dst[0];
          ev.aux = (uint32_t)ri;
          target = arr[0];
        }
      }
    }
    // a dropped envelope takes its pooled payload with it: GSF's slab has no other owner, Handel's holds only the envelope's
    // reference (hMakePayload).  A staged payload is never ingested (its staging area is reset every pass).
    if (target < 0 && (d.proto == PROTO_GSF || d.proto == PROTO_HANDEL) && metaKind(ds.meta) == PK_POOL && !(ds.meta & META_STAGED))
      freeDirect(d, (int)metaLevel(ds.meta), (uint32_t)ds.pl);
    else if (target >= 0 && shard && d.proto == PROTO_HANDEL && metaKind(ds.meta) == PK_POOL && ownerOf(d, (int)ev.to) != d.rank)
      hStageAtEmit(d, ev);
  }
  if (d.farCap > 0) {
    if (target >= 0 && target - ctl.tick >= farHorizon(d)) {
      if (shard && ownerOf(d, (int)ev.to) != d.rank)  // the calendar is local: far-future envelopes are tasks of the shard's own nodes
        setError(d, ERR_UNSUPPORTED, 7);
      else
        farAppend(d, ev, target, g);
      target = -1;
    }
  } else if (target >= 0 && target - ctl.tick >= d.ring) {
    setError(d, ERR_FAR_FUTURE, target);
    target = -1;
  }
  if (shard) {  // straight into the arrays of the shard that owns the destination; dropped envelopes leave no trace
    if (target >= 0) xStoreEnvelope(d, ownerOf(d, (int)ev.to), g, ev, target);
    return;
  }
  d.newEv[g] = ev;
  d.newTarget[g] = target;
}

// conditional-task inserts come first in creation order (slot = scan over nodes)
WTG_HD void emitCond(const Dev& d, int n) {
  const size_t h = condHalf(d, d.ctl->tick);
  if (!d.condFired[h + n]) return;
  int g = d.slotBase[n - d.n0];
  if (d.G > 1) g += d.ctl->condXoffS;  // the lower shards' nodes come first
  if (g >= d.newEvCap) {
    setError(d, ERR_DESC_OVERFLOW, g);
    return;
  }
  int target = d.condTarget[h + n];
  if (target - d.ctl->tick >= d.ring) {
    setError(d, ERR_FAR_FUTURE, target);
    target = -1;
  }
  if (d.G > 1 && target < 0) return;
  d.newEv[g] = d.condEv[h + n];
  d.newTarget[g] = target;
}

// ------------------------------------------------------------------------------------------
// tick bookkeeping (single thread)
// ------------------------------------------------------------------------------------------
// condAhead: this pass's checkSigs has already run, beside the previous pass's emission (k_cond_begin set its clock and
// counters)
WTG_HD void tickBegin(const Dev& d, int mode, bool condAhead = false) {
  Ctl& c = *d.ctl;
  if (mode == 1) {
    c.time += 1;  // nextMessage(): time++   (Network.java:541)
    c.tick = c.time;
    c.condMode = 1;
    c.nEv = d.bucketCount[c.tick & (d.ring - 1)];
  } else if (mode == 0) {
    c.tick = c.time;
    c.condMode = 0;
    c.nEv = d.bucketCount[c.tick & (d.ring - 1)];
  } else {  // the extra time++ past `until`; runMs then forces time = endAt (Network.java:336)
    c.tick = c.time + 1;
    c.condMode = 2;
    c.nEv = 0;
  }
  for (int t = 0; t < ARENA_STRIPES; ++t) {
    c.descCnt[t] = 0;
    c.destCnt[t] = 0;
    if (!condAhead) {
      c.workCnt[t] = 0;
      c.dueCnt[t] = 0;
    }
    c.taskCnt[t] = 0;
  }
  if (!condAhead) {
    c.condTick = c.tick;
    c.condCall = c.callId;
  }
  c.nItems = 0;
  c.totalSlots = 0;
  c.totalDraws = 0;
  c.hReject = 0;
  c.allCnt = 0;
  c.allRecBase = c.recTop;
  c.shufReject = 0;
  c.peerCnt = 0;
  if (c.nEv > c.maxBucket) c.maxBucket = c.nEv;
  if (d.G > 1) {
    c.xseq += 1;
    c.nEvGlobal = 0;
    for (int q = 0; q < MAX_SHARDS; ++q) c.stageTop[q] = 0;
  }
}
// tickBegin for protocols that keep the far-future calendar but tick every millisecond (conditional tasks): the calendar
// entries that come within the horizon of this tick move to the head of their buckets first (one coop)
template <class C>
WTG_HD void tickBeginFar(const Dev& d, C& c, int mode, bool condAhead = false) {
  if (mode != 2) farMigrate(d, c, mode == 1 ? d.ctl->time + 1 : d.ctl->time);
  c.sync();
  if (c.lane() == 0) tickBegin(d, mode, condAhead);
  c.sync();
}
// GSF's pool low-water mark, sampled every 16 ticks after the pass's deferred frees
WTG_HD void samplePoolMinFree(const Dev& d) {
  Ctl& c = *d.ctl;
  if (d.proto == PROTO_GSF && (c.tick & 15) == 0)
    for (int l = INLINE_MAX_LEVEL + 1; l < d.L; ++l) {
      int f = 0;
      for (int t = 0; t < POOL_STRIPES; ++t) f += c.poolFreeCnt[l][t];
      if (f < c.poolMinFree[l]) c.poolMinFree[l] = f;
    }
}
// condAhead: the next pass's checkSigs ran beside this pass's emission; condBegin took the sample before its evictions
WTG_HD void tickEnd(const Dev& d, int mode, bool condAhead = false) {
  Ctl& c = *d.ctl;
  c.rng = lcgAdvance(d.jumpA, d.jumpC, c.rng, (u64)c.totalDraws);
  c.statDraws += (unsigned long long)c.totalDraws;
  c.statEvents += (unsigned long long)c.nItems;
  if ((d.G > 1 ? c.nEvGlobal : c.nEv) > 0) {
    c.callId += 1;  // every processed message starts a new nextMessage() call
    c.didSomething = 1;
  }
  if (mode != 2 && mode != 3) d.bucketCount[c.tick & (d.ring - 1)] = 0;  // 3: host-injected sends at the current time
  for (int t = 0; t < ARENA_STRIPES; ++t) c.freeCnt[t] = 0;
  if (d.proto == PROTO_CASPER && d.G > 1 && d.cg->createdThisTick > 1) setError(d, ERR_UNSUPPORTED, 4);  // unsharded: casperRenumber
  if (d.G > 1 && d.allCap > 0 && mode != 3) c.allSeq = (int)(((unsigned)c.allSeq + (unsigned)xAllTotal(d)) & 0x3fffffffu);  // record slots of the next pass
  if (!condAhead) samplePoolMinFree(d);
}
// Unsharded GSF, mode 1, after the handlers and the deferred frees of pass `tick` and before the checkSigs of pass tick + 1
// runs ahead: that checkSigs's clock (the callId tickEnd will leave), condMode and counters, which the next tickBegin then
// leaves alone; and this pass's pool sample, which the evictions of that checkSigs must not reach.
WTG_HD void condBegin(const Dev& d) {
  Ctl& c = *d.ctl;
  samplePoolMinFree(d);
  c.condTick = c.tick + 1;
  c.condCall = c.callId + (c.nEv > 0 ? 1u : 0u);
  c.condMode = 1;
  for (int t = 0; t < ARENA_STRIPES; ++t) {
    c.workCnt[t] = 0;
    c.dueCnt[t] = 0;
  }
}
// deferred frees -> pool free stacks (no allocation runs concurrently).  i indexes the striped list.
WTG_HD void freeApply(const Dev& d, int i) {
  uint32_t w = d.freeList[i];
  freeDirect(d, (int)(w >> 27), w & 0x7FFFFFFu);
}
// map a dense work index onto the striped arena: returns the arena index or -1
WTG_HD int stripedIndex(const int* cnt, int per, int t) {
  for (int s = 0; s < ARENA_STRIPES; ++s) {
    int c = cnt[s];
    if (c > per) c = per;
    if (t < c) return s * per + t;
    t -= c;
  }
  return -1;
}
WTG_HD int stripedTotal(const int* cnt, int per) {
  int tot = 0;
  for (int s = 0; s < ARENA_STRIPES; ++s) tot += cnt[s] > per ? per : cnt[s];
  return tot;
}

// ------------------------------------------------------------------------------------------
// GSF init bodies
// ------------------------------------------------------------------------------------------
WTG_HD void gsfInitNodeBody(const Dev& d, int n) {  // GSFNode ctor :176-179, SFLevel ctors :260-280
  d.verified[(size_t)n * d.W64 + (n >> 6)] = 1ULL << (n & 63);
  d.totalCard[n] = 1;
  d.minStart[n] = 1;  // registerConditionalTask(checkSigs, 1, nodePairingTime, ...) :631-632
  if (!d.ndown[n]) {  // initLevel() runs for live nodes only (:627-629)
    d.cntVer[n * d.L] = 1;
    d.cntUnion[n * d.L] = 1;
    for (int l = 1; l < d.L; ++l) d.remaining[n * d.L + l] = 1 << (l - 1);
  }
  for (int l = 0; l < d.L; ++l) d.lvVer[n * d.L + l] = 1;
}

// positions in [start, start+len) of the stream after s0 whose next(31) value could be rejected by
// nextInt(bound) for some bound <= maxBound (u >= 2^31 - maxBound)
WTG_HD void rngCandidateChunk(const Dev& d, u64 s0, u64 start, u64 len, int maxBound, u64* out, int* outCount, int cap) {
  u64 s = lcgAdvance(d.jumpA, d.jumpC, s0, start);
  const uint32_t thr = 0x80000000u - (uint32_t)maxBound;
  for (u64 i = 0; i < len; ++i) {
    s = (s * 0x5DEECE66DULL + 0xBULL) & LCG_MASK;
    uint32_t u = (uint32_t)(s >> 17);
    if (u >= thr) {
      int k = WTG_ATOMIC_ADD(outCount, 1);
      if (k < cap) out[k] = start + i;
    }
  }
}

// Collections.shuffle(peers_l, network.rd) for one (node, level)  (GSFSignature.java:462-476)
template <class PeerT>
WTG_HD void gsfShuffleLevel(const Dev& d, int n, int l, u64 s0, const int* liveRank, const u64* rejOrd, int nRej) {
  int r = liveRank[n];
  if (r < 0) return;
  const int size = 1 << (l - 1);
  const int sib = levelBlock(n ^ (1 << (l - 1)), l).base;
  PeerT* arr = (PeerT*)d.peers + (size_t)n * (size_t)(d.N - 1) + (size_t)(size - 1);
  const PeerT add = sizeof(PeerT) == 2 ? (PeerT)0 : (PeerT)sib;
  for (int i = 0; i < size; ++i) arr[i] = (PeerT)(add + (PeerT)i);  // ids in increasing order (nextSetBit walk)
  if (size < 2) return;
  const u64 D = (u64)(d.N - d.L);
  u64 q = (u64)r * D + ((1ULL << (l - 1)) - (u64)l);
  int lo = 0, hi = nRej;  // rejections before ordinal q shift the stream position
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (rejOrd[mid] < q)
      lo = mid + 1;
    else
      hi = mid;
  }
  u64 s = lcgAdvance(d.jumpA, d.jumpC, s0, q + (u64)lo);
  for (int i = size; i > 1; --i) {
    int j;
    s = (s * 0x5DEECE66DULL + 0xBULL) & LCG_MASK;
    int32_t rr = (int32_t)(uint32_t)(s >> 17);
    if ((i & (i - 1)) == 0) {
      j = (int)(((long long)i * (long long)rr) >> 31);
    } else {
      int32_t u = rr;
      for (;;) {
        j = u % i;
        if ((int32_t)((uint32_t)u - (uint32_t)j + (uint32_t)(i - 1)) >= 0) break;
        s = (s * 0x5DEECE66DULL + 0xBULL) & LCG_MASK;
        u = (int32_t)(uint32_t)(s >> 17);
      }
    }
    PeerT t = arr[i - 1];
    arr[i - 1] = arr[j];
    arr[j] = t;
  }
}

// scan item accessors (pair scans)
//   scan A: [0,nEv) -> (subCount, 0);  [nEv, nEv+N) -> (0, inboxCnt)
//   scan B: [0,N)   -> (condFired, 0); [N, N+nItems) -> (evSlots, evDraws)
struct Pair {
  int a, b;
};
WTG_HD Pair scanLoad(const Dev& d, int which, int j) {
  Pair p;
  if (which == 2) {  // Handel: draws of the conditional pass, over nodes
    p.a = d.condDraws[d.n0 + j];
    p.b = 0;
    return p;
  }
  if (which == 0) {
    int nEv = d.ctl->nEv;
    if (j < nEv) {
      p.a = d.subCount[j];
      p.b = 0;
    } else {
      p.a = 0;
      p.b = d.inboxCnt[d.n0 + j - nEv];
    }
  } else {
    if (j < d.nLoc) {
      p.a = d.condFired[condHalf(d, d.ctl->tick) + d.n0 + j];
      p.b = d.condDraws[d.n0 + j];
    } else {
      p.a = d.evSlots[j - d.nLoc];
      p.b = d.evDraws[j - d.nLoc];
    }
  }
  return p;
}
WTG_HD int scanCount(const Dev& d, int which) { return which == 2 ? d.nLoc : which == 0 ? d.ctl->nEv + d.nLoc : d.nLoc + d.ctl->nItems; }
WTG_HD void scanStore(const Dev& d, int which, int j, Pair ex) {
  if (which == 2) {
    d.hDrawBase[d.n0 + j] = ex.a;
    return;
  }
  if (which == 0) {
    int nEv = d.ctl->nEv;
    if (j < nEv)
      d.itemBase[j] = ex.a;
    else {
      d.inboxOff[d.n0 + j - nEv] = ex.b;
      d.inboxCnt[d.n0 + j - nEv] = 0;
    }
  } else {
    d.slotBase[j] = ex.a;
    d.drawBase[j] = ex.b;
  }
}
WTG_HD void scanTotals(const Dev& d, int which, Pair tot) {
  if (which == 2) return;
  if (which == 0) {
    d.ctl->nItems = tot.a;
    if (tot.a > d.itemCap || tot.b > d.itemCap) setError(d, ERR_INBOX_OVERFLOW, tot.a);
  } else {
    d.ctl->totalSlots = tot.a;
    d.ctl->totalDraws = tot.b;
    if (tot.a > d.newEvCap) setError(d, ERR_DESC_OVERFLOW, tot.a);
  }
}

}  // namespace wtg
