// wittgenstein_b200 — engine orchestration: owns the device state, runs protocol init and the
// runMs tick loop through a Backend (the CUDA backend in wtg_cuda.cu; a host backend exists only
// under tests/emu for debugging the exact-order logic).
//
// Reference surface mirrored here (core/Network.java): runMs :318-338, setNetworkLatency
// :665-677, partition :693-707, msgs.size() :204-210, time :49, rd :32; Protocol.init() of
// protocols/PingPong.java:82-87 and protocols/GSFSignature.java:611-635.
#pragma once
#include <chrono>
#include <cstdio>
#include <functional>
#include <thread>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "wtg_host.hpp"
#include "wtg_logic.cuh"
#include "wtg_types.h"

namespace wtg {

struct GsfParams {
  int nodeCount, threshold, pairingTime, timeoutPerLevelMs, periodDurationMs, acceleratedCallsCount, nodesDown;
};

struct SfParams {
  int nodeCount, threshold, pairingTime, signatureSize, replyTimeout, candidateCount;
};

struct HandelParams {
  int nodeCount, threshold, pairingTime, levelWaitTime, extraCycle, disseminationPeriodMs, fastPath, nodesDown, desynchronizedStart,
      byzantineSuicide, hiddenByzantine;
};

struct CapposParams {  // SanFerminCappos.SanFerminParameters (protocols/SanFerminCappos.java:86-103), constructor order
  int nodeCount, threshold, pairingTime, signatureSize, timeout, candidateCount;
};

struct CasperParams {  // CasperParemeters (protocols/CasperIMD.java:18-71), in declaration order
  int cycleLength, randomOnTies, blockProducersCount, attestersPerRound, blockConstructionTime, attestationConstructionTime;
};

struct Tunables {  // capacities; 0 = derive from N
  long long bcap = 0, qcap = 0, poolSlotsPerNode = 0, descCap = 0, recCap = 0, ring = 0;
  long long casperVotes = 0;   // CasperIMD: attestations one attester may publish in a run (default 6)
  long long casperBlocks = 0;  // CasperIMD: blocks of a run (default from casperVotes)
  long long peerBits32 = 0;    // GSF: absolute 32-bit peer ids even when 16-bit block-relative ones would do
  long long farCap = 0;        // far-future calendar entries (latency models with multi-second arrivals)
  long long stageWords = 0;    // node-sharded GSF: staging capacity per (sending shard, pass parity) in 64-bit words
};

struct Backend {
  virtual ~Backend() {}
  virtual void* alloc(size_t bytes) = 0;  // zero-initialised device memory
  virtual void release(void* p) = 0;
  virtual void upload(void* dst, const void* src, size_t bytes) = 0;
  virtual void download(void* dst, const void* src, size_t bytes) = 0;
  virtual void sync() = 0;
  // one tick of the pipeline; mode 0 = messages of the current time only, 1 = clock tick + conditional
  // tasks + messages, 2 = end-of-window conditional pass
  virtual void tick(const Dev& d, int mode) = 0;
  // `count` consecutive mode-1 ticks (lets the CUDA backend replay a captured graph)
  virtual void ticks(const Dev& d, int count) {
    for (int i = 0; i < count; ++i) tick(d, 1);
  }
  // device-side timing (CUDA events on the engine's stream); no-ops on backends without a device
  virtual void timerStart() {}
  virtual double timerStopMs() { return 0.0; }
  virtual void profileEnable(bool, bool) {}  // (on, report the dispatch's scan A apart from scan B)
  virtual int profileRead(double* ms, long long* launches, const char** names, int cap) { (void)ms; (void)launches; (void)names; (void)cap; return 0; }
  // node-sharded runs: one exchange region per shard that the other shards' kernels write into.  `allocShared` returns
  // zero-initialised memory that can be mapped by other processes; exportShared / importShared carry the 64-byte handle
  // (CUDA IPC); backends whose shards live in one address space never need them.
  virtual void* allocShared(size_t bytes) { return alloc(bytes); }
  // handle: SHARD_HANDLE_BYTES = 128 bytes: [0,64) interprocess handle, [64,72) process id, [72,80) address, [80,84) device
  virtual void exportShared(void* p, unsigned char* handle) {
    std::memset(handle, 0, 128);
    std::memcpy(handle + 72, &p, sizeof(p));
  }
  virtual void* importShared(const unsigned char* handle) {
    void* p;
    std::memcpy(&p, handle + 72, sizeof(p));
    return p;
  }
  virtual int deviceId() const { return 0; }
  virtual void gsfInitNodes(const Dev& d) = 0;
  // scan `count` stream positions after state s0 for values that nextInt(bound<=maxBound) could reject
  virtual void rngCandidates(const Dev& d, unsigned long long s0, unsigned long long count, int maxBound,
                             std::vector<unsigned long long>& out) = 0;
  // Fisher-Yates of every (live node, level) peer list; rejOrd = sorted ordinals of rejected draws
  virtual void gsfShufflePeers(const Dev& d, unsigned long long s0, const int* liveRank, const unsigned long long* rejOrd, int nRej) = 0;
};

class Engine {
 public:
  std::unique_ptr<Backend> be;
  HostModel hm;
  Dev d;
  Tunables tun;
  std::vector<void*> allocs;
  bool inited = false;
  int time = 0;
  int ringMask = 0;
  bool pendingAtNow = false;  // host inserted an event arriving at the current time
  std::vector<int> partitionsInX;
  int msgDiscardTime = 0x7fffffff;
  std::string err;
  std::vector<int> liveRank;  // GSF: rank among live nodes, -1 when down
  unsigned long long initDraws = 0;

  // ---- node-sharded simulation: this engine is shard `shardRank` of `shardWorld` (set before init) ----
  int shardRank = 0, shardWorld = 1;
  bool linked = false;          // peers' exchange regions are mapped
  void* xRegion = nullptr;      // this shard's exchange region
  size_t xBytes = 0;
  long long stageWordsWanted = 0;  // protocol-specific staging capacity per (sender, parity), in 64-bit words
  long long farWanted = 0;         // protocol-specific size of the far-future calendar when the latency model needs one
  struct XLayout {
    size_t hdr, flags, items, newEv, newTarget, stage, rec, recDest, recArrival, beg, all, allCnt, proto, total;
  } xl{};
  // protocol-specific parts of the exchange region, set before allocCommon (CasperIMD: replicated block / attestation tables,
  // sendAll descriptors of a pass; Handel: the pick exchange); unevenShards: the protocol's node count need not split into
  // power-of-two shards
  size_t xProtoBytes = 0;
  int xAllCapWanted = 0;
  bool unevenShards = false;
  bool shardFarOk = false;  // the protocol's far-future envelopes are tasks of the shard's own nodes

  explicit Engine(Backend* b) : be(b) { std::memset(&d, 0, sizeof(d)); }
  void setShard(int rank, int world) {
    requireNotInited();
    if (world < 1 || world > MAX_SHARDS || (world & (world - 1)) != 0) throw std::invalid_argument("the number of shards must be a power of two <= 8");
    if (rank < 0 || rank >= world) throw std::invalid_argument("shard rank");
    shardRank = rank;
    shardWorld = world;
  }
  bool sharded() const { return shardWorld > 1; }
  void requireUnsharded(const char* what) const {
    if (sharded()) throw std::logic_error(std::string(what) + " is not available on a node-sharded network");
  }
  // per-node arrays of a shard hold nLoc rows and are addressed by global id: the base is biased by -n0 rows
  template <class T>
  T* dallocNodes(size_t perNode = 1) {
    T* p = dalloc<T>((size_t)d.nLoc * perNode);
    return p - (size_t)d.n0 * perNode;
  }
  template <class T>
  T* duploadNodes(const std::vector<T>& full, size_t perNode = 1) {  // `full` holds all N rows; the shard keeps its own
    T* p = dalloc<T>((size_t)d.nLoc * perNode);
    be->upload(p, full.data() + (size_t)d.n0 * perNode, (size_t)d.nLoc * perNode * sizeof(T));
    return p - (size_t)d.n0 * perNode;
  }
  Peer peerView(void* base) const {
    char* b = (char*)base;
    Peer q;
    q.hdr = (XHdr*)(b + xl.hdr);
    q.flags = (int*)(b + xl.flags);
    q.items = (XItem*)(b + xl.items);
    q.newEv = (Ev*)(b + xl.newEv);
    q.newTarget = (int*)(b + xl.newTarget);
    q.stage = (unsigned long long*)(b + xl.stage);
    q.rec = (MultiRec*)(b + xl.rec);
    q.recDest = (uint32_t*)(b + xl.recDest);
    q.recArrival = (int*)(b + xl.recArrival);
    q.beg = (XBegin*)(b + xl.beg);
    q.all = (XAll*)(b + xl.all);
    q.allCnt = (int*)(b + xl.allCnt);
    q.proto = b + xl.proto;
    return q;
  }
  // exchange region: everything another shard's kernels write (one allocation = one IPC handle)
  void allocExchange() {
    auto al = [](size_t x) { return (x + 255) / 256 * 256; };
    size_t o = 0;
    xl.hdr = o;        o += al(sizeof(XHdr) * MAX_SHARDS);
    xl.flags = o;      o += al(sizeof(int) * 4 * MAX_SHARDS);
    xl.items = o;      o += al(sizeof(XItem) * (size_t)d.G * d.xItemCap);
    xl.newEv = o;      o += al(sizeof(Ev) * (size_t)d.newEvCap);
    xl.newTarget = o;  o += al(sizeof(int) * (size_t)d.newEvCap);
    xl.stage = o;      o += al(sizeof(unsigned long long) * 2 * (size_t)d.G * (size_t)d.stageCapWords);
    xl.rec = o;        o += al(sizeof(MultiRec) * (size_t)d.recCap);
    xl.recDest = o;    o += al(sizeof(uint32_t) * (size_t)d.recDestCap);
    xl.recArrival = o; o += al(sizeof(int) * (size_t)d.recDestCap);
    xl.beg = o;        o += al(sizeof(XBegin) * MAX_SHARDS);
    xl.all = o;        o += al(sizeof(XAll) * (size_t)d.G * (size_t)std::max(1, d.xAllCap));
    xl.allCnt = o;     o += al(sizeof(int) * MAX_SHARDS);
    xl.proto = o;      o += al(xProtoBytes);
    xl.total = o;
    xBytes = o;
    xRegion = be->allocShared(o);
    allocs.push_back(xRegion);
    for (int q = 0; q < MAX_SHARDS; ++q) std::memset(&d.peer[q], 0, sizeof(Peer));
    d.peer[d.rank] = peerView(xRegion);
    d.newEv = d.peer[d.rank].newEv;
    d.newTarget = d.peer[d.rank].newTarget;
    d.rec = d.peer[d.rank].rec;
    d.recDest = d.peer[d.rank].recDest;
    d.recArrival = d.peer[d.rank].recArrival;
    std::vector<int> m1((size_t)d.newEvCap, -1);  // "nothing for this shard"
    be->upload(d.newTarget, m1.data(), m1.size() * sizeof(int));
  }
  void exportExchange(unsigned char* handle128) {
    requireInited();
    if (!sharded()) throw std::logic_error("not a node-sharded network");
    be->exportShared(xRegion, handle128);
  }
  // handles: world x 128 bytes, in rank order (the own entry is ignored)
  void linkExchange(const unsigned char* handles) {
    requireInited();
    if (!sharded()) throw std::logic_error("not a node-sharded network");
    for (int q = 0; q < shardWorld; ++q) {
      if (q == shardRank) continue;
      d.peer[q] = peerView(be->importShared(handles + (size_t)q * 128));
    }
    linked = true;
  }
  ~Engine() { freeAll(); }

  void freeAll() {
    for (void* p : allocs) be->release(p);
    allocs.clear();
  }
  template <class T>
  T* dalloc(size_t n) {
    void* p = be->alloc(std::max<size_t>(n, 1) * sizeof(T));
    allocs.push_back(p);
    return (T*)p;
  }
  template <class T>
  T* dupload(const std::vector<T>& v) {
    T* p = dalloc<T>(v.size());
    if (!v.empty()) be->upload(p, v.data(), v.size() * sizeof(T));
    return p;
  }
  void requireNotInited() const {
    if (inited) throw std::logic_error("network already initialised");
  }
  void requireInited() const {
    if (!inited) throw std::logic_error("protocol not initialised");
  }

  // ---- configuration (before init) ----
  void setSeed(long long s) {
    requireNotInited();
    hm.rd.setSeed(s);
  }

  // ---- common device state ----
  void allocCommon(int N, int proto) {
    d.N = N;
    d.proto = proto;
    d.G = shardWorld;
    d.rank = shardRank;
    if (N % shardWorld != 0 && !unevenShards) throw std::invalid_argument("the node count must be a multiple of the number of shards");
    d.perShard = (N + shardWorld - 1) / shardWorld;
    d.n0 = shardRank * d.perShard;
    d.nLoc = std::min(d.perShard, N - d.n0);
    if (d.nLoc <= 0) throw std::invalid_argument("more shards than the node count can fill");
    d.ownShift = 0;
    d.xAllCap = xAllCapWanted;
    if (sharded()) {
      if ((d.perShard & (d.perShard - 1)) != 0) {
        if (!unevenShards) throw std::invalid_argument("a node-sharded network needs a power-of-two number of nodes per shard");
        d.ownShift = -1;  // ownerOf divides
      } else {
        while ((1 << d.ownShift) < d.perShard) ++d.ownShift;
      }
    }
    const int NL = d.perShard;  // capacities are those of a full shard: every shard lays its exchange region out identically
    d.msgDiscardTime = msgDiscardTime;
    int ring = 2048;
    int need = hm.latMax + 64 + ringExtra;
    if (!farEnabled && need > 4096) {
      // latency models with multi-second arrivals (EthScan 12 000 ms, Fixed / Uniform(8000)): the ring stays at 4 096
      // buckets (the multisplit keeps a histogram of the ring in shared memory) and arrivals 2 048 ms or more ahead go
      // through the far-future calendar; the protocol still ticks every millisecond
      if (sharded()) throw std::logic_error("this latency model needs the far-future calendar for messages, which node-sharded networks do not have");
      farEnabled = true;
      farTicking = true;
      need = std::min(need, 2048 - 64 + ringExtra);
    }
    if (farEnabled) need *= 2;  // envelopes are "near" up to ring/2 ms ahead
    while (ring < need) ring <<= 1;
    if (tun.ring) {
      if (tun.ring < need || (tun.ring & (tun.ring - 1)) != 0) throw std::invalid_argument("tunable ring must be a power of two >= " + std::to_string(need));
      ring = (int)tun.ring;
    }
    d.ring = ring;
    ringMask = ring - 1;
    long long bcap = tun.bcap ? tun.bcap : std::max<long long>(16384, 3LL * NL);
    d.bcap = (int)bcap;
    d.itemCap = (int)(2 * bcap + 1024);
    d.descCap = (int)(tun.descCap ? tun.descCap : std::max<long long>(65536, 32LL * NL));
    d.descCap = (d.descCap + ARENA_STRIPES - 1) / ARENA_STRIPES * ARENA_STRIPES;
    d.destScratchCap = destScratchOverride ? destScratchOverride : d.descCap;
    // sharded: the new-envelope arrays are indexed by the creation index over all shards
    d.newEvCap = sharded() ? (int)std::min<long long>(0x7fffffffLL, (long long)shardWorld * (d.descCap + NL)) : d.descCap + N;
    d.recCap = (int)(tun.recCap ? tun.recCap : std::max<long long>(65536, 32LL * NL));
    d.recDestCap = recDestOverride ? recDestOverride : d.recCap * 4 + N + 1024;
    d.freeCap = d.descCap;
    d.latKind = hm.latKind;
    d.latParam = hm.latParam;

    d.ctl = dalloc<Ctl>(1);
    d.stats = dalloc<unsigned long long>((size_t)STAT_SLOTS * ST_COUNT);
    std::vector<int16_t> x(N), y(N), ex(N);
    std::vector<uint8_t> city(N), down(N), part(N, 0);
    for (int i = 0; i < N; ++i) {
      x[i] = (int16_t)hm.nodes[i].x;
      y[i] = (int16_t)hm.nodes[i].y;
      ex[i] = (int16_t)hm.nodes[i].extra;
      city[i] = (uint8_t)hm.nodes[i].city;
      down[i] = hm.nodes[i].down ? 1 : 0;
    }
    d.nx = dupload(x);  // node attributes are replicated on every shard (latency needs both ends)
    d.ny = dupload(y);
    d.nextra = dupload(ex);
    d.ncity = dupload(city);
    d.ndown = dupload(down);
    d.npart = dupload(part);
    d.msgReceived = dallocNodes<long long>();
    d.msgSent = dallocNodes<long long>();
    d.bytesSent = dallocNodes<long long>();
    d.bytesReceived = dallocNodes<long long>();
    d.doneAt = dallocNodes<long long>();
    d.latTab = dupload(hm.latTab);
    d.latBase = dupload(hm.latBase);
    d.latJit = dupload(hm.latJit);
    std::vector<unsigned long long> ja(48), jc(48);
    lcgJumpTables((uint64_t*)ja.data(), (uint64_t*)jc.data());
    d.jumpA = dupload(ja);
    d.jumpC = dupload(jc);
    d.buckets = dalloc<Ev>((size_t)ring * (size_t)d.bcap);
    d.bucketCount = dalloc<int>(ring);
    d.inboxCnt = dallocNodes<int>();
    d.inboxOff = dallocNodes<int>();
    d.inboxFill = dallocNodes<int>();
    d.nodeTasks = dallocNodes<int>();
    d.listStripeCap = ((NL + 31) / 32 + ARENA_STRIPES - 1) / ARENA_STRIPES * 32 + 32;
    d.dueList = dalloc<int>((size_t)ARENA_STRIPES * d.listStripeCap);
    d.taskList = dalloc<int>((size_t)ARENA_STRIPES * d.listStripeCap);
    d.taskWord = dalloc<unsigned long long>((size_t)ARENA_STRIPES * d.listStripeCap);
    d.inbox = dalloc<unsigned long long>((size_t)d.itemCap);
    d.subCount = dalloc<int>(d.bcap);
    d.itemBase = dalloc<int>(d.bcap);
    d.evSlots = dalloc<int>(d.itemCap);
    d.evDraws = dalloc<int>(d.itemCap);
    // GSF: two halves, by the parity of checkSigs' tick (condHalf); the next pass's checkSigs may run beside this
    // pass's emission, which reads the other half
    d.condStride = proto == PROTO_GSF ? d.nLoc : 0;
    d.condAhead = proto == PROTO_GSF && !sharded() ? condAhead : 0;
    d.condFired = dalloc<int>((size_t)d.nLoc + d.condStride) - d.n0;
    d.condDraws = dallocNodes<int>();
    d.condDue = dallocNodes<int>();
    d.workCap = (int)std::max<long long>(1 << 16, 64LL * NL) / ARENA_STRIPES * ARENA_STRIPES;
    d.workList = dalloc<uint32_t>(d.workCap);
    d.condEv = dalloc<Ev>((size_t)d.nLoc + d.condStride) - d.n0;
    d.condTarget = dalloc<int>((size_t)d.nLoc + d.condStride) - d.n0;
    d.slotBase = dalloc<int>((size_t)NL + d.itemCap);
    d.drawBase = dalloc<int>((size_t)NL + d.itemCap);
    d.scanPartial = dalloc<int>(2 * 8192);
    d.desc = dalloc<Desc>(d.descCap);
    d.destScratch = dalloc<uint32_t>(d.destScratchCap);
    d.msWarps = 8;
    while (d.msWarps > 1 && (size_t)d.msWarps * ring * sizeof(int) > 200 * 1024) d.msWarps >>= 1;  // shared-memory histograms
    d.msChunks = (d.newEvCap + d.msWarps * MS_SUB_ENVELOPES - 1) / (d.msWarps * MS_SUB_ENVELOPES);
    d.msCount = dalloc<int>((size_t)d.msChunks * (size_t)ring);
    d.freeList = dalloc<uint32_t>(d.freeCap);
    if (sharded()) {
      if (farEnabled && !shardFarOk) throw std::logic_error("this protocol cannot run node-sharded yet (far-future calendar)");
      d.xItemCap = d.itemCap + 1;
      d.stageCapWords = (int)std::min<long long>(0x7fffffffLL, stageWordsWanted);
      d.recCap = d.recCap / shardWorld * shardWorld;
      d.recDestCap = d.recDestCap / shardWorld * shardWorld;
      d.xRecCap = d.recCap / shardWorld;
      d.xRecDestCap = d.recDestCap / shardWorld;
      allocExchange();
      d.bucketKey = dalloc<unsigned long long>((size_t)ring * (size_t)d.bcap);
      d.itemKey = dalloc<unsigned long long>((size_t)d.itemCap);
      d.xoffS = dalloc<uint32_t>((size_t)d.itemCap);
      d.xoffD = dalloc<uint32_t>((size_t)d.itemCap);
    } else {
      d.newEv = dalloc<Ev>(d.newEvCap);
      d.newTarget = dalloc<int>(d.newEvCap);
      d.rec = dalloc<MultiRec>(d.recCap);
      d.recDest = dalloc<uint32_t>(d.recDestCap);
      d.recArrival = dalloc<int>(d.recDestCap);
    }
    if (farEnabled) {
      d.ffwd = farTicking ? 0 : 1;
      d.farCap = tun.farCap ? (int)tun.farCap : (farTicking ? (int)std::min<long long>(1LL << 26, std::max<long long>(64LL * N + 4096, farWanted))
                                                                  : (int)std::max<long long>(2LL * N + 1024, farWanted));
      d.far = dalloc<FarEv>(d.farCap);
      d.farSel = dalloc<int>(d.farCap);
    }
  }
  int recDestOverride = 0;  // sendAll protocols size the destination arena themselves
  int destScratchOverride = 0;
  bool forceShufSerial = false;  // tunable force_shuffle_serial (test hook)
  bool forcePickSerial = false;  // tunable force_pick_serial (test hook, Handel)
  int condAhead = 1;             // tunable cond_ahead (Dev::condAhead; 0 runs every pass's checkSigs in the pass)
  int ringExtra = 0;        // longest handler-chosen delay of a near envelope (e.g. blockConstructionTime)
  bool farEnabled = false;  // far-future calendar (+ fast-forward for protocols without conditional tasks)
  bool farTicking = false;  // calendar without fast-forward: the latency model, not the protocol, asked for it

  Ctl readCtl() {
    Ctl c;
    be->sync();
    be->download(&c, d.ctl, sizeof(Ctl));
    return c;
  }
  void writeCtl(const Ctl& c) { be->upload(d.ctl, &c, sizeof(Ctl)); }

  void checkLatencyBuilder() const {
    if (hm.latKind == LAT_CITY && hm.builder != HostModel::B_AWS)
      throw std::invalid_argument("AwsRegionNetworkLatency needs nodes built by an AWS_* node builder");  // NetworkLatency.java:146-148
    if (hm.latKind == LAT_CITY_MAT && hm.builder != HostModel::B_CITIES)
      throw std::logic_error("Can't use NetworkLatencyByCity model with default city location");  // NetworkLatency.java:178-181
  }

  // ---- PingPong.init()  (protocols/PingPong.java:82-87) ----
  void pingpongInit(int nodeCt) {
    requireNotInited();
    requireUnsharded("this protocol");
    if (nodeCt <= 0) throw std::invalid_argument("nodeCt");
    checkLatencyBuilder();
    hm.buildNodes(nodeCt);
    allocCommon(nodeCt, PROTO_PINGPONG);
    d.pong = dalloc<int>(nodeCt);
    // network.sendAll(new Ping(), node0): one draw, per-destination arrival, stable sort (Network.java:420-467)
    int32_t seed = hm.rd.nextInt();
    Dev hd = hostView();
    struct Arr {
      int arrival;
      uint32_t dest;
    };
    std::vector<Arr> da;
    for (int to = 0; to < nodeCt; ++to) {
      int nt = latency(hd, 0, to, pseudoRandom(to, seed));
      if (nt < msgDiscardTime) da.push_back({1 + nt, (uint32_t)to});
    }
    std::stable_sort(da.begin(), da.end(), [](const Arr& a, const Arr& b) { return a.arrival < b.arrival; });
    std::vector<long long> sent(nodeCt, 0);
    sent[0] = nodeCt;  // msgSent++ / bytesSent += 1 per destination (Network.java:476-477)
    be->upload(d.msgSent, sent.data(), sizeof(long long) * nodeCt);
    be->upload(d.bytesSent, sent.data(), sizeof(long long) * nodeCt);
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    c.callId = 1;
    if (!da.empty()) {
      if ((int)da.size() > d.recDestCap) throw std::runtime_error("record arena too small");
      Ev ev;
      std::memset(&ev, 0, sizeof(ev));
      ev.pad = 2;  // sendAll at time 0: sendTime 1 (+1)
      ev.from = 0;
      ev.meta = PP_PING;
      ev.to = da[0].dest;
      if (da.size() == 1) {
        ev.kind = EV_MSG;
      } else {
        ev.kind = EV_MULTI;
        ev.aux = 0;
        MultiRec rc;
        std::memset(&rc, 0, sizeof(rc));
        rc.pad = 2;
        rc.from = 0;
        rc.meta = PP_PING;
        rc.n = (uint32_t)da.size();
        rc.cur = 0;
        rc.off = 0;
        be->upload(d.rec, &rc, sizeof(rc));
        std::vector<uint32_t> dst(da.size());
        std::vector<int> arr(da.size());
        for (size_t i = 0; i < da.size(); ++i) {
          dst[i] = da[i].dest;
          arr[i] = da[i].arrival;
        }
        be->upload(d.recDest, dst.data(), dst.size() * 4);
        be->upload(d.recArrival, arr.data(), arr.size() * 4);
        c.recTop = 1;
        c.recDestTop = (int)da.size();
      }
      int tgt = da[0].arrival;
      if (tgt >= (farEnabled ? d.ring / 2 : d.ring)) throw std::runtime_error("latency exceeds the time ring");
      be->upload(d.buckets + (size_t)(tgt & ringMask) * d.bcap, &ev, sizeof(ev));
      int one = 1;
      be->upload(d.bucketCount + (tgt & ringMask), &one, sizeof(int));
    }
    c.rng = hm.rd.seed;
    writeCtl(c);
    inited = true;
  }

  // host-side view of node attributes for the few latency evaluations done at init
  std::vector<int16_t> hx_, hy_, hex_;
  std::vector<uint8_t> hcity_;
  Dev hostView() {
    int N = (int)hm.nodes.size();
    hx_.resize(N);
    hy_.resize(N);
    hex_.resize(N);
    hcity_.resize(N);
    for (int i = 0; i < N; ++i) {
      hx_[i] = (int16_t)hm.nodes[i].x;
      hy_[i] = (int16_t)hm.nodes[i].y;
      hex_[i] = (int16_t)hm.nodes[i].extra;
      hcity_[i] = (uint8_t)hm.nodes[i].city;
    }
    Dev h;
    std::memset(&h, 0, sizeof(h));
    h.N = N;
    h.nx = hx_.data();
    h.ny = hy_.data();
    h.nextra = hex_.data();
    h.ncity = hcity_.data();
    h.latKind = hm.latKind;
    h.latParam = hm.latParam;
    h.latTab = hm.latTab.data();
    h.latBase = hm.latBase.data();
    h.latJit = hm.latJit.data();
    return h;
  }

  // ---- GSFSignature.init()  (protocols/GSFSignature.java:611-635) ----
  GsfParams gp{};
  void gsfInit(const GsfParams& p) {
    requireNotInited();
    const int N = p.nodeCount;
    if (p.nodesDown >= N || p.nodesDown < 0 || p.threshold > N || (p.nodesDown + p.threshold > N))  // :69-74
      throw std::invalid_argument("nodeCount=" + std::to_string(N) + ", threshold=" + std::to_string(p.threshold));
    if (N < 2 || (N & (N - 1)) != 0) throw std::invalid_argument("the device engine needs a power-of-two nodeCount >= 2 for GSFSignature");
    if (p.acceleratedCallsCount > MAX_ACC || p.acceleratedCallsCount < 0) throw std::invalid_argument("acceleratedCallsCount must be in [0,16]");
    if (p.periodDurationMs <= 0 || p.pairingTime < 0) throw std::invalid_argument("period/pairing");
    checkLatencyBuilder();
    gp = p;
    hm.buildNodes(N);
    // dead nodes: nextInt(nodeCount) until nodesDown distinct ids != 1 are chosen (:617-625)
    for (int setDown = 0; setDown < p.nodesDown;) {
      int down = hm.rd.nextInt(N);
      if (!hm.nodes[down].down && down != 1) {
        hm.nodes[down].down = true;
        setDown++;
      }
    }
    int L = 1;
    while ((1 << L) <= N) ++L;  // levels 0..log2(N)   (:186)
    // envelopes in flight beyond the ring's horizon under a multi-second latency model: every node sends at most once per
    // level and period, and keeps it in flight for at most latMax
    farWanted = (long long)N * L * (hm.latMax / std::max(1, p.periodDurationMs) + 1) / 2 + 4096;
    if (sharded()) {
      // pooled payloads that cross shards are staged on the receiving shard (one area per sender and pass parity): in one
      // pass a shard receives from one sender at most about one level block per sending node (DESIGN.md §8)
      const long long nl = N / shardWorld;
      stageWordsWanted = std::max<long long>(65536, nl * std::max<long long>(1, nl / 64) * 5 / 4 + 8192);
      if (tun.stageWords) stageWordsWanted = tun.stageWords;
    }
    allocCommon(N, PROTO_GSF);
    const int NL = d.nLoc;
    d.L = L;
    d.W64 = std::max(1, N / 64);
    d.threshold = p.threshold;
    d.timeoutPerLevel = p.timeoutPerLevelMs;
    d.period = p.periodDurationMs;
    d.accel = p.acceleratedCallsCount;
    d.qcap = (int)(tun.qcap ? tun.qcap : std::min<long long>(4096, std::max<long long>(64, 2LL * N)));
    d.qcap = (d.qcap + 31) / 32 * 32;
    d.verified = dallocNodes<unsigned long long>(d.W64);
    d.indivSeen = dallocNodes<unsigned long long>(d.W64);
    d.indivVer = dallocNodes<unsigned long long>(d.W64);
    d.pos = dallocNodes<int>(L);
    d.remaining = dallocNodes<int>(L);
    d.cntVer = dallocNodes<int>(L);
    d.cntIndiv = dallocNodes<int>(L);
    d.cntUnion = dallocNodes<int>(L);
    d.totalCard = dallocNodes<int>();
    d.minStart = dallocNodes<int>();
    d.stamp = dallocNodes<uint32_t>();
    d.qLen = dallocNodes<int>();
    d.sigChecked = dallocNodes<int>();
    d.sigQueueSize = dallocNodes<int>();
    d.queue = dallocNodes<QEntry>(d.qcap);
    d.qScore = dallocNodes<int>(d.qcap);
    d.qStamp = dallocNodes<uint32_t>(d.qcap);
    d.lvVer = dallocNodes<uint32_t>(L);
    std::vector<int> pairing(N);
    for (int i = 0; i < N; ++i) pairing[i] = (int)std::max(1.0, p.pairingTime * hm.nodes[i].speed);  // :170
    d.pairing = duploadNodes(pairing);
    d.peerBits = (N / 2 <= 65536 && !tun.peerBits32) ? 16 : 32;  // 16-bit entries are block-relative; tunable peer_bits_32 forces the wide layout at small N (tests)
    {
      const size_t rowBytes = (size_t)(N - 1) * (size_t)(d.peerBits / 8);
      void* pp = be->alloc((size_t)NL * rowBytes);
      allocs.push_back(pp);
      d.peers = (char*)pp - (size_t)d.n0 * rowBytes;
    }
    // payload pools for levels whose block is wider than one word
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    long long perNode = tun.poolSlotsPerNode ? tun.poolSlotsPerNode : 24;
    // multi-second latency models keep a payload in flight for latMax / period cycles of its sender
    if (!tun.poolSlotsPerNode && farTicking) perNode = std::max<long long>(perNode, 2LL * hm.latMax / std::max(1, p.periodDurationMs) + 24);
    for (int l = INLINE_MAX_LEVEL + 1; l < L; ++l) {
      long long slots = std::max<long long>(1024, perNode * NL);
      slots = (slots + POOL_STRIPES - 1) / POOL_STRIPES * POOL_STRIPES;
      d.poolCap[l] = (int)slots;
      d.pool[l] = dalloc<unsigned long long>((size_t)slots * (size_t)poolWords(l));
      std::vector<uint32_t> fl((size_t)slots);
      long long per = slots / POOL_STRIPES;
      for (int sidx = 0; sidx < POOL_STRIPES; ++sidx) {
        for (long long i = 0; i < per; ++i) fl[(size_t)(sidx * per + i)] = (uint32_t)(sidx * per + (per - 1 - i));
        c.poolFreeCnt[l][sidx] = (int)per;
      }
      d.poolFree[l] = dupload(fl);
      c.poolMinFree[l] = (int)slots;
    }
    c.callId = 1;
    writeCtl(c);
    be->gsfInitNodes(d);

    // peer lists: Collections.shuffle of every level of every live node on the network RNG (:462-476)
    liveRank.assign(N, -1);
    int live = 0;
    for (int i = 0; i < N; ++i)
      if (!hm.nodes[i].down) liveRank[i] = live++;
    const unsigned long long D = (unsigned long long)(N - L);  // draws per node without rejections
    unsigned long long s0 = hm.rd.seed;
    std::vector<unsigned long long> rejOrd;
    if (N > 2) {
      std::vector<unsigned long long> cand;
      unsigned long long nominal = (unsigned long long)live * D;
      be->rngCandidates(d, s0, nominal + nominal / 16384 + 4096, N / 2, cand);
      std::sort(cand.begin(), cand.end());
      // serial fix-up: which candidates are real rejections, and how far they shift the stream
      unsigned long long shift = 0;
      for (unsigned long long pos : cand) {
        unsigned long long o = pos - shift;
        if (o >= nominal) break;
        unsigned long long rem = o % D;
        int l = 1;
        while (true) {  // level whose draw range contains rem: cum(l) = 2^(l-1) - l
          unsigned long long nxt = (1ULL << l) - (unsigned long long)(l + 1);
          if (rem < nxt) break;
          ++l;
        }
        unsigned long long cum = (1ULL << (l - 1)) - (unsigned long long)l;
        int bound = (1 << (l - 1)) - (int)(rem - cum);
        if ((bound & (bound - 1)) == 0) continue;
        uint64_t st = lcgAdvance((const u64*)hostJumpA(), (const u64*)hostJumpC(), s0, pos + 1);
        int32_t u = (int32_t)(uint32_t)(st >> 17);  // next(31)
        int32_t r = u % bound;
        if ((int32_t)((uint32_t)u - (uint32_t)r + (uint32_t)(bound - 1)) < 0) {
          rejOrd.push_back(o);
          ++shift;
        }
      }
      unsigned long long total = nominal + shift;
      hm.rd.seed = lcgAdvance((const u64*)hostJumpA(), (const u64*)hostJumpC(), s0, total);
      initDraws = total;
    }
    int* dRank = dupload(liveRank);
    unsigned long long* dRej = dupload(rejOrd);
    be->gsfShufflePeers(d, s0, dRank, dRej, (int)rejOrd.size());

    // registerPeriodicTask(doCycle, 1, period) for live nodes in id order (:630) -> bucket of ms 1
    std::vector<Ev> per;
    std::vector<unsigned long long> keys;
    for (int i = d.n0; i < d.n0 + d.nLoc; ++i)
      if (!hm.nodes[i].down) {
        Ev ev;
        std::memset(&ev, 0, sizeof(ev));
        ev.pad = 1;  // registered at time 0 (Envelope.sendTime + 1)
        ev.kind = EV_PERIODIC;
        ev.to = (uint32_t)i;
        ev.from = (uint32_t)i;
        per.push_back(ev);
        keys.push_back(orderKey(0, (unsigned)i));
      }
    if ((int)per.size() > d.bcap) throw std::runtime_error("bucket capacity too small");
    be->upload(d.buckets + (size_t)1 * d.bcap, per.data(), per.size() * sizeof(Ev));
    if (sharded() && !keys.empty()) be->upload(d.bucketKey + (size_t)1 * d.bcap, keys.data(), keys.size() * sizeof(unsigned long long));
    int cnt = (int)per.size();
    be->upload(d.bucketCount + 1, &cnt, sizeof(int));
    c = readCtl();
    c.rng = hm.rd.seed;
    writeCtl(c);
    inited = true;
  }
  uint64_t hja_[48], hjc_[48];
  bool hjInit_ = false;
  const uint64_t* hostJumpA() {
    if (!hjInit_) {
      lcgJumpTables(hja_, hjc_);
      hjInit_ = true;
    }
    return hja_;
  }
  const uint64_t* hostJumpC() {
    hostJumpA();
    return hjc_;
  }

  // ---- SanFerminSignature: constructor builds the nodes (:112-129), init() registers goNextLevel at t=1 (:136-138) ----
  SfParams sp{};
  bool sfConstructed = false;
  void sanferminConstruct(const SfParams& p) {
    requireNotInited();
    if (sfConstructed) throw std::logic_error("already constructed");
    const int N = p.nodeCount;
    if (N < 2 || (N & (N - 1)) != 0) throw std::invalid_argument("the device engine needs a power-of-two nodeCount >= 2 for SanFerminSignature");
    if (p.candidateCount < 1 || p.candidateCount + 1 > SHUFFLE_MAX) throw std::invalid_argument("candidateCount must be in [1, 63]");
    if (p.pairingTime <= 0 || p.replyTimeout <= 0) throw std::invalid_argument("pairingTime / replyTimeout must be positive");
    checkLatencyBuilder();
    sp = p;
    hm.buildNodes(N);  // new SanFerminNode(nb) draws from network.rd here, before any later rd.setSeed()
    sfConstructed = true;
  }
  void sanferminInit() {
    requireNotInited();
    requireUnsharded("this protocol");
    if (!sfConstructed) throw std::logic_error("SanFerminSignature not constructed");
    const int N = sp.nodeCount;
    {
      int P0 = 0;
      while ((1 << (P0 + 1)) <= N) ++P0;
      const long long perSend = sp.candidateCount + 1;
      destScratchOverride = (int)std::min<long long>(0x7fffffffLL, (2 * perSend * N + 4096 + ARENA_STRIPES - 1) / ARENA_STRIPES * ARENA_STRIPES);
      if (!tun.recCap) tun.recCap = std::max<long long>(65536, 4LL * N * (P0 + 1));
      recDestOverride = (int)std::min<long long>(0x7fffffffLL, (long long)tun.recCap * perSend / 2 + N + 1024);
    }
    allocCommon(N, PROTO_SANFERMIN);
    int P = 0;
    while ((1 << (P + 1)) <= N) ++P;
    d.sfP = P;
    d.sfThreshold = sp.threshold;
    d.sfPairing = sp.pairingTime;
    d.sfSigSize = sp.signatureSize;
    d.sfReplyTimeout = sp.replyTimeout;
    d.sfCandCount = sp.candidateCount;
    std::vector<int> cpl(N, P), agg(N, 1);
    d.sfCpl = dupload(cpl);
    d.sfAgg = dupload(agg);
    d.sfFlags = dalloc<int>(N);
    d.sfThresholdAt = dalloc<long long>(N);
    d.sfSentReq = dalloc<int>(N);
    d.sfRecvReq = dalloc<int>(N);
    d.sfCacheMask = dalloc<uint32_t>(N);
    d.sfCache = dalloc<int>((size_t)N * 32);
    d.sfUsedWords = std::max(1, N / 128);
    d.sfUsedBits = dalloc<unsigned long long>((size_t)N * d.sfUsedWords);
    d.sfPendBits = dalloc<unsigned long long>((size_t)N * d.sfUsedWords);
    d.shufCap = d.newEvCap;
    d.forceShufSerial = forceShufSerial ? 1 : 0;
    d.byG = dalloc<int>(d.newEvCap);
    {
      std::vector<int> m1((size_t)d.newEvCap, -1);
      d.byGTick = dupload(m1);
    }
    d.descDraw = dalloc<int>(d.descCap);
    std::vector<Ev> tasks((size_t)N);
    for (int i = 0; i < N; ++i) {
      Ev ev;
      std::memset(&ev, 0, sizeof(ev));
      ev.pad = 1;  // registered at time 0 (Envelope.sendTime + 1)
      ev.kind = EV_TASK;
      ev.to = (uint32_t)i;
      ev.from = (uint32_t)i;
      ev.meta = SF_T_GO;
      tasks[(size_t)i] = ev;
    }
    if (N > d.bcap) throw std::runtime_error("bucket capacity too small");
    be->upload(d.buckets + (size_t)1 * d.bcap, tasks.data(), tasks.size() * sizeof(Ev));
    be->upload(d.bucketCount + 1, &N, sizeof(int));
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    c.callId = 1;
    c.rng = hm.rd.seed;
    writeCtl(c);
    inited = true;
  }

  // ---- Handel.init()  (protocols/Handel.java:957-1014).  Everything init() draws from network.rd is sequential
  //      (bad nodes, start times, node attributes, N cumulative shuffles for the reception ranks, tie shuffles of
  //      the emission lists), so it runs on the host like in the reference; the tables are then uploaded.  Node-sharded:
  //      every shard runs the whole init (so `rd` ends in the same state everywhere) and keeps its own nodes' state. ----
  HandelParams hp{};
  void handelInit(const HandelParams& p) {
    requireNotInited();
    const int N = p.nodeCount;
    if (p.nodesDown >= N || p.nodesDown < 0 || p.threshold > N || (p.nodesDown + p.threshold > N))  // :112-117
      throw std::invalid_argument("nodeCount=" + std::to_string(N) + ", threshold=" + std::to_string(p.threshold));
    if (N < 2 || (N & (N - 1)) != 0) throw std::invalid_argument("We support only power of two nodes in this simulation");  // :118-120
    if (p.byzantineSuicide && p.hiddenByzantine) throw std::invalid_argument("Only one attack at a time");  // :122-124
    if (p.fastPath < 0 || p.fastPath > MAX_ACC) throw std::invalid_argument("fastPath must be in [0,16]");
    if (p.disseminationPeriodMs <= 0 || p.pairingTime < 0 || p.desynchronizedStart < 0) throw std::invalid_argument("period/pairing/desynchronizedStart");
    checkLatencyBuilder();
    hp = p;
    // Network.chooseBadNodes first (:960-963)
    std::vector<char> bad((size_t)N, 0);
    for (int setDown = 0; setDown < p.nodesDown;) {
      int down = hm.rd.nextInt(N);
      if (down != 1 && !bad[(size_t)down]) {
        bad[(size_t)down] = 1;
        setDown++;
      }
    }
    std::vector<int> startAt((size_t)N, 0);
    for (int i = 0; i < N; ++i) {  // :965-974
      startAt[(size_t)i] = p.desynchronizedStart == 0 ? 0 : hm.rd.nextInt(p.desynchronizedStart);
      hm.buildNodes(1);
      if (bad[(size_t)i]) hm.nodes[(size_t)i].down = true;
    }
    int L = 1;
    while ((1 << L) <= N) ++L;
    if (sharded()) {
      // pooled payloads that cross shards are staged on the receiving shard (one area per sender and pass parity).  A node
      // disseminates at most once per pass, one message per level, and only the levels whose sibling block spans whole
      // shards cross: at most one block of each of those levels per sending node (DESIGN.md §8)
      const long long nl = N / shardWorld;
      long long words = 0;
      for (int l = INLINE_MAX_LEVEL + 1; l < L; ++l)
        if ((1LL << (l - 1)) >= nl) words += (1LL << (l - 1)) / 64;
      stageWordsWanted = std::max<long long>(65536, nl * words + 8192);
      if (tun.stageWords) stageWordsWanted = tun.stageWords;
      xProtoBytes = hPickBytes(shardWorld, (int)nl);  // the pick exchange: one byte per pick, at most one per node and pass
    }
    allocCommon(N, PROTO_HANDEL);
    for (int i = 0; i < N; ++i)
      if (startAt[(size_t)i] + 1 >= d.ring) throw std::invalid_argument("desynchronizedStart exceeds the time ring");
    const int NL = d.nLoc, n0 = d.n0;
    d.L = L;
    d.W64 = std::max(1, N / 64);
    d.threshold = p.threshold;
    d.period = p.disseminationPeriodMs;
    d.hLevelWait = p.levelWaitTime;
    d.hFastPath = p.fastPath;
    d.hExtraCycle = p.extraCycle;
    d.hByzSuicide = p.byzantineSuicide;
    d.hWinInit = 16;  // WindowParameters() :157-159
    d.hWinMin = 1;
    d.hWinMax = 128;
    d.qcap = (int)(tun.qcap ? tun.qcap : std::min<long long>(4096, std::max<long long>(64, 2LL * N)));
    d.qcap = (d.qcap + 31) / 32 * 32;
    const size_t W = (size_t)d.W64;
    // level 0: own signature in lastAggVerified / verifiedIndSignatures / totalIncoming (:409-417); initLevel() runs for every node
    {
      std::vector<unsigned long long> diag((size_t)NL * W, 0);
      for (int i = n0; i < n0 + NL; ++i) diag[(size_t)(i - n0) * W + (size_t)(i >> 6)] = 1ULL << (i & 63);
      for (unsigned long long** row : {&d.hLastAgg, &d.hTotInc, &d.hVerInd}) {
        *row = dallocNodes<unsigned long long>(W);
        be->upload(*row + (size_t)n0 * W, diag.data(), diag.size() * sizeof(unsigned long long));
      }
    }
    d.hToVerInd = dallocNodes<unsigned long long>(W);
    d.hFinPeers = dallocNodes<unsigned long long>(W);
    d.hBlack = dallocNodes<unsigned long long>(W);
    std::vector<int> zerosNL((size_t)N * L, 0), outFin((size_t)N * L, 0), biz((size_t)N * L, p.byzantineSuicide ? 0 : -1), cnt0((size_t)N * L, 0);
    std::vector<uint32_t> ver((size_t)N * L, 1);
    for (int i = 0; i < N; ++i) {
      outFin[(size_t)i * L] = 1;  // level 0: outgoingFinished = true
      cnt0[(size_t)i * L] = 1;
    }
    d.hPos = duploadNodes(zerosNL, L);
    d.hOutFin = duploadNodes(outFin, L);
    d.hBiz = duploadNodes(biz, L);
    {
      std::vector<int> nohit((size_t)N * L, -2147483647 - 1);
      d.hBizNoHit = duploadNodes(nohit, L);
    }
    d.hCntLast = duploadNodes(cnt0, L);
    d.hCntInc = duploadNodes(cnt0, L);
    d.hCntInd = duploadNodes(cnt0, L);
    d.lvVer = duploadNodes(ver, L);
    std::vector<int> ones((size_t)N, 1), win((size_t)N, d.hWinInit), added((size_t)N, p.extraCycle), pairing((size_t)N), minStart((size_t)N);
    for (int i = 0; i < N; ++i) {
      pairing[(size_t)i] = (int)std::max(1.0, p.pairingTime * hm.nodes[(size_t)i].speed);  // :282
      minStart[(size_t)i] = startAt[(size_t)i] + 1;                                        // :981-982
    }
    d.hTotal = duploadNodes(ones);
    d.hWindow = duploadNodes(win);
    d.hAddedCycle = duploadNodes(added);
    d.pairing = duploadNodes(pairing);
    d.minStart = duploadNodes(minStart);
    d.stamp = dallocNodes<uint32_t>();
    d.hStartAt = duploadNodes(startAt);
    d.hSigsChecked = dallocNodes<int>();
    d.hSigQueueSize = dallocNodes<int>();
    d.hMsgFiltered = dallocNodes<int>();
    d.hSeq = dallocNodes<int>();
    d.qLen = dallocNodes<int>();
    d.hQueue = dallocNodes<HQEntry>((size_t)d.qcap);
    d.qStamp = dallocNodes<uint32_t>((size_t)d.qcap);
    d.hCand = dallocNodes<int>(32);
    d.hCandK = dallocNodes<int>();
    d.hDrawBase = dallocNodes<int>();
    d.drawScanPartial = dalloc<int>(2 * 8192);
    d.hHidden = p.hiddenByzantine ? 1 : 0;
    d.forcePickSerial = forcePickSerial ? 1 : 0;
    d.hbNoPeers = dallocNodes<int>();
    {
      std::vector<int> m1((size_t)N, -1);
      d.hbLastId = duploadNodes(m1);
    }
    d.hbLastFrom = dallocNodes<int>();
    const bool timing_ = std::getenv("WTG_INIT_TIMING") != nullptr;
    auto t0_ = std::chrono::steady_clock::now();
    auto lap_ = [&](const char* what) {
      if (!timing_) return;
      auto t1 = std::chrono::steady_clock::now();
      std::fprintf(stderr, "[handel init] %s: %.2f s\n", what, std::chrono::duration<double>(t1 - t0_).count());
      t0_ = t1;
    };
    lap_("nodes + rows");
    unsigned hw = std::thread::hardware_concurrency();
    int T = (int)std::max(1u, std::min(hw ? hw : 1u, 64u));
    if (N < 2048) T = 1;
    auto parallelFor = [&](int n, const std::function<void(int, int)>& body) {  // body(begin, end), contiguous chunks
      if (T == 1) {
        body(0, n);
        return;
      }
      std::vector<std::thread> th;
      int per = (n + T - 1) / T;
      for (int t = 0; t < T; ++t) {
        int b0 = t * per, b1 = std::min(n, b0 + per);
        if (b0 < b1) th.emplace_back(body, b0, b1);
      }
      for (auto& x : th) x.join();
    };
    // setReceivingRanks (:940-948): N cumulative shuffles of one list.  Every shard draws all of them and keeps its own rows
    // plus the transposed table (the emission list of sender s reads column s, and every sender's tie shuffles draw from rd).
    // Host peak: the transposed table (N^2) + the own rows (nLoc x N) + the own senders' lists (nLoc x (N-1)).
    std::vector<int> ranksOwn((size_t)NL * N);
    std::unique_ptr<int[]> ranksT_(new int[(size_t)N * N]);  // first touched by the transposing threads
    int* const ranksT = ranksT_.get();
    {
      std::vector<int> expected((size_t)N);
      for (int i = 0; i < N; ++i) expected[(size_t)i] = i;
      const int RB = std::min(N, 1024);  // rows drawn before they are transposed
      std::vector<int> blk((size_t)RB * N);
      for (int r0 = 0; r0 < N; r0 += RB) {
        const int r1 = std::min(N, r0 + RB);
        for (int n = r0; n < r1; ++n) {
          for (int i = N; i > 1; --i) std::swap(expected[(size_t)i - 1], expected[(size_t)hm.rd.nextInt(i)]);
          int* row = blk.data() + (size_t)(n - r0) * N;
          for (int i = 0; i < N; ++i) row[expected[(size_t)i]] = i;
        }
        for (int n = std::max(r0, n0); n < std::min(r1, n0 + NL); ++n)
          std::memcpy(ranksOwn.data() + (size_t)(n - n0) * N, blk.data() + (size_t)(n - r0) * N, sizeof(int) * (size_t)N);
        parallelFor(N, [&](int c0, int c1) {  // contiguous writes: rows [r0, r1) of columns [c0, c1)
          for (int c = c0; c < c1; ++c) {
            int* dst = ranksT + (size_t)c * N + r0;
            for (int r = r0; r < r1; ++r) dst[r - r0] = blk[(size_t)(r - r0) * N + c];
          }
        });
      }
    }
    lap_("reception ranks");
    // emission lists (:991-1013): receivers of each level sorted by the rank they gave the sender, ties shuffled.  The order of
    // every list is a pure function of the rank table; only the shuffles of equal-rank runs draw from the network RNG, and they
    // must do so in (sender, level, position) order.  Senders go in chunks: their lists are sorted on all host threads (the
    // lists of the shard's own senders are kept, of the others only the equal-rank runs), then one sequential pass shuffles the
    // ties of the chunk.
    std::vector<uint32_t> peersOwn((size_t)NL * (size_t)(N - 1), 0);
    {
      struct Run {
        uint32_t off, len;  // position in the sender's list (all levels), length >= 2
      };
      const int CH = std::min(N, 16 * T);
      std::vector<std::vector<Run>> runs((size_t)CH);
      auto ownList = [&](int sIdx) { return sIdx >= n0 && sIdx < n0 + NL ? peersOwn.data() + (size_t)(sIdx - n0) * (size_t)(N - 1) : nullptr; };
      auto sortSender = [&](int sIdx, std::vector<unsigned long long>& keys, std::vector<Run>& rs) {
        rs.clear();
        if (hm.nodes[(size_t)sIdx].down) return;
        const int* col = ranksT + (size_t)sIdx * N;
        uint32_t* list = ownList(sIdx);
        for (int l = 1; l < L; ++l) {
          Blk wb = levelBlock(sIdx ^ (1 << (l - 1)), l);
          keys.resize((size_t)wb.size);
          for (int i = 0; i < wb.size; ++i)  // unique keys: (rank, receiver) — ascending receiver inside a tie == stable order
            keys[(size_t)i] = ((unsigned long long)(uint32_t)col[wb.base + i] << 32) | (unsigned long long)(uint32_t)(wb.base + i);
          std::sort(keys.begin(), keys.end());
          const uint32_t lo = (1u << (l - 1)) - 1u;
          if (list)
            for (int i = 0; i < wb.size; ++i) list[lo + (uint32_t)i] = (uint32_t)(keys[(size_t)i] & 0xFFFFFFFFULL);
          for (int i = 0; i < wb.size;) {
            int j = i + 1;
            while (j < wb.size && (keys[(size_t)j] >> 32) == (keys[(size_t)i] >> 32)) ++j;
            if (j - i > 1) rs.push_back(Run{lo + (uint32_t)i, (uint32_t)(j - i)});
            i = j;
          }
        }
      };
      for (int c0 = 0; c0 < N; c0 += CH) {
        const int c1 = std::min(N, c0 + CH);
        parallelFor(c1 - c0, [&](int a, int b) {
          std::vector<unsigned long long> keys;
          for (int i = a; i < b; ++i) sortSender(c0 + i, keys, runs[(size_t)i]);
        });
        for (int sIdx = c0; sIdx < c1; ++sIdx) {  // Collections.shuffle of every run of equal ranks, in the reference's order
          uint32_t* list = ownList(sIdx);
          for (const Run& r : runs[(size_t)(sIdx - c0)])
            for (int m = (int)r.len; m > 1; --m) {
              const int j = hm.rd.nextInt(m);
              if (list) std::swap(list[r.off + (uint32_t)m - 1], list[r.off + (uint32_t)j]);
            }
        }
      }
    }
    lap_("emission lists");
    ranksT_.reset();
    {
      int* pr = dalloc<int>((size_t)NL * N);
      be->upload(pr, ranksOwn.data(), ranksOwn.size() * sizeof(int));
      d.hRanks = pr - (size_t)n0 * N;
      uint32_t* pp = dalloc<uint32_t>((size_t)NL * (size_t)(N - 1));
      be->upload(pp, peersOwn.data(), peersOwn.size() * sizeof(uint32_t));
      d.peers = pp - (size_t)n0 * (size_t)(N - 1);
    }
    d.peerBits = 32;
    lap_("upload");
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    long long perNode = tun.poolSlotsPerNode ? tun.poolSlotsPerNode : 24;
    for (int l = INLINE_MAX_LEVEL + 1; l < L; ++l) {
      long long slots = std::max<long long>(1024, perNode * NL);
      slots = (slots + POOL_STRIPES - 1) / POOL_STRIPES * POOL_STRIPES;
      d.poolCap[l] = (int)slots;
      d.pool[l] = dalloc<unsigned long long>((size_t)slots * (size_t)poolWords(l));
      d.poolRef[l] = dalloc<int>((size_t)slots);
      std::vector<uint32_t> fl((size_t)slots);
      long long per = slots / POOL_STRIPES;
      for (int sidx = 0; sidx < POOL_STRIPES; ++sidx) {
        for (long long i = 0; i < per; ++i) fl[(size_t)(sidx * per + i)] = (uint32_t)(sidx * per + (per - 1 - i));
        c.poolFreeCnt[l][sidx] = (int)per;
      }
      d.poolFree[l] = dupload(fl);
      c.poolMinFree[l] = (int)slots;
    }
    // periodic dissemination at startAt + 1 for live nodes, in id order (:978-983); a shard registers its own nodes' tasks,
    // with the ordering key of "pass 0" (wtg_shard.cuh)
    std::vector<std::vector<Ev>> per((size_t)d.ring);
    std::vector<std::vector<unsigned long long>> perKey((size_t)d.ring);
    for (int i = n0; i < n0 + NL; ++i)
      if (!hm.nodes[(size_t)i].down) {
        Ev ev;
        std::memset(&ev, 0, sizeof(ev));
        ev.pad = 1;  // registered at time 0 (Envelope.sendTime + 1)
        ev.kind = EV_PERIODIC;
        ev.to = (uint32_t)i;
        ev.from = (uint32_t)i;
        per[(size_t)(startAt[(size_t)i] + 1)].push_back(ev);
        perKey[(size_t)(startAt[(size_t)i] + 1)].push_back(orderKey(0, (unsigned)i));
      }
    for (int t = 0; t < d.ring; ++t)
      if (!per[(size_t)t].empty()) {
        if ((int)per[(size_t)t].size() > d.bcap) throw std::runtime_error("bucket capacity too small");
        be->upload(d.buckets + (size_t)t * d.bcap, per[(size_t)t].data(), per[(size_t)t].size() * sizeof(Ev));
        if (sharded()) be->upload(d.bucketKey + (size_t)t * d.bcap, perKey[(size_t)t].data(), perKey[(size_t)t].size() * sizeof(unsigned long long));
        int cnt = (int)per[(size_t)t].size();
        be->upload(d.bucketCount + t, &cnt, sizeof(int));
      }
    c.callId = 1;
    c.rng = hm.rd.seed;
    writeCtl(c);
    inited = true;
  }

  // ---- SanFerminCappos.init()  (protocols/SanFerminCappos.java:120-134): nodes, helpers, goNextLevel at t = 1 ----
  CapposParams qp{};
  void capposInit(const CapposParams& p) {
    requireNotInited();
    requireUnsharded("this protocol");
    const int N = p.nodeCount;
    if (N < 2 || (N & (N - 1)) != 0) throw std::invalid_argument("the device engine needs a power-of-two nodeCount >= 2 for SanFerminCappos");
    if (p.candidateCount < 1 || p.candidateCount + 1 > SHUFFLE_MAX) throw std::invalid_argument("candidateCount must be in [1, 63]");
    if (p.pairingTime <= 0 || p.timeout <= 0) throw std::invalid_argument("pairingTime / timeout must be positive");
    checkLatencyBuilder();
    qp = p;
    hm.buildNodes(N);
    int P = 0;
    while ((1 << (P + 1)) <= N) ++P;
    const long long perSend = p.candidateCount + 1;
    destScratchOverride = (int)std::min<long long>(0x7fffffffLL, (2 * perSend * N + 4096 + ARENA_STRIPES - 1) / ARENA_STRIPES * ARENA_STRIPES);
    if (!tun.recCap) tun.recCap = std::max<long long>(65536, 4LL * N * (P + 1));
    recDestOverride = (int)std::min<long long>(0x7fffffffLL, (long long)tun.recCap * perSend / 2 + N + 1024);
    allocCommon(N, PROTO_CAPPOS);
    d.sfP = P;
    d.sfThreshold = p.threshold;
    d.sfPairing = p.pairingTime;
    d.sfSigSize = p.signatureSize;
    d.sfTimeout = p.timeout;
    d.sfCandCount = p.candidateCount;
    std::vector<int> cpl(N, P);
    d.sfCpl = dupload(cpl);
    d.sfFlags = dalloc<int>(N);
    d.sfThresholdAt = dalloc<long long>(N);
    d.sfCacheMask = dalloc<uint32_t>(N);
    d.sfCache = dalloc<int>((size_t)N * 32);
    d.sfUsedWords = std::max(1, N / 128);
    d.sfUsedBits = dalloc<unsigned long long>((size_t)N * d.sfUsedWords);
    d.shufCap = d.newEvCap;
    d.forceShufSerial = forceShufSerial ? 1 : 0;
    d.byG = dalloc<int>(d.newEvCap);
    {
      std::vector<int> m1((size_t)d.newEvCap, -1);
      d.byGTick = dupload(m1);
    }
    d.descDraw = dalloc<int>(d.descCap);
    std::vector<Ev> tasks((size_t)N);
    for (int i = 0; i < N; ++i) {
      Ev ev;
      std::memset(&ev, 0, sizeof(ev));
      ev.pad = 1;  // registered at time 0 (Envelope.sendTime + 1)
      ev.kind = EV_TASK;
      ev.to = (uint32_t)i;
      ev.from = (uint32_t)i;
      ev.meta = CP_T_GO;
      tasks[(size_t)i] = ev;
    }
    if (N > d.bcap) throw std::runtime_error("bucket capacity too small");
    be->upload(d.buckets + (size_t)1 * d.bcap, tasks.data(), tasks.size() * sizeof(Ev));
    be->upload(d.bucketCount + 1, &N, sizeof(int));
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    c.callId = 1;
    c.rng = hm.rd.seed;
    writeCtl(c);
    inited = true;
  }

  // ---- Slush.init() / Snowflake.init()  (protocols/Slush.java:63-74, Snowflake.java:77-88): NODES_AV nodes on network.rd,
  //      then node 0 takes colour 1 and node 1 colour 2, each calling sendQuery(1) — on the host, with the draws the emit
  //      step would make (javaSampleAt, then the send's seed).  B < 0: Slush.  Ticks every millisecond like PingPong. ----
  void slushInit(int N, int M, int K, double A, int B) {
    requireNotInited();
    requireUnsharded("this protocol");  // the samples are drawn in the emit step, in creation order over all nodes
    if (N < 2) throw std::invalid_argument("NODES_AV must be at least 2");
    if (K < 1 || K > N - 1 || K > SHUFFLE_MAX - 1)
      throw std::invalid_argument("K must be in [1, min(63, NODES_AV - 1)]: with K >= NODES_AV randomRemotes never returns, with K = 0 "
                                  "no query is sent");
    checkLatencyBuilder();
    hm.buildNodes(N);
    const long long recs = tun.recCap ? tun.recCap : std::max<long long>(65536, 32LL * N);
    recDestOverride = (int)std::min<long long>(0x7fffffffLL, recs * K + N + 1024);  // a record holds K destinations
    allocCommon(N, B < 0 ? PROTO_SLUSH : PROTO_SNOWFLAKE);
    d.sampleK = K;
    d.sampleM = M;
    d.sampleB = B;
    d.sampleAK = (double)K * A;  // Slush: K * A, Snowflake: A * K (the same double)
    std::vector<uint8_t> color((size_t)N, 0);
    std::vector<int> nonce((size_t)N, 0);
    std::vector<uint8_t> pend((size_t)N, 0);
    d.avRound = dalloc<int>(N);
    d.avFound = dalloc<uint8_t>((size_t)N * 2);
    d.shufCap = d.newEvCap;
    d.forceShufSerial = forceShufSerial ? 1 : 0;
    d.byG = dalloc<int>(d.newEvCap);
    {
      std::vector<int> m1((size_t)d.newEvCap, -1);
      d.byGTick = dupload(m1);
    }
    d.descDraw = dalloc<int>(d.descCap);
    // the two initial queries: sendQuery(1) of node 0 (colour 1), then of node 1 (colour 2), both sent at time 0
    Dev hd = hostView();
    std::vector<long long> sent((size_t)N, 0);
    std::vector<MultiRec> recs0;
    std::vector<uint32_t> recDst;
    std::vector<int> recArr;
    std::vector<std::vector<Ev>> near((size_t)d.ring);
    for (int n = 0; n < 2; ++n) {
      color[(size_t)n] = (uint8_t)(n + 1);
      nonce[(size_t)n] = 1;
      pend[(size_t)n] = 1;
      std::vector<uint32_t> list((size_t)K);
      int used = javaSampleAt((const u64*)hostJumpA(), (const u64*)hostJumpC(), hm.rd.seed, 0, n, N, K, list.data());
      hm.rd.seed = lcgAdvance((const u64*)hostJumpA(), (const u64*)hostJumpC(), hm.rd.seed, (u64)used);
      int32_t seed = hm.rd.nextInt();
      sent[(size_t)n] = K;  // msgSent++ / bytesSent += 1 per destination (Network.java:476-477)
      struct Arr {
        int arrival;
        uint32_t dest;
      };
      std::vector<Arr> da;
      for (uint32_t to : list) {
        int nt = latency(hd, n, (int)to, pseudoRandom((int)to, seed));
        if (nt < msgDiscardTime) da.push_back({1 + nt, to});
      }
      std::stable_sort(da.begin(), da.end(), [](const Arr& a, const Arr& b) { return a.arrival < b.arrival; });
      if (da.empty()) continue;
      Ev ev;
      std::memset(&ev, 0, sizeof(ev));
      ev.pad = 2;  // sent at time 0: sendTime 1 (+1)
      ev.from = (uint32_t)n;
      ev.meta = AV_QUERY;
      ev.pl = avPl(1, n + 1);
      ev.to = da[0].dest;
      ev.kind = EV_MSG;
      if (da.size() > 1) {
        MultiRec rc;
        std::memset(&rc, 0, sizeof(rc));
        rc.pad = 2;
        rc.from = (uint32_t)n;
        rc.meta = AV_QUERY;
        rc.pl = ev.pl;
        rc.n = (uint32_t)da.size();
        rc.off = (uint32_t)recDst.size();
        ev.kind = EV_MULTI;
        ev.aux = (uint32_t)recs0.size();
        recs0.push_back(rc);
        for (const Arr& a : da) {
          recDst.push_back(a.dest);
          recArr.push_back(a.arrival);
        }
      }
      const int tgt = da[0].arrival;
      if (da.back().arrival >= d.ring) throw std::runtime_error("latency exceeds the time ring");
      near[(size_t)tgt].push_back(ev);
    }
    for (int t = 0; t < d.ring; ++t)
      if (!near[(size_t)t].empty()) {
        int c = (int)near[(size_t)t].size();
        be->upload(d.buckets + (size_t)t * d.bcap, near[(size_t)t].data(), (size_t)c * sizeof(Ev));
        be->upload(d.bucketCount + t, &c, sizeof(int));
      }
    if (!recs0.empty()) {
      be->upload(d.rec, recs0.data(), recs0.size() * sizeof(MultiRec));
      be->upload(d.recDest, recDst.data(), recDst.size() * sizeof(uint32_t));
      be->upload(d.recArrival, recArr.data(), recArr.size() * sizeof(int));
    }
    be->upload(d.msgSent, sent.data(), sent.size() * sizeof(long long));
    be->upload(d.bytesSent, sent.data(), sent.size() * sizeof(long long));
    d.avColor = dupload(color);
    d.avNonce = dupload(nonce);
    d.avPend = dupload(pend);
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    c.callId = 1;
    c.recTop = (int)recs0.size();
    c.recDestTop = (int)recDst.size();
    c.rng = hm.rd.seed;
    writeCtl(c);
    inited = true;
  }

  // ---- P2PFlood.init()  (protocols/P2PFlood.java:146-165): nodeCount nodes on network.rd (the first deadNodeCount built
  //      Byzantine and stopped), setPeers(), then rd.nextInt(nodeCount) until msgCount distinct live senders are drawn, each
  //      calling sendPeers (P2PNetwork.java:127-132) at once — on the host, with the draws the emit step would make (the
  //      shuffle of the sender's whole peer list, then the send's seed).  No conditional tasks: the calendar and
  //      fast-forward run it, like CasperIMD. ----
  std::vector<uint32_t> hPeerOff, hPeerIds;  // the peer graph (CSR), kept for the read-backs
  void p2pFloodInit(int N, int dead, int resend, int msgCount, int peersCount, int between) {
    requireNotInited();
    requireUnsharded("this protocol");  // the shuffles are drawn in the emit step, in creation order over all nodes
    if (N <= 0 || dead < 0 || resend < 0 || msgCount < 0 || peersCount < 0 || between < 0)
      throw std::invalid_argument("P2PFlood parameters must not be negative (nodeCount > 0)");
    if (between >= (1 << 20)) throw std::invalid_argument("delayBetweenSends must be below 2^20 (descriptor field)");
    if (resend >= (1 << 30)) throw std::invalid_argument("delayBeforeResent must be below 2^30");
    if (peersCount >= N)  // P2PNetwork.java:27-33
      throw std::invalid_argument("Wrong configuration: #nodes=" + std::to_string(N) + ", connection target=" + std::to_string(peersCount));
    const int live = N - std::min(dead, N);
    if (msgCount > live)
      throw std::invalid_argument("msgCount=" + std::to_string(msgCount) + " exceeds the " + std::to_string(live) +
                                  " live nodes: the reference never finds that many senders");
    checkLatencyBuilder();
    hm.buildNodes(N);
    for (int i = 0; i < std::min(dead, N); ++i) hm.nodes[(size_t)i].down = true;  // new P2PFloodNode(nb, true): stop()
    buildPeerGraph(hm.rd, N, peersCount, hPeerOff, hPeerIds);
    int maxDeg = 0;
    for (int n = 0; n < N; ++n) maxDeg = std::max(maxDeg, (int)(hPeerOff[(size_t)n + 1] - hPeerOff[(size_t)n]));
    if (maxDeg > PEERS_MAX)
      throw std::invalid_argument("the peer graph has a node of degree " + std::to_string(maxDeg) + ": the emit warp shuffles at most " +
                                  std::to_string(PEERS_MAX) + " peers");
    // Every node forwards each message at most once (a stopped node started again included), and a forward keeps at most its
    // degree of destinations: the record arenas never overflow, and the calendar holds every envelope in flight.
    const long long recs = (long long)N * std::max(1, msgCount);
    const long long dests = (long long)std::max(1, msgCount) * (long long)hPeerIds.size() + 1;
    if (recs > 0x7fffffffLL || dests > 0x7fffffffLL)
      throw std::invalid_argument("nodeCount x msgCount x degree does not fit the record arenas (2^31 entries)");
    tun.recCap = recs;
    recDestOverride = (int)dests;
    farWanted = recs + 1024;
    farEnabled = true;
    allocCommon(N, PROTO_P2PFLOOD);
    d.floodMsgs = msgCount;
    d.floodWords = std::max(1, (msgCount + 63) / 64);
    d.floodResend = resend;
    d.floodBetween = between;
    d.peerOff = dupload(hPeerOff);
    d.peerIds = dupload(hPeerIds);
    d.peerList = dalloc<int>(d.descCap);
    d.shufCap = d.newEvCap;
    d.forceShufSerial = forceShufSerial ? 1 : 0;
    d.byG = dalloc<int>(d.newEvCap);
    {
      std::vector<int> m1((size_t)d.newEvCap, -1);
      d.byGTick = dupload(m1);
    }
    d.descDraw = dalloc<int>(d.descCap);
    // the senders and their sendPeers, in draw order
    Dev hd = hostView();
    std::vector<int> cnt((size_t)N, 0);
    std::vector<unsigned long long> bits((size_t)N * d.floodWords, 0);
    std::vector<long long> sent((size_t)N, 0), doneAt((size_t)N, 0);
    std::vector<uint8_t> isSender((size_t)N, 0);
    std::vector<MultiRec> recs0;
    std::vector<uint32_t> recDst;
    std::vector<int> recArr;
    std::vector<std::vector<Ev>> near((size_t)d.ring);
    std::vector<FarEv> far;
    int farMin = 0x7fffffff;
    const int sendTime = 1 + resend;  // time + 1 + msg.localDelay, at time 0
    const int step = between > 0 ? between + 1 : 0;
    for (int k = 0; k < msgCount;) {
      const int from = hm.rd.nextInt(N);
      if (hm.nodes[(size_t)from].down || isSender[(size_t)from]) continue;
      isSender[(size_t)from] = 1;
      const int msg = k++;
      cnt[(size_t)from] = 1;  // msg.addToReceived(from)
      bits[(size_t)from * d.floodWords + (size_t)(msg >> 6)] |= 1ULL << (msg & 63);
      if (msgCount == 1) doneAt[(size_t)from] = 1;
      std::vector<uint32_t> list(hPeerIds.begin() + hPeerOff[(size_t)from], hPeerIds.begin() + hPeerOff[(size_t)from + 1]);
      for (int i = (int)list.size(); i > 1; --i) std::swap(list[(size_t)i - 1], list[(size_t)hm.rd.nextInt(i)]);  // Collections.shuffle
      const int32_t seed = hm.rd.nextInt();
      sent[(size_t)from] += (long long)list.size();
      struct Arr {
        int arrival;
        uint32_t dest;
      };
      std::vector<Arr> da;
      for (size_t i = 0; i < list.size(); ++i) {
        const int to = (int)list[i];
        if (hm.nodes[(size_t)from].down || hm.nodes[(size_t)to].down) continue;
        const int nt = latency(hd, from, to, pseudoRandom(to, seed));
        if (nt < msgDiscardTime) da.push_back({sendTime + (int)i * step + nt, (uint32_t)to});
      }
      std::stable_sort(da.begin(), da.end(), [](const Arr& a, const Arr& b) { return a.arrival < b.arrival; });
      if (da.empty()) continue;
      Ev ev;
      std::memset(&ev, 0, sizeof(ev));
      ev.pad = (uint32_t)sendTime + 1u;
      ev.from = (uint32_t)from;
      ev.meta = P2P_FLOOD;
      ev.pl = (unsigned long long)msg;
      ev.to = da[0].dest;
      ev.kind = EV_MSG;
      if (da.size() > 1) {
        MultiRec rc;
        std::memset(&rc, 0, sizeof(rc));
        rc.pad = ev.pad;
        rc.from = ev.from;
        rc.meta = ev.meta;
        rc.pl = ev.pl;
        rc.n = (uint32_t)da.size();
        rc.off = (uint32_t)recDst.size();
        ev.kind = EV_MULTI;
        ev.aux = (uint32_t)recs0.size();
        recs0.push_back(rc);
        for (const Arr& a : da) {
          recDst.push_back(a.dest);
          recArr.push_back(a.arrival);
        }
      }
      const int tgt = da[0].arrival;
      if (tgt < d.ring / 2) {
        near[(size_t)tgt].push_back(ev);
      } else {  // insertion order among calendar entries: creation order
        FarEv f;
        std::memset(&f, 0, sizeof(f));
        f.ev = ev;
        f.target = tgt;
        f.key = (unsigned long long)msg;
        far.push_back(f);
        farMin = std::min(farMin, tgt);
      }
    }
    for (int t = 0; t < d.ring; ++t)
      if (!near[(size_t)t].empty()) {
        const int c = (int)near[(size_t)t].size();
        if (c > d.bcap) throw std::runtime_error("bucket capacity too small for the initial sends");
        be->upload(d.buckets + (size_t)t * d.bcap, near[(size_t)t].data(), (size_t)c * sizeof(Ev));
        be->upload(d.bucketCount + t, &c, sizeof(int));
      }
    if (!far.empty()) be->upload(d.far, far.data(), far.size() * sizeof(FarEv));
    if (!recs0.empty()) {
      be->upload(d.rec, recs0.data(), recs0.size() * sizeof(MultiRec));
      be->upload(d.recDest, recDst.data(), recDst.size() * sizeof(uint32_t));
      be->upload(d.recArrival, recArr.data(), recArr.size() * sizeof(int));
    }
    be->upload(d.msgSent, sent.data(), sent.size() * sizeof(long long));
    be->upload(d.bytesSent, sent.data(), sent.size() * sizeof(long long));
    be->upload(d.doneAt, doneAt.data(), doneAt.size() * sizeof(long long));
    d.floodCnt = dupload(cnt);
    d.floodBits = dupload(bits);
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    c.callId = 1;
    c.recTop = (int)recs0.size();
    c.recDestTop = (int)recDst.size();
    c.rng = hm.rd.seed;
    c.farCnt = (int)far.size();
    c.farMin = farMin;
    c.nextEvent = 0;  // unknown: the first window looks for itself
    writeCtl(c);
    inited = true;
  }

  // ---- CasperIMD: the constructor builds the observer (CasperIMD.java:81-88); init(byzantineNode) the producers and
  //      attesters with their periodic tasks (:478-508) ----
  CasperParams cp{};
  bool casperConstructed = false;
  void casperConstruct(const CasperParams& p) {
    requireNotInited();
    if (casperConstructed) throw std::logic_error("already constructed");
    if (p.cycleLength <= 0 || p.blockProducersCount <= 0 || p.attestersPerRound <= 0) throw std::invalid_argument("cycleLength / blockProducersCount / attestersPerRound must be positive");
    if (p.blockConstructionTime <= 0 || p.attestationConstructionTime <= 0) throw std::invalid_argument("construction times must be positive (sendTime > time, Network.java:470-473)");
    checkLatencyBuilder();
    cp = p;
    hm.buildNodes(1);  // network.addObserver(new CasperNode(false, genesis) {})
    casperConstructed = true;
  }
  void casperInit(int byzDelay, int byzKind = CK_BYZ_WF) {
    requireNotInited();
    if (!casperConstructed) throw std::logic_error("CasperIMD not constructed");
    const int attCount = cp.attestersPerRound * cp.cycleLength;
    const int N = 1 + cp.blockProducersCount + attCount;
    if (CASPER_SLOT + byzDelay <= 0) throw std::invalid_argument("the Byzantine producer's first slot would start in the past");
    if (byzKind != CK_BYZ && byzKind != CK_BYZ_SF && byzKind != CK_BYZ_NS && byzKind != CK_BYZ_WF) throw std::invalid_argument("unknown Byzantine producer kind");
    if (sharded() && N > (int)KEY_SUB_MAX) throw std::invalid_argument("a node-sharded sendAll protocol holds at most 65535 nodes (ordering-key layout)");
    hm.buildNodes(N - 1);  // byzantine producer, producers 1.., attesters — in this order (:479-507); registering tasks draws nothing
    ringExtra = std::max(cp.blockConstructionTime, cp.attestationConstructionTime);
    farEnabled = true;
    long long slots = 4LL * (cp.attestersPerRound + 2) + 64;  // sendAll envelopes alive at once, with margin
    if (tun.recCap > slots) slots = tun.recCap;
    if (slots * N > 0x7fffffffLL) throw std::invalid_argument("attestersPerRound x nodes too large for the sendAll arena");
    recDestOverride = (int)(slots * N);
    if (!tun.recCap) tun.recCap = slots;
    const int maxVotes = (int)(tun.casperVotes ? tun.casperVotes : 6);
    long long maxBlocks = tun.casperBlocks ? tun.casperBlocks : (long long)cp.cycleLength * (maxVotes + 1) + 64;
    maxBlocks = (maxBlocks + 63) / 64 * 64;
    if (maxBlocks > 64 * CASPER_MAX_BLKWORDS) maxBlocks = 64 * CASPER_MAX_BLKWORDS;
    const int maxAtts = (attCount * maxVotes + 63) / 64 * 64;
    if (sharded()) {  // node ids split into G contiguous ranges (1 + producers + attesters is no power of two); the block /
                      // attestation tables are replicated inside the exchange region; periodic tasks are the only far envelopes
      unevenShards = true;
      shardFarOk = true;
      xProtoBytes = casperTabsBytes((int)maxBlocks, maxAtts, maxAtts / 64);
      xAllCapWanted = N / shardWorld + 64;
    }
    allocCommon(N, PROTO_CASPER);
    d.cCycle = cp.cycleLength;
    d.cBpCount = cp.blockProducersCount;
    d.cAttPerRound = cp.attestersPerRound;
    d.cAttCount = attCount;
    d.cBlockTime = cp.blockConstructionTime;
    d.cAttTime = cp.attestationConstructionTime;
    d.cRandomTies = cp.randomOnTies;
    d.cByzDelay = byzDelay;
    d.cMaxBlocks = (int)maxBlocks;
    d.cBlkWords = (int)(maxBlocks / 64);
    d.cMaxAtts = maxAtts;
    d.cAttWords = d.cMaxAtts / 64;
    d.cFirstAtt = 1 + cp.blockProducersCount;
    std::vector<uint8_t> kind((size_t)N, CK_ATTESTER);
    kind[0] = CK_OBSERVER;
    kind[1] = (uint8_t)byzKind;
    for (int i = 1; i < cp.blockProducersCount; ++i) kind[(size_t)(1 + i)] = CK_PRODUCER;
    d.cKind = dupload(kind);
    d.cHead = dallocNodes<int>();
    d.cVotes = dallocNodes<int>();
    d.cAttRecv = dallocNodes<unsigned long long>((size_t)d.cAttWords);
    std::vector<unsigned long long> br((size_t)N * d.cBlkWords, 0);
    for (int i = 0; i < N; ++i) br[(size_t)i * d.cBlkWords] = 1ULL;  // blocksReceivedByBlockId.put(genesis.id, genesis)
    d.cBlkRecv = duploadNodes(br, (size_t)d.cBlkWords);
    d.cToReeval = dallocNodes<unsigned long long>((size_t)d.cBlkWords);
    std::vector<int> minus1((size_t)d.cMaxBlocks, -1);
    CasperG g;
    std::memset(&g, 0, sizeof(g));
    g.nBlocks = 1;
    g.byzToSend = 1;
    if (sharded()) {
      std::vector<char> zero(xProtoBytes, 0);
      be->upload(d.peer[d.rank].proto, zero.data(), zero.size());
      CasperTabs t = casperTabsAt(d.peer[d.rank].proto, d.cMaxBlocks, d.cMaxAtts);
      d.cg = t.cg;
      d.cbHeight = t.cbHeight;
      d.cbParent = t.cbParent;
      d.cbProducer = t.cbProducer;
      d.cbTime = t.cbTime;
      d.cbIncluded = t.cbIncluded;
      d.attHead = t.attHead;
      d.attHeight = t.attHeight;
      be->upload(d.cbParent, minus1.data(), minus1.size() * sizeof(int));
      be->upload(d.cbProducer, minus1.data(), minus1.size() * sizeof(int));
    } else {
      d.cbHeight = dalloc<int>(d.cMaxBlocks);
      d.cbParent = dupload(minus1);
      d.cbProducer = dupload(minus1);
      d.cbTime = dalloc<int>(d.cMaxBlocks);
      d.cbIncluded = dalloc<unsigned long long>((size_t)d.cMaxBlocks * d.cAttWords);
      d.attHead = dalloc<int>(d.cMaxAtts);
      d.attHeight = dalloc<int>(d.cMaxAtts);
      d.cg = dalloc<CasperG>(1);
    }
    be->upload(d.cg, &g, sizeof(g));
    {  // randomOnTies: nodes suspended at a fork-choice tie (wtg_casper.cuh, casperResolveTies)
      std::vector<int> none((size_t)N, -1);
      d.cTieItem = dupload(none);
      d.cTieCnt = dalloc<int>(N);
      d.cTieList = dalloc<int>(N);
      d.cbItem = dalloc<int>(d.cMaxBlocks);
      d.cbTmp = dalloc<unsigned long long>((size_t)CASPER_MAX_NEW * d.cAttWords);
      d.cbTmpRow = dalloc<int>(CASPER_MAX_NEW * 5);
    }
    // sendAll machinery: records recycled over recSlots slots of N destinations
    d.allCap = N + 64;
    if (sharded()) d.allCap = d.xAllCap;
    d.allList = dalloc<int>(d.allCap);
    d.allWarps = 512;
    d.allTmp = dalloc<int>((size_t)d.allWarps * N);
    d.recSlots = std::min<int>(d.recCap, std::max(1, d.recDestCap / N));
    // periodic tasks in registration order (:481-506): near ones straight into their bucket, the others into the calendar
    struct Reg {
      int node, startAt;
    };
    std::vector<Reg> regs;
    regs.push_back({1, CASPER_SLOT + byzDelay});
    for (int i = 1; i < cp.blockProducersCount; ++i) regs.push_back({1 + i, CASPER_SLOT * (i + 1)});
    for (int i = 0; i < attCount; ++i) regs.push_back({d.cFirstAtt + i, CASPER_SLOT * (1 + i % cp.cycleLength) + 4000});
    std::vector<FarEv> far;
    std::vector<std::vector<Ev>> near((size_t)d.ring);
    std::vector<std::vector<unsigned long long>> nearKey((size_t)d.ring);
    int farMin = 0x7fffffff;
    unsigned long long seq = 0;
    for (const Reg& r : regs) {
      Ev ev;
      std::memset(&ev, 0, sizeof(ev));
      ev.pad = 1;  // registered at time 0 (Envelope.sendTime + 1)
      ev.kind = EV_PERIODIC;
      ev.to = (uint32_t)r.node;
      ev.from = (uint32_t)r.node;
      const bool mine = r.node >= d.n0 && r.node < d.n0 + d.nLoc;  // a shard keeps the tasks of its own nodes
      // insertion order = registration order; node-sharded: as the ordering key of "pass 0" (wtg_shard.cuh)
      const unsigned long long key = sharded() ? orderKey(0, (unsigned)seq) : seq;
      if (!mine) {
      } else if (r.startAt < d.ring / 2) {
        near[(size_t)r.startAt].push_back(ev);
        nearKey[(size_t)r.startAt].push_back(key);
      } else {
        FarEv f;
        std::memset(&f, 0, sizeof(f));
        f.ev = ev;
        f.target = r.startAt;
        f.key = key;
        far.push_back(f);
        farMin = std::min(farMin, r.startAt);
      }
      ++seq;
    }
    if ((int)far.size() > d.farCap) throw std::runtime_error("calendar capacity too small");
    if (!far.empty()) be->upload(d.far, far.data(), far.size() * sizeof(FarEv));
    for (int t = 0; t < d.ring; ++t)
      if (!near[(size_t)t].empty()) {
        if ((int)near[(size_t)t].size() > d.bcap) throw std::runtime_error("bucket capacity too small");
        be->upload(d.buckets + (size_t)t * d.bcap, near[(size_t)t].data(), near[(size_t)t].size() * sizeof(Ev));
        if (sharded()) be->upload(d.bucketKey + (size_t)t * d.bcap, nearKey[(size_t)t].data(), nearKey[(size_t)t].size() * sizeof(unsigned long long));
        int cnt = (int)near[(size_t)t].size();
        be->upload(d.bucketCount + t, &cnt, sizeof(int));
      }
    Ctl c;
    std::memset(&c, 0, sizeof(c));
    c.callId = 1;
    c.rng = hm.rd.seed;
    c.farCnt = (int)far.size();
    c.farMin = farMin;
    c.nextEvent = 0;  // unknown: the first window looks for itself
    writeCtl(c);
    inited = true;
  }

  // ---- sends issued by the caller between two runMs windows: network.send / sendAll (Network.java:341-366) and, for a
  //      block-chain network, the re-send of BlockChainNetwork.endPartition (BlockChainNetwork.java:46-54).  The caller's
  //      sends are descriptors like a handler's; only the emission half of the pipeline runs (backend mode 3). ----
  struct HostSend {
    int from;
    uint32_t meta;
    unsigned long long pl;
    std::vector<int> to;  // empty: sendAll
    int sendTime = 0;     // 0: time + 1
    int delay = 0;        // delaysBetweenMessage of a multi-destination send
  };
  int msgSizeOf(uint32_t) const {
    if (d.proto == PROTO_PINGPONG || d.proto == PROTO_CASPER) return 1;  // Message.size() default (messages/Message.java:27-29)
    throw std::logic_error("host-side sends are offered for PingPong and CasperIMD messages only");
  }
  void inject(const std::vector<HostSend>& sends) {
    requireInited();
    requireUnsharded("a send issued by the caller");
    if (sends.empty()) return;
    const int n = (int)sends.size();
    if (n > d.descCap || n > d.itemCap) throw std::runtime_error("too many sends in one call");
    Ctl c = readCtl();
    if (c.error) throwDeviceError(c);
    std::vector<Desc> descs((size_t)n);
    std::vector<uint32_t> scratch;
    std::vector<int> allList;
    std::vector<long long> sent((size_t)d.N, 0), bytes((size_t)d.N, 0);
    for (int i = 0; i < n; ++i) {
      const HostSend& hs = sends[(size_t)i];
      if (hs.from < 0 || hs.from >= d.N) throw std::invalid_argument("The from node is not in the network");  // Network.java:370-372
      Desc ds;
      std::memset(&ds, 0, sizeof(ds));
      ds.item = (uint32_t)(d.N + i);
      ds.sub = 0;
      ds.from = (uint32_t)hs.from;
      ds.evKind = EV_MSG;
      ds.meta = hs.meta;
      ds.pl = hs.pl;
      int fan = 0;
      if (hs.sendTime != 0) {
        if (hs.sendTime <= time) throw std::invalid_argument("sendTime <= time");  // Network.java:470-473
        ds.aux |= DESC_SENDTIME;
        ds.target = hs.sendTime;
      }
      if (hs.delay < 0 || hs.delay >= (1 << 20)) throw std::invalid_argument("delaysBetweenMessage");
      if (hs.delay > 0 && hs.to.size() < 2) throw std::invalid_argument("a delay between messages needs several destinations");
      ds.aux |= (uint32_t)hs.delay << DESC_DELAY_SHIFT;
      if (hs.to.empty()) {
        if (d.allCap <= 0) throw std::logic_error("sendAll from the host needs a protocol with the sendAll path (CasperIMD)");
        ds.dkind = DK_SEND_ALL;
        ds.evKind = EV_MULTI;
        ds.nDest = (uint32_t)d.N;
        ds.target = hs.sendTime != 0 ? hs.sendTime : time + 1;
        ds.aux = 0;
        allList.push_back(i);
        fan = d.N;
      } else if (hs.to.size() == 1) {
        if (hs.to[0] < 0 || hs.to[0] >= d.N) throw std::invalid_argument("The to node is not in the network");
        ds.dkind = DK_SEND_SINGLE;
        ds.to = (uint32_t)hs.to[0];
        ds.nDest = 1;
        fan = 1;
      } else {
        ds.dkind = DK_SEND_MULTI;
        ds.to = (uint32_t)scratch.size();
        ds.nDest = (uint32_t)hs.to.size();
        for (int t : hs.to) {
          if (t < 0 || t >= d.N) throw std::invalid_argument("The to node is not in the network");
          scratch.push_back((uint32_t)t);
        }
        if ((int)hs.to.size() > MAX_ACC) scratch.insert(scratch.end(), hs.to.size(), 0u);  // room for the arrivals (emitBigMulti)
        fan = (int)hs.to.size();
      }
      descs[(size_t)i] = ds;
      sent[(size_t)hs.from] += fan;
      bytes[(size_t)hs.from] += (long long)fan * msgSizeOf(hs.meta);
    }
    if ((int)scratch.size() > d.destScratchCap || (int)allList.size() > d.allCap)  // no handler runs in this pass: the whole scratch is the caller's
      throw std::runtime_error("too many destinations in one call");
    // control block of a "tick" at the current time with no bucket events, n items of one descriptor and one draw each
    c.tick = time;
    c.condMode = 0;
    c.nEv = 0;
    c.nItems = n;
    c.totalSlots = c.totalDraws = 0;
    c.hReject = 0;
    c.shufReject = 0;
    c.allCnt = (int)allList.size();
    c.nextEvent = 0;  // fast-forward: the next window looks for the earliest arrival itself
    const int per = d.descCap / ARENA_STRIPES;
    for (int t = 0; t < ARENA_STRIPES; ++t) {
      c.descCnt[t] = std::max(0, std::min(per, n - t * per));
      c.destCnt[t] = c.workCnt[t] = c.dueCnt[t] = c.taskCnt[t] = 0;
    }
    be->upload(d.desc, descs.data(), descs.size() * sizeof(Desc));
    std::vector<int> ones((size_t)n, 1), zerosN((size_t)d.N, 0);
    be->upload(d.evSlots, ones.data(), ones.size() * sizeof(int));
    be->upload(d.evDraws, ones.data(), ones.size() * sizeof(int));
    be->upload(d.condFired + condHalf(d, time), zerosN.data(), zerosN.size() * sizeof(int));
    if (!scratch.empty()) be->upload(d.destScratch, scratch.data(), scratch.size() * sizeof(uint32_t));
    if (!allList.empty()) be->upload(d.allList, allList.data(), allList.size() * sizeof(int));
    {  // msgSent++ / bytesSent += size per destination (Network.java:476-477)
      std::vector<long long> ms((size_t)d.N), bs((size_t)d.N);
      be->download(ms.data(), d.msgSent, ms.size() * sizeof(long long));
      be->download(bs.data(), d.bytesSent, bs.size() * sizeof(long long));
      for (int i = 0; i < d.N; ++i) {
        ms[(size_t)i] += sent[(size_t)i];
        bs[(size_t)i] += bytes[(size_t)i];
      }
      be->upload(d.msgSent, ms.data(), ms.size() * sizeof(long long));
      be->upload(d.bytesSent, bs.data(), bs.size() * sizeof(long long));
    }
    writeCtl(c);
    be->tick(d, 3);
    c = readCtl();
    if (c.error) throwDeviceError(c);
  }

  // ---- runMs  (Network.java:318-338) ----
  int runMs(int ms) {
    requireInited();
    if (sharded() && !linked) throw std::logic_error("node-sharded network: link the shards' exchange regions before runMs");
    if (ms <= 0) throw std::invalid_argument("Should be greater than 0. ms=" + std::to_string(ms));
    long long endAt = (long long)time + ms;
    if (endAt > 0x7fffffffLL) throw std::runtime_error("Maximum time reached!");
    Ctl c = readCtl();
    if (c.error) throwDeviceError(c);
    c.until = (int)endAt;
    c.callId += 1;  // a new nextMessage() call starts with the window
    c.didSomething = 0;
    if (d.ffwd) {  // no conditional tasks: only the milliseconds that hold an envelope are run
      if (c.nextEvent > endAt) {  // nothing arrives in this window
        c.time = (int)endAt;
        writeCtl(c);
        time = (int)endAt;
        return 0;
      }
      c.idle = 0;
      writeCtl(c);
      int grow = 8;
      for (long long done = 0;;) {
        int batch = (int)std::min<long long>(grow, std::max<long long>(1, ms - done));
        if (grow < 64) grow *= 2;  // busy windows: fewer host round trips
        runWindow(0, batch, 0);
        done += batch;
        c = readCtl();
        if (c.error) throwDeviceError(c);
        if (c.idle) break;
        if (done > 2LL * ms + 16) throw std::runtime_error("internal: fast-forward did not converge");
      }
      time = (int)endAt;
      if (c.time != time) throw std::runtime_error("internal: device clock out of step");
      return c.didSomething ? 1 : 0;
    }
    writeCtl(c);
    runWindow(pendingAtNow ? 1 : 0, ms, 1);
    pendingAtNow = false;
    c = readCtl();
    if (c.error) throwDeviceError(c);
    time = (int)endAt;
    if (c.time != time) throw std::runtime_error("internal: device clock out of step");
    return c.didSomething ? 1 : 0;
  }
  void throwDeviceError(const Ctl& c) {
    static const char* names[] = {"ok", "time-bucket capacity exceeded", "toVerify queue capacity exceeded", "payload pool exhausted",
                                  "arrival beyond the time ring", "descriptor arena exceeded", "multi-destination record arena exceeded",
                                  "deferred-free list exceeded", "internal error", "inbox overflow", "far-future calendar exceeded",
                                  "the protocol reached a state where the reference throws (IllegalState/IllegalArgument)",
                                  "situation not supported by the device path"};
    throw std::runtime_error(std::string("device engine error: ") + names[c.error < 13 ? c.error : 8] + " (detail " + std::to_string(c.errorDetail) + ")");
  }

  // node-sharded runs: a multi-destination envelope has one bucket entry on every shard that owns a destination of its next
  // group; msgs.size() counts it once — on the shard that owns the group's first destination
  int countBucket(int slot, int cnt) {
    if (!sharded()) return cnt;
    std::vector<Ev> evs((size_t)cnt);
    be->download(evs.data(), d.buckets + (size_t)slot * (size_t)d.bcap, evs.size() * sizeof(Ev));
    int c = 0;
    for (const Ev& e : evs) {
      if (e.kind != EV_MULTI) {
        ++c;
        continue;
      }
      MultiRec rc;
      be->download(&rc, d.rec + e.aux, sizeof(MultiRec));
      uint32_t first = 0;  // replicated records: the group starts at Ev.pl; shipped record copies: at their cursor
      be->download(&first, d.recDest + rc.off + (d.allCap > 0 ? (uint32_t)e.pl : rc.cur), sizeof(uint32_t));
      if (ownerOf(d, (int)first) == d.rank) ++c;
    }
    return c;
  }
  int msgsSize() {
    requireInited();
    std::vector<int> bc(d.ring);
    be->sync();
    be->download(bc.data(), d.bucketCount, sizeof(int) * d.ring);
    long long s = 0;
    for (int b = 0; b < d.ring; ++b)
      if (bc[(size_t)b] > 0) s += countBucket(b, bc[(size_t)b]);
    if (d.farCap > 0) s += farHeld();
    return (int)s;
  }
  // entries of the far-future calendar: farCnt keeps counting past farCap once the calendar has overflowed
  int farHeld() { return std::min(readCtl().farCnt, d.farCap); }
  int msgsSizeAt(int t) {
    requireInited();
    if (t < time) return 0;
    int v = 0;
    be->sync();
    if (t < time + d.ring) be->download(&v, d.bucketCount + (t & ringMask), sizeof(int));
    if (v > 0) v = countBucket(t & ringMask, v);
    if (d.farCap > 0) {
      std::vector<FarEv> far((size_t)farHeld());
      if (!far.empty()) be->download(far.data(), d.far, far.size() * sizeof(FarEv));
      for (const FarEv& f : far)
        if (f.target == t) ++v;
    }
    return v;
  }

  // network.msgs.peekMessages() (Network.java:279-286, Envelope.infos :34-37, :145-154, :219-227, :297-300): one
  // EnvelopeInfo {from, to, sentAt, arrivingAt, message} per pending arrival — every remaining destination of a
  // multi-destination envelope counts — sorted by arrival time (EnvelopeInfo.compareTo; ties here by from, to, sentAt).
  // Host-side read-back of the time ring (and of the far-future calendar); rows: from, to, sentAt (-1: not recorded),
  // arrivingAt, event kind (EV_*), message type (Ev.meta).  Returns the number of pending arrivals; at most `cap` are written.
  struct PeekRow {
    int from, to, sentAt, arrivingAt, kind;
    uint32_t meta;
  };
  long long peekMessages(std::vector<PeekRow>& out, long long cap) {
    requireInited();
    out.clear();
    long long total = 0;
    std::vector<int> bc(d.ring);
    be->sync();
    be->download(bc.data(), d.bucketCount, sizeof(int) * d.ring);
    std::vector<Ev> evs;
    std::vector<uint32_t> rd;
    std::vector<int> ra;
    // node-sharded sendAll protocols: the records are replicated and a shard holds a bucket entry only while it owns a
    // destination of the envelope's next group, so the pending arrivals at this shard's nodes are read from the records
    // themselves (a slot is live while its last arrival lies ahead; arrivals up to `time` have been delivered)
    const bool replicated = sharded() && d.allCap > 0;
    if (replicated) {
      std::vector<MultiRec> recs((size_t)d.recSlots);
      be->download(recs.data(), d.rec, recs.size() * sizeof(MultiRec));
      for (const MultiRec& rc : recs) {
        if (rc.n == 0) continue;
        int last = 0;
        be->download(&last, d.recArrival + rc.off + rc.n - 1, sizeof(int));
        if (last <= time) continue;
        rd.resize(rc.n);
        ra.resize(rc.n);
        be->download(rd.data(), d.recDest + rc.off, sizeof(uint32_t) * rc.n);
        be->download(ra.data(), d.recArrival + rc.off, sizeof(int) * rc.n);
        for (uint32_t i = 0; i < rc.n; ++i) {
          if (ra[i] <= time || ownerOf(d, (int)rd[i]) != d.rank) continue;
          ++total;
          if ((long long)out.size() < cap) out.push_back(PeekRow{(int)rc.from, (int)rd[i], (int)rc.pad - 1, ra[i], (int)EV_MSG, rc.meta});
        }
      }
    }
    auto addOne = [&](const Ev& e, int arrival) {
      if (e.kind == EV_MULTI && replicated) return;
      if (e.kind == EV_MULTI) {
        MultiRec rc;
        be->download(&rc, d.rec + e.aux, sizeof(MultiRec));
        const int m = (int)rc.n - (int)rc.cur;
        if (m <= 0) return;
        if (sharded()) {  // the envelope has an entry (and a copy of the record) on every shard that owns a destination of its
                          // next group: the shard of the group's first destination reports all remaining destinations
          uint32_t first = 0;
          be->download(&first, d.recDest + rc.off + rc.cur, sizeof(uint32_t));
          if (ownerOf(d, (int)first) != d.rank) return;
        }
        total += m;
        long long room = cap - (long long)out.size();
        int take = (int)std::max<long long>(0, std::min<long long>(room, m));
        if (take > 0) {
          rd.resize((size_t)take);
          ra.resize((size_t)take);
          be->download(rd.data(), d.recDest + rc.off + rc.cur, sizeof(uint32_t) * (size_t)take);
          be->download(ra.data(), d.recArrival + rc.off + rc.cur, sizeof(int) * (size_t)take);
          for (int i = 0; i < take; ++i)
            out.push_back(PeekRow{(int)rc.from, (int)rd[(size_t)i], (int)rc.pad - 1, ra[(size_t)i], (int)EV_MSG, rc.meta});
        }
      } else {
        total += 1;
        // tasks are self-addressed envelopes (Network.java:505-519); Ev.from of a task is protocol payload (e.g. the signer)
        const int from = (e.kind == EV_TASK || e.kind == EV_PERIODIC) ? (int)e.to : (int)e.from;
        if ((long long)out.size() < cap) out.push_back(PeekRow{from, (int)e.to, (int)e.pad - 1, arrival, (int)e.kind, e.meta});
      }
    };
    for (int b = 0; b < d.ring; ++b) {
      if (bc[(size_t)b] <= 0) continue;
      const int arrival = time + ((b - time) & ringMask);
      evs.resize((size_t)bc[(size_t)b]);
      be->download(evs.data(), d.buckets + (size_t)b * (size_t)d.bcap, evs.size() * sizeof(Ev));
      for (const Ev& e : evs) addOne(e, arrival);
    }
    if (d.farCap > 0) {
      std::vector<FarEv> far((size_t)farHeld());
      if (!far.empty()) be->download(far.data(), d.far, far.size() * sizeof(FarEv));
      for (const FarEv& f : far) addOne(f.ev, f.target);
    }
    std::stable_sort(out.begin(), out.end(), [](const PeekRow& a, const PeekRow& b) {
      if (a.arrivingAt != b.arrivingAt) return a.arrivingAt < b.arrivingAt;
      if (a.from != b.from) return a.from < b.from;
      if (a.to != b.to) return a.to < b.to;
      return a.sentAt < b.sentAt;
    });
    return total;
  }

  void setDown(int id, bool down) {
    requireInited();
    if (id < 0 || id >= d.N) throw std::invalid_argument("node id");
    hm.nodes[id].down = down;
    uint8_t v = down ? 1 : 0;
    be->sync();
    be->upload(d.ndown + id, &v, 1);
    if (d.proto == PROTO_HANDEL) {  // the cached per-level minimum rank of the down peers is stale now
      std::vector<int> dirty((size_t)d.nLoc * d.L, -2147483647 - 1);
      be->upload(d.hBizNoHit + (size_t)d.n0 * d.L, dirty.data(), dirty.size() * sizeof(int));
    }
  }
  void uploadPartitions() {
    std::vector<uint8_t> part(d.N);
    for (int i = 0; i < d.N; ++i) {
      int pId = 0;  // Network.java:639-649
      for (int x : partitionsInX) {
        if (x > hm.nodes[i].x) break;
        pId++;
      }
      part[i] = (uint8_t)pId;
    }
    be->sync();
    be->upload(d.npart, part.data(), part.size());
  }
  void partition(float part) {  // Network.java:693-703
    requireInited();
    if (part <= 0 || part >= 1) throw std::invalid_argument("part needs to be a percentage between 0 & 100 excluded");
    int xPoint = (int)(2000 * part);
    if (std::find(partitionsInX.begin(), partitionsInX.end(), xPoint) != partitionsInX.end())
      throw std::invalid_argument("this partition exists already");
    partitionsInX.push_back(xPoint);
    std::sort(partitionsInX.begin(), partitionsInX.end());
    uploadPartitions();
  }
  void endPartition() {
    requireInited();
    partitionsInX.clear();
    uploadPartitions();
    if (d.proto == PROTO_CASPER) {  // BlockChainNetwork.endPartition (BlockChainNetwork.java:46-54): every node re-sends its head to everybody
      if (d.recSlots < d.N + 64) throw std::runtime_error("endPartition of a block-chain network keeps one sendAll per node in flight: raise rec_cap to nodes + 64 before init()");
      std::vector<int> heads((size_t)d.N);
      fetch(heads.data(), d.cHead, heads.size());
      std::vector<HostSend> sends;
      for (int i = 0; i < d.N; ++i) sends.push_back(HostSend{i, CM_BLOCK, (unsigned long long)(uint32_t)heads[(size_t)i], {}});
      inject(sends);
    }
  }

  // striped statistics summed (or max-ed) over the slots
  std::vector<unsigned long long> readStats() {
    std::vector<unsigned long long> raw((size_t)STAT_SLOTS * ST_COUNT), out(ST_COUNT, 0);
    be->sync();
    be->download(raw.data(), d.stats, raw.size() * sizeof(unsigned long long));
    for (int sl = 0; sl < STAT_SLOTS; ++sl)
      for (int k = 0; k < ST_COUNT; ++k) {
        unsigned long long v = raw[(size_t)sl * ST_COUNT + k];
        if (k == ST_MAXQUEUE || k == ST_MAXINBOX)
          out[k] = std::max(out[k], v);
        else
          out[k] += v;
      }
    return out;
  }
  template <class T>
  void fetch(T* out, const T* dev, size_t n) {
    be->sync();
    be->download(out, dev, n * sizeof(T));
  }

 private:
  // a whole runMs window: pre0 passes of mode 0, count1 clock ticks, post2 end-of-window passes
  void runWindow(int pre0, int count1, int post2) {
    if (pre0) be->tick(d, 0);
    if (count1) be->ticks(d, count1);
    if (post2) be->tick(d, 2);
  }
};

}  // namespace wtg
