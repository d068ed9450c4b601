// wittgenstein_b200 — H100-native discrete-event engine behind the reference's
// Protocol / Network / Node / Message surface.  Shared POD types (host + device).
//
// Data layout in HBM (see DESIGN.md §3):
//   * node attributes / counters: SoA arrays indexed by node id
//   * time ring: RING buckets of fixed capacity, each an append-only array of 32-byte Ev
//     records kept in *insertion order* (the reference's per-ms list is LIFO by insertion:
//     core/Network.java:145-147, so processing position = count-1-index)
//   * GSF: three N-bit rows per node (verified / individual-seen / individual-verified);
//     level l of a node is the aligned sub-range (block) of the row, so no per-level bitsets
//   * payload pools: per-level slabs of 2^(l-1) bits for in-flight / queued aggregates
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define WTG_HD __host__ __device__ __forceinline__
#else
#define WTG_HD inline
#endif

namespace wtg {

constexpr int POOL_STRIPES = 64;     // independent free stacks per pool level (allocation contention / 64)
constexpr int ARENA_STRIPES = 64;    // per-tick arenas are striped by node id for the same reason
constexpr int MS_SUB_ENVELOPES = 256; // new envelopes per warp of a multisplit block (chunk = Dev.msWarps * 256)
constexpr int MAX_LEVELS = 24;
constexpr int MAX_ACC = 16;          // max destinations of a protocol multi-send handled on device
constexpr int INLINE_MAX_LEVEL = 7;  // level-l block has 2^(l-1) bits: <= 64 bits for l <= 7
constexpr int MAX_DIST = 1144;       // core/Node.java:17-18
constexpr int MAX_SHARDS = 8;        // node-id shards of one simulation (one GPU each); power of two

// protocols
enum : int { PROTO_NONE = 0, PROTO_PINGPONG = 1, PROTO_GSF = 2, PROTO_SANFERMIN = 3, PROTO_HANDEL = 4, PROTO_CASPER = 5, PROTO_CAPPOS = 6,
             PROTO_SLUSH = 7, PROTO_SNOWFLAKE = 8, PROTO_P2PFLOOD = 9 };

// event kinds (Ev.kind)
enum : uint32_t {
  EV_MSG = 0,       // single-destination message      (Envelope.SingleDestEnvelope)
  EV_MULTI = 1,     // multi-destination message, aux = record index (Envelope.MultipleDest*Envelope)
  EV_TASK = 2,      // one-shot task on node `to`       (messages/Task.java)
  EV_PERIODIC = 3   // periodic task on node `to`       (messages/PeriodicTask.java)
};

// message / payload kinds, low 2 bits of Ev.meta / QEntry.meta for GSF
enum : uint32_t {
  PK_INLINE = 0,  // bits of the level block stored in `pl` (block <= 64 bits, bits in row position)
  PK_POOL = 1,    // bits stored in a pool slab; pl = slot | (cardinality << 32)
  PK_FULL = 2,    // the aligned 2^k block around `from` (k in meta)
  PK_INDIV = 3    // the single signature of `from`
};
WTG_HD uint32_t metaMake(uint32_t kind, uint32_t level, uint32_t k) { return kind | (level << 2) | (k << 7); }
WTG_HD uint32_t metaKind(uint32_t m) { return m & 3u; }
WTG_HD uint32_t metaLevel(uint32_t m) { return (m >> 2) & 31u; }
WTG_HD uint32_t metaK(uint32_t m) { return (m >> 7) & 31u; }
// PingPong message types (Ev.meta)
enum : uint32_t { PP_PING = 1, PP_PONG = 2 };
// SanFermin message / task types (Ev.meta); Ev.pl = level | (value << 32)
enum : uint32_t { SF_REQ = 1, SF_REPLY_OK = 2, SF_REPLY_NO = 3, SF_T_GO = 4, SF_T_TIMEOUT = 5, SF_T_TRANSITION = 6 };
// CasperIMD message / task types (Ev.meta); Ev.pl = attestation index, block index, or block | height << 32
enum : uint32_t { CM_ATT = 1, CM_BLOCK = 2, CT_BUILD = 3 };
// CasperIMD node kinds (CasperIMD.java: observer :87, BlockProducer :365, Attester :444, ByzBlockProducerWF :647)
enum : uint8_t { CK_OBSERVER = 0, CK_PRODUCER = 1, CK_ATTESTER = 2, CK_BYZ = 3, CK_BYZ_SF = 4, CK_BYZ_NS = 5, CK_BYZ_WF = 6 };
constexpr int CASPER_SLOT = 8000;  // CasperParemeters.SLOT_DURATION (CasperIMD.java:19)
constexpr int CASPER_MAX_BLKWORDS = 8;  // at most 512 blocks per run on the device
// SanFerminCappos message / task types (Ev.meta); Ev.pl = level | (value << 32)
enum : uint32_t { CP_SWAP_REPLY = 1, CP_SWAP = 2, CP_T_GO = 4, CP_T_TIMEOUT = 5, CP_T_TRANSITION = 6 };
constexpr int SHUFFLE_MAX = 64;          // longest destination list shuffled before a send (candidateCount + 1)
constexpr uint32_t DESC_SHUFFLEK = 2u;   // Desc.aux: Collections.shuffle of the nDest destinations before the send (nDest - 1 draws + rejections)
constexpr uint32_t DESC_SENDTIME = 4u;   // Desc.aux: Desc.target holds the explicit send time (send(m, sendTime, from, ...), Network.java:369-447)
constexpr int DESC_DELAY_SHIFT = 8;      // Desc.aux >> 8: delaysBetweenMessage of a multi-destination send (Network.java:420-467)
constexpr uint32_t DESC_SHUFFLE2 = 1u;  // Desc.aux: Collections.shuffle of the 2 destinations before the send (one extra draw)
constexpr uint32_t DESC_SAMPLEK = 8u;   // Desc.aux: the nDest destinations are drawn at emission (Slush / Snowflake randomRemotes:
                                        // one nextInt(N) per attempt until nDest distinct ids other than the sender's; nDest draws
                                        // when no attempt repeats an id or hits the sender)
// Slush / Snowflake message types (Ev.meta); Ev.pl = query id | (colour << 32)
enum : uint32_t { AV_QUERY = 1, AV_ANSWER = 2 };
constexpr uint32_t DESC_PEERS = 16u;  // Desc.aux: the destinations are the CSR peer row of Desc.from without node Desc.to (nDest of
                                      // them), shuffled at emission by k_emit_peers (P2PFlood's FloodMessage forward)
constexpr int PEERS_MAX = 256;        // longest peer list one emit warp shuffles (P2PFlood: maximum degree of the graph)
// P2PFlood message type (Ev.meta); Ev.pl = index of the originating message (init's draw order)
enum : uint32_t { P2P_FLOOD = 1 };

struct Ev {  // 32 bytes: one in-flight envelope / task
  uint32_t kind;
  uint32_t to;
  uint32_t from;
  uint32_t meta;
  uint64_t pl;
  uint32_t aux;
  uint32_t pad;
};

struct QEntry {  // 16 bytes: one entry of a GSF node's toVerify list
  uint32_t from;
  uint32_t meta;
  uint64_t pl;
};

struct HQEntry {  // 32 bytes: one Handel SigToVerify (protocols/Handel.java:919-938) + cached evaluation
  uint32_t from;
  uint32_t meta;  // payload kind | level << 2 | k << 7 | badSig << 12
  uint64_t pl;
  uint32_t rank;
  uint32_t id;    // identity of the object (toVerifyAgg.remove(vs) is by reference)
  int32_t s;      // sizeIfIncluded, valid while qStamp == lvVer of the level
  int32_t score;  // score(level, sig)
};

struct MultiRec {  // multi-destination envelope: sorted destinations + explicit arrivals
  uint32_t from;
  uint32_t meta;
  uint64_t pl;
  uint32_t n;
  uint32_t cur;
  uint32_t off;  // offset into recDest / recArrival
  uint32_t pad;
};

// descriptor kinds: what a handler asks the engine to do (in program order)
enum : uint32_t {
  DK_SEND_SINGLE = 0,  // network.send(msg, from, to): one rd.nextInt()
  DK_SEND_MULTI = 1,   // network.send(msg, from, dests): one rd.nextInt()
  DK_INSERT_AT = 2,    // sendArriveAt / registerTask / multi-dest re-push: no draw
  DK_SEND_ALL = 3      // network.sendAll(msg, sendTime, from): one rd.nextInt(); Desc.target = sendTime
};
struct Desc {  // 48 bytes
  uint32_t dkind;
  uint32_t item;  // scan item (N + pos for events)
  uint32_t sub;   // program-order index inside the event
  uint32_t from;
  uint32_t to;      // SINGLE: dest; MULTI: offset into destScratch; INSERT_AT: dest node
  uint32_t nDest;   // MULTI
  uint32_t evKind;  // kind of the Ev to create
  uint32_t meta;
  uint64_t pl;
  int32_t target;  // INSERT_AT: arrival tick
  uint32_t aux;
};

// latency model kinds (device form: integer tables built on the host, SURVEY.md H7)
enum : int {
  LAT_DIST_DELTA = 0,  // tab[dist*100+delta]           NetworkLatencyByDistanceWJitter
  LAT_CITY = 1,        // same city -> 1 else max(1, base[cf*11+ct] + jit[delta])   AwsRegionNetworkLatency
  LAT_CONST = 2,       // param                          NetworkFixedLatency / NetworkNoLatency
  LAT_DELTA = 3,       // tab[delta]                     NetworkUniformLatency / MeasuredNetworkLatency
  LAT_DELTA_2X = 4,    // max(1, extra+extra+tab[delta]) then extras again (EthScanNetworkLatency quirk)
  LAT_DIST = 5,        // tab[dist]                      IC3NetworkLatency
  LAT_CITY_MAT = 6     // tab[(cityFrom * K + cityTo) * stride + (stride == 100 ? delta : 0)]; K = param & 0xffff, stride = param >> 16 ? 100 : 1
                       //                                NetworkLatencyByCity / NetworkLatencyByCityWJitter
};

struct FarEv {  // an envelope whose arrival lies beyond the time ring's horizon (periodic tasks with long periods)
  Ev ev;
  int target;
  int pad;
  unsigned long long key;  // (creation tick << 32) | creation index: insertion order among far envelopes
};

// ---- node-sharded simulation (DESIGN.md §8): what the shards exchange every pipeline pass ----
// Shard r owns the ids [r * perShard, (r + 1) * perShard) (the last one may hold fewer).  Every bucket entry carries an ordering key
//   (creating pass << 40) | (creation index << 16) | (65535 - j)    j = position inside a multi-destination record
// so that "processed earlier" (LIFO by insertion, Network.java:145-147) == larger key on every shard.  (16 bits of position:
// a sendAll record holds one destination per node.)
constexpr unsigned KEY_SUB_MAX = 65535u;
constexpr int KEY_G_SHIFT = 16, KEY_PASS_SHIFT = 40;
struct XItem {  // one scan item of a shard, in its local processing order
  unsigned long long key;
  uint32_t ps, pd;  // exclusive prefix of (slots, draws) over the shard's items
};
struct XHdr {  // per pass and shard
  int seq, nEv, nItems, condSlots, condDraws, itemSlots, itemDraws, error;
};
struct XBegin {  // fast-forwarding protocols (CasperIMD): what a shard knows about the next millisecond that holds an event
  int seq, next, after, error;
};
struct XPick {  // Handel: the picks (rd.nextInt(k) of checkSigs) a shard presumes for this pass, one draw each
  int seq, picks, error, pad;
};
struct XAll {  // a sendAll of this pass: every shard builds the same sorted record from it (the record is replicated, not shipped)
  uint32_t from, meta;
  unsigned long long pl;
  int sendTime, g;
  unsigned long long draw;
};
constexpr uint32_t META_STAGED = 1u << 15;  // GSF / Handel: the pooled payload still sits in the staging area written by shard (meta >> 16) & 7
constexpr int META_SRC_SHIFT = 16;
struct MultiRec;
struct Ev;
struct Peer {  // exchange region of one shard as mapped into this process (own region included: peer[rank])
  XHdr* hdr;            // [G]            written by shard q at [q]
  XItem* items;         // [G][xItemCap]  written by shard q at [q][*]
  int* flags;           // [4][G]         pass sequence number of the last completed publication (0: items, 1: envelopes, 2: next event,
                        //                3: Handel picks)
  Ev* newEv;            // [newEvCap]     this tick's new envelopes, indexed by global creation index
  int* newTarget;       // [newEvCap]     arrival tick, -1 = nothing for this shard
  unsigned long long* stage;  // [2][G][stageCapWords] pooled payloads of envelopes addressed to this shard
  MultiRec* rec;        // [G][recCap / G] multi-destination records, one sub-arena per sending shard
  uint32_t* recDest;    // [G][recDestCap / G]
  int* recArrival;      // [G][recDestCap / G]
  XBegin* beg;          // [G]            written by shard q at [q] at the start of a pass (fast-forwarding protocols)
  XAll* all;            // [G][xAllCap]   sendAll descriptors of the pass, written by shard q at [q][*]
  int* allCnt;          // [G]
  char* proto;          // protocol-specific: CasperIMD's block / attestation tables, replicated on every shard (writers store
                        // to all copies); Handel's pick exchange (XPick [G], then k of every pick [G][perShard], wtg_handel.cuh)
};

struct CasperG {  // CasperIMD: block counter and the Byzantine producer's scalars (CasperIMD.java:511-518, 648-649)
  int nBlocks;    // blocks created so far, genesis included (Block.blockId, per engine)
  int byzToSend, byzH, byzLate, byzOnTime;
  int createdThisTick;  // two blocks created in one millisecond would need the reference's event order for their ids
  int byzDirect, byzOlder, byzNotBest, byzSkipped;  // onDirectFather, onOlderAncestor, incNotTheBestFather (:515-517), skipped (:615)
  int pad[2];
};

struct Ctl {  // device-resident control block (one per engine)
  int time;       // network.time
  int until;      // end of the current runMs window (inclusive)
  int tick;       // tick being processed
  int condMode;   // 0 = no conditional-task pass, 1 = normal, 2 = end-of-window overshoot pass
  int nEv;        // events in this tick's bucket
  int nItems;     // scan items this tick (N + nEv)
  int totalSlots, totalDraws;
  uint32_t callId;  // identity of the reference's current nextMessage() call (conditional-task snapshot)
  int didSomething;
  unsigned long long rng;  // java.util.Random state
  int error;               // first error code (0 = ok)
  int errorDetail;
  int recTop, recDestTop;  // multi-destination record arenas
  int hReject;             // Handel: some nextInt(k) of this tick's conditional pass hit the rejection loop
  int farCnt, farMin;      // far-future calendar: entries, earliest arrival (INT_MAX when empty)
  int idle;                // fast-forward: nothing left to do before `until`
  int nextEvent;           // fast-forward: earliest arrival after `until` known when the window went idle
  int allCnt;              // sendAll descriptors of this tick
  int shufReject;          // some Collections.shuffle of this tick hit nextInt's rejection loop: draw indices are re-derived serially
  int maxBucket;
  unsigned long long statDraws, statEvents;
  int descCnt[ARENA_STRIPES];   // descriptors allocated this tick, per stripe (stripe = node id & 63)
  int destCnt[ARENA_STRIPES];   // multi-send destination scratch, per stripe
  int freeCnt[ARENA_STRIPES];   // deferred payload frees, per stripe
  int workCnt[ARENA_STRIPES];   // stale pooled queue entries to re-score this tick, per stripe
  int dueCnt[ARENA_STRIPES];    // nodes whose conditional task runs this tick, per stripe
  int taskCnt[ARENA_STRIPES];   // nodes with task events this tick, per stripe
  // ---- node-sharded simulation ----
  int xseq;                      // pipeline passes so far (identical on every shard): sequence number of the exchanges
  int nEvGlobal;                 // bucket entries of this tick over all shards
  int condXoffS, condXoffD;      // creation / draw index of this shard's first conditional-task insert
  int allCondS, allCondD;        // conditional-task inserts / draws of all shards
  int stageTop[MAX_SHARDS];      // words staged for shard q in this pass
  int xRecTop[MAX_SHARDS];       // records / destinations allocated in this shard's sub-arena of shard q
  int xRecDestTop[MAX_SHARDS];
  int tieCnt;                    // CasperIMD randomOnTies: nodes suspended at a fork-choice tie in this pass
  int allSeq;                    // sendAll envelopes created so far over all shards: the next record slot (replicated records)
  int xNext, xAfter;             // global results of the begin exchange of this pass
  int poolMinFree[MAX_LEVELS];                 // low-water mark of free slots per level (sampled at tick end)
  int poolFreeCnt[MAX_LEVELS][POOL_STRIPES];   // free slots per (level, stripe)
  long long serialPasses;        // passes whose draw indices shuffleSerial re-derived (shuffle rejections, sample collisions)
  int peerCnt;                   // DESC_PEERS descriptors of this pass (P2PFlood forwards, emitted by k_emit_peers)
  // GSF's checkSigs reads its clock from these: tick and callId of the pass it belongs to.  tickBegin sets them to the
  // pass's own; k_cond_begin sets them to the next pass's when that pass's checkSigs runs ahead (DESIGN.md §4)
  int condTick;
  uint32_t condCall;
  int allRecBase;  // recTop when this pass's sendAlls began taking record slots (CasperIMD's recycled slots, one engine)
};

// striped statistics (node-id striping keeps hot-path counters off a single L2 address)
enum : int {
  ST_DELIVERIES = 0, ST_TASKS, ST_CONDRUNS, ST_EVALENTRIES, ST_EVALWORDS, ST_UPDATES, ST_CYCLES, ST_SENDS, ST_MULTISENDS,
  ST_SENDWORDS, ST_EVALPOOL, ST_UPDATEWORDS, ST_MAXQUEUE, ST_MAXINBOX, ST_COUNT = 16
};
constexpr int STAT_SLOTS = 1024;

enum : int {
  ERR_NONE = 0,
  ERR_BUCKET_OVERFLOW = 1,
  ERR_QUEUE_OVERFLOW = 2,
  ERR_POOL_EXHAUSTED = 3,
  ERR_FAR_FUTURE = 4,
  ERR_DESC_OVERFLOW = 5,
  ERR_REC_OVERFLOW = 6,
  ERR_FREE_OVERFLOW = 7,
  ERR_INTERNAL = 8,
  ERR_INBOX_OVERFLOW = 9,
  ERR_FAR_OVERFLOW = 10,
  ERR_PROTO_STATE = 11,   // the reference would have thrown IllegalStateException / IllegalArgumentException in a handler
  ERR_UNSUPPORTED = 12,   // a situation the device path does not implement (detail says which)
  ERR_PEER_TIMEOUT = 13,  // a shard did not publish its part of the exchange in time
  ERR_PEER_ERROR = 14,    // another shard reported an error
  ERR_STAGE_OVERFLOW = 15 // staging area for cross-shard payloads exceeded
};

// All device pointers + sizes; passed by value to kernels.
struct Dev {
  // ---- sizes / parameters ----
  int N, L, W64;
  int ring;      // buckets in the time ring (power of two > largest latency + period)
  int msChunks;  // rows of msCount
  int msWarps;   // warps (histograms over the ring) per multisplit block: 8, fewer for very long rings
  int proto;
  int threshold, timeoutPerLevel, period, accel;
  int qcap, bcap;
  int msgDiscardTime;
  int descCap, destScratchCap, recCap, recDestCap, freeCap, newEvCap, itemCap, workCap;
  int latKind, latParam;
  int peerBits;  // 16 or 32
  // ---- node-sharded simulation: this engine owns the ids [n0, n0 + nLoc); per-node arrays hold nLoc rows and are
  //      addressed by global id (their base pointers are biased by -n0 rows); node attributes are replicated ----
  int n0, nLoc, G, rank, ownShift;
  int xItemCap, stageCapWords, xRecCap, xRecDestCap;
  int perShard;   // ids per shard (ceil(N / G)); ownShift = log2(perShard) when that is a power of two, else -1
  int xAllCap;    // sendAll descriptors per pass and shard (node-sharded CasperIMD)
  Peer peer[MAX_SHARDS];
  unsigned long long* bucketKey;  // [ring][bcap] ordering key of every bucket entry (sharded runs only)
  unsigned long long* itemKey;    // [itemCap]
  uint32_t* xoffS;                // [itemCap] creation indices / draws of the other shards that precede the item
  uint32_t* xoffD;
  // ---- control ----
  Ctl* ctl;
  unsigned long long* stats;  // [STAT_SLOTS][ST_COUNT]
  // ---- nodes ----
  int16_t* nx;
  int16_t* ny;
  int16_t* nextra;
  uint8_t* ncity;
  uint8_t* ndown;
  uint8_t* npart;
  long long* msgReceived;
  long long* msgSent;
  long long* bytesSent;
  long long* bytesReceived;
  long long* doneAt;
  // ---- latency tables ----
  const int16_t* latTab;   // LAT_DIST_DELTA: [1145*100]; LAT_DELTA*: [100]; LAT_DIST: [1145]
  const int16_t* latBase;  // LAT_CITY: [11*11]
  const int16_t* latJit;   // LAT_CITY: [100]
  const unsigned long long* jumpA;  // LCG jump tables: a^(2^i), c(2^i), 48 entries
  const unsigned long long* jumpC;
  // ---- time ring ----
  Ev* buckets;        // [ring][bcap]
  int* bucketCount;   // [ring]
  // ---- per-tick scratch ----
  int* inboxCnt;      // [N]  events addressed to the node this tick
  int* inboxOff;      // [N]
  int* inboxFill;     // [N]
  int* nodeTasks;     // [N] node still has task items to run after the per-thread message pass
  int* dueList;       // [64][listStripeCap] nodes whose conditional task runs this tick
  int* taskList;      // [64][listStripeCap] nodes with task events this tick
  unsigned long long* taskWord;  // [64][listStripeCap] inbox word of the node's only task, ~0 when it has several
  int listStripeCap;
  unsigned long long* inbox;  // [bcap*? ] (key<<32 | entry index)
  int* subCount;      // [bcap] deliveries (+ re-push) of the event at processing position p
  int* itemBase;      // [bcap] exclusive scan of subCount
  int* evSlots;       // [itemCap] descriptors emitted by scan item
  int* evDraws;       // [itemCap] rd.nextInt() draws consumed by scan item
  int* condDue;       // [N] conditional task of node n is examined this tick and its queue is not empty
  uint32_t* workList; // [workCap] global queue-entry index (n*qcap+i) of stale pooled entries, striped
  int* condFired;     // [N], GSF: [2][N]: the half of checkSigs' tick parity (condHalf)
  int* condDraws;     // [N] rd draws consumed by the node's conditional task this tick (Handel: nextInt(k))
  Ev* condEv;         // [N] task created by the conditional task of node n; GSF: [2][N] like condFired
  int* condTarget;    // [N]; GSF: [2][N] like condFired
  int condStride;     // elements between the two halves of condFired / condEv / condTarget (GSF: nLoc; others: 0, one copy)
  int* slotBase;      // [N + itemCap]
  int* drawBase;      // [N + itemCap]
  int* scanPartial;   // [2 * tiles]
  Desc* desc;         // [descCap]
  uint32_t* destScratch;  // [destScratchCap]
  Ev* newEv;          // [newEvCap] in creation order
  int* newTarget;     // [newEvCap]
  int* msCount;       // [msChunks][ring]
  MultiRec* rec;      // [recCap]
  uint32_t* recDest;  // [recDestCap]
  int* recArrival;    // [recDestCap]
  uint32_t* freeList; // [freeCap] level<<27 | slot
  // ---- far-future calendar / fast-forward over empty ticks (protocols without conditional tasks) ----
  int ffwd;       // 1: a tick is the next non-empty millisecond of the window, not the next millisecond
  int farCap;     // 0: arrivals beyond the ring are an error
  FarEv* far;     // [farCap]
  int* farSel;    // [farCap] scratch of the migration pass
  // ---- sendAll ----
  int allCap;     // sendAll descriptors per tick
  int* allList;   // [allCap] descriptor indices
  int* allTmp;    // [allWarps][N] unsorted arrivals of one sendAll
  int allWarps;
  int recSlots;   // sendAll records are recycled round-robin over this many slots of N destinations each
  // ---- shuffled multi-sends (Collections.shuffle inside a handler, SanFerminHelper.java:155) ----
  int shufCap;      // 0: protocol has no k-element shuffles
  int forceShufSerial;  // test hook: always take the serial re-derivation path
  int* byG;         // [newEvCap] descriptor index of creation index g ...
  int* byGTick;     // [newEvCap] ... valid when it equals the tick
  int* descDraw;    // [descCap] corrected draw index of a descriptor (valid when ctl->shufReject)
  // ---- PingPong ----
  int* pong;  // [N]
  // ---- CasperIMD ----
  int cCycle, cBpCount, cAttPerRound, cAttCount, cBlockTime, cAttTime, cRandomTies, cByzDelay;
  int cMaxBlocks, cMaxAtts, cAttWords, cBlkWords, cFirstAtt;
  CasperG* cg;
  uint8_t* cKind;   // [N]
  int* cHead;       // [N] block index of the node's head
  int* cVotes;      // [N] attestations published so far (attesters)
  unsigned long long* cAttRecv;   // [N][cAttWords] attestations received (attestationsByHead, all heads)
  unsigned long long* cBlkRecv;   // [N][cBlkWords] blocksReceivedByBlockId
  unsigned long long* cToReeval;  // [N][cBlkWords] blocksToReevaluate
  int* cbHeight;    // [cMaxBlocks]
  int* cbParent;    // [cMaxBlocks] (-1 for genesis)
  int* cbProducer;  // [cMaxBlocks] node id (-1 for genesis)
  int* cbTime;      // [cMaxBlocks] proposalTime
  unsigned long long* cbIncluded;  // [cMaxBlocks][cAttWords] attestations newly included by the block
  int* attHead;     // [cMaxAtts] block index the attestation votes for
  int* attHeight;   // [cMaxAtts] slot of the vote
  int* cbItem;      // [cMaxBlocks] scan item of the event that created the block (ids follow the processing order)
  unsigned long long* cbTmp;  // [8][cAttWords] scratch of the renumbering pass
  int* cbTmpRow;    // [8][5]
  int* cTieItem;    // [N] randomOnTies: scan item of the event the node is suspended at (-1: not suspended)
  int* cTieCnt;     // [N] ... and the size of its inbox in that pass
  int* cTieList;    // [N] suspended nodes of the pass
  // ---- Handel ----
  int hLevelWait, hFastPath, hExtraCycle, hByzSuicide, hWinInit, hWinMin, hWinMax;
  unsigned long long* hLastAgg;   // [N][W64] lastAggVerified (all levels of a node in one row)
  unsigned long long* hTotInc;    // [N][W64] totalIncoming
  unsigned long long* hVerInd;    // [N][W64] verifiedIndSignatures
  unsigned long long* hToVerInd;  // [N][W64] toVerifyInd
  unsigned long long* hFinPeers;  // [N][W64] finishedPeers
  unsigned long long* hBlack;     // [N][W64] blacklist
  int* hPos;        // [N][L] posInLevel
  int* hOutFin;     // [N][L] outgoingFinished
  int* hBiz;        // [N][L] suicideBizAfter
  int* hBizNoHit;   // [N][L] minimum reception rank over the level's non-blacklisted Byzantine peers (INT_MIN = recompute)
  int* hCntLast;    // [N][L] |lastAggVerified|
  int* hCntInc;     // [N][L] |totalIncoming|
  int* hCntInd;     // [N][L] |verifiedIndSignatures|
  int* hTotal;      // [N] sum of |totalIncoming| over levels
  int* hWindow;     // [N] currWindowSize
  int* hAddedCycle; // [N]
  int* hSigsChecked;   // [N]
  int* hSigQueueSize;  // [N]
  int* hMsgFiltered;   // [N]
  int* hStartAt;    // [N]
  int* hSeq;        // [N] next SigToVerify id
  int* hRanks;      // [N][N] receptionRanks
  HQEntry* hQueue;  // [N][qcap] toVerifyAgg of all levels, arrival order
  int* hCand;       // [N][32] per level: queue index of bestToVerify() or -1
  int* hCandK;      // [N] number of levels with a candidate
  int* hDrawBase;   // [N] exclusive scan of condDraws
  int hHidden;      // params.hiddenByzantine: every honest node carries a HiddenByzantine (Handel.java:303, 840-917)
  int* hbNoPeers;   // [N] HiddenByzantine.noByzantinePeers
  int* hbLastId;    // [N] id of HiddenByzantine.last (-1 = null)
  int* hbLastFrom;  // [N] last.from
  int* poolRef[MAX_LEVELS];  // reference counts of pooled payloads (queue entry + pending update tasks)
  // ---- SanFermin ----
  int sfThreshold, sfPairing, sfSigSize, sfReplyTimeout, sfCandCount, sfP;
  int* sfCpl;        // [N] currentPrefixLength
  int* sfAgg;        // [N] aggValue
  int* sfFlags;      // [N] bit0 isSwapping, bit1 done, bit2 thresholdDone
  long long* sfThresholdAt;  // [N]
  int* sfSentReq;    // [N]
  int* sfRecvReq;    // [N]
  uint32_t* sfCacheMask;  // [N] levels present in signatureCache
  int* sfCache;      // [N][32]
  int sfTimeout;     // SanFerminCappos: params.timeout
  int sfUsedWords;   // words of a row of sfUsedBits
  unsigned long long* sfUsedBits;  // [N][sfUsedWords] SanFerminHelper.usedNodes of the current level
  unsigned long long* sfPendBits;  // [N][sfUsedWords] SanFerminSignature: pendingNodes (positions in the current candidate block)
  // ---- GSF ----
  unsigned long long* verified;   // [N][W64]
  unsigned long long* indivSeen;  // [N][W64]
  unsigned long long* indivVer;   // [N][W64]
  int* pos;        // [N][L]
  int* remaining;  // [N][L]
  int* cntVer;     // [N][L]
  int* cntIndiv;   // [N][L]
  int* cntUnion;   // [N][L]
  int* totalCard;  // [N]
  int* minStart;   // [N]
  uint32_t* stamp; // [N]
  int* pairing;    // [N]
  int* qLen;       // [N]
  int* sigChecked; // [N]
  int* sigQueueSize;  // [N]
  QEntry* queue;   // [N][qcap]
  int* qScore;     // [N][qcap] cached evaluateSig score of the entry ...
  uint32_t* qStamp;  // [N][qcap] ... valid while it equals lvVer of the entry's level (0 = never evaluated)
  uint32_t* lvVer;   // [N][L] bumped whenever the level's verified / individual sets change
  void* peers;     // [N][N-1] uint16 (block-relative) or uint32 (absolute ids)
  unsigned long long* pool[MAX_LEVELS];  // slabs
  uint32_t* poolFree[MAX_LEVELS];        // free stacks
  int poolCap[MAX_LEVELS];
  int forcePickSerial;  // test hook (Handel): always draw the checkSigs picks serially
  int condAhead;        // unsharded GSF: 0 = every pass runs its own checkSigs; 1 = the next pass's runs beside the emission tail
                        // (host build: before the tail; 2: after it)
  int* drawScanPartial;  // [2 * tiles] Handel: tile partials of the draw scan, apart from scanPartial (scan A runs beside it)
  // ---- Slush / Snowflake (wtg_avalanche.cuh) ----
  int sampleK, sampleM, sampleB;  // params.K, M, B (B < 0: Slush)
  double sampleAK;                // params.AK = K * A, compared in double like the reference
  uint8_t* avColor;   // [N] myColor (0 = uncoloured)
  int* avNonce;       // [N] myQueryNonce
  int* avRound;       // [N] Slush: round; Snowflake: cnt
  uint8_t* avPend;    // [N] the Answer of query avNonce is open (at most one query per node is pending)
  uint8_t* avFound;   // [N][2] its colorsFound[1], colorsFound[2]
  // ---- P2PFlood (wtg_p2p.cuh) ----
  int floodMsgs, floodWords;  // params.msgCount, words of a node's bitmap (ceil(msgCount / 64))
  int floodResend, floodBetween;  // FloodMessage.localDelay (delayBeforeResent), delayBetweenPeers (delayBetweenSends)
  const uint32_t* peerOff;    // [N + 1] CSR: the peers of n are peerIds[peerOff[n] .. peerOff[n + 1]), in P2PNode.peers order
  const uint32_t* peerIds;    // [sum of degrees]
  int* floodCnt;              // [N] received(-1).size()
  unsigned long long* floodBits;  // [N][floodWords] which of the originating messages the node has received
  int* peerList;              // [descCap] DESC_PEERS descriptors of the pass (Ctl.peerCnt of them)
};

}  // namespace wtg
