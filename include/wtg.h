/* wittgenstein_b200 — C ABI of the H100-native simulation engine.
 *
 * The reference (ConsenSys/wittgenstein, Java) has no FFI of its own: the seam is the Java API
 * `Protocol { network(); copy(); init(); }` (core/Protocol.java:7-22) and the public members of
 * `core.Network`.  Each entry point below names the reference member it stands in for; a JNI
 * (or ctypes) binding maps them 1:1 — see INTEGRATION.md.  All paths are relative to
 * core/src/main/java/net/consensys/wittgenstein/core/ unless they start with protocols/.
 *
 * Conventions (SURVEY.md §8b):
 *   - single caller thread per network, like the reference (Network.java:10);
 *   - functions returning int return >= 0 on success and -1 on failure; the message of the
 *     IllegalArgumentException / IllegalStateException the reference would have thrown is then
 *     available from wtg_last_error() (thread-local);
 *   - the engine owns all node/message state (device memory); read-back functions copy out;
 *   - same seed => identical results, bit for bit, as the reference engine.
 *   - there is no CPU fallback: wtg_create() fails when no CUDA device is present.
 */
#ifndef WTG_H
#define WTG_H

#ifdef __cplusplus
extern "C" {
#endif

typedef void wtg_net; /* opaque: one core.Network + the protocol state living on it */

const char* wtg_last_error(void);

/* new Network<>()  — Network.java:13-49: rd = new Random(0), time = 0, IC3NetworkLatency */
wtg_net* wtg_create(void);
/* the same on CUDA device `device` (default: LOCAL_RANK / WTG_DEVICE / 0).  Independent networks — e.g. the seeds of a
 * RunMultipleTimes sweep — can live on different GPUs of one process, one caller thread per network. */
wtg_net* wtg_create_on(int device);
void wtg_destroy(wtg_net* net);

/* ---- node-sharded simulation (SURVEY.md §8e; the reference has no counterpart: core/Network.java is one thread) ----
 * ONE network spread over `world` engines (a power of two <= 8, one GPU each): shard `rank` owns the node ids
 * [rank * N / world, (rank + 1) * N / world).  Every shard is configured and initialised with IDENTICAL calls (seed,
 * builder, latency, protocol parameters) from its own thread (all shards in one process: the JNI case) or its own
 * process (one rank per GPU); after the protocol's init each shard exports the 128-byte handle of its exchange region,
 * all handles are handed to wtg_shard_link of every shard (same-process shards are mapped directly with peer access,
 * other processes through CUDA IPC), and from then on every shard calls wtg_run_ms with the same arguments.  The data
 * path between shards is device-to-device stores inside the tick kernels (no host call, no collective per tick).
 * Node-indexed read-backs of a shard (counters, GSF / Handel rows and scalars, CasperIMD node state) cover its own ids
 * only: wtg_shard_range.  Available for GSFSignature, Handel and CasperIMD; the other protocols refuse to initialise on a
 * sharded network.  Latency models with multi-second arrivals (no far-future calendar for messages on sharded networks)
 * and caller-issued sends (wtg_send*) are refused there too. */
wtg_net* wtg_shard_create(int rank, int world, int device /* -1: default */);
int wtg_shard_export(wtg_net* net, unsigned char* handle128);
int wtg_shard_link(wtg_net* net, const unsigned char* handles /* world x 128 bytes, rank order */);
int wtg_shard_range(wtg_net* net, int* first_id, int* count);
/* CUDA device the network lives on */
int wtg_device(wtg_net* net);

/* network.rd.setSeed(seed) before Protocol.init() — RunMultipleTimes.java:47, ProgressPerTime.java:71 */
int wtg_set_seed(wtg_net* net, long long seed);

/* network.setNetworkLatency(RegistryNetworkLatencies.singleton.getByName(name)) —
 * Network.java:669-677, RegistryNetworkLatencies.java:28-58.  name == NULL selects
 * NetworkLatencyByDistanceWJitter like the registry does.  Supported: NetworkLatencyByDistanceWJitter,
 * AwsRegionNetworkLatency, NetworkNoLatency, EthScanNetworkLatency, IC3NetworkLatency,
 * "NetworkFixedLatency(f)" / "NetworkUniformLatency(f)" for the registry's f values. */
int wtg_set_network_latency(wtg_net* net, const char* name);
/* network.setNetworkLatency(int[] distribProp, int[] distribVal) — Network.java:665-667 */
int wtg_set_network_latency_measured(wtg_net* net, const int* proportions, const int* values, int n);

/* nb = RegistryNodeBuilders.singleton.getByName(name) — RegistryNodeBuilders.java:71-81
 * ("<AWS|RANDOM>_SPEED=<CONSTANT|GAUSSIAN>_TOR=<d.dd>"; NULL/blank = RANDOM, constant speed, no Tor) */
int wtg_set_node_builder(wtg_net* net, const char* name);

/* network.setMsgDiscardTime(ms) — Network.java:103-106 */
int wtg_set_msg_discard_time(wtg_net* net, int ms);

/* device capacities (no reference counterpart): "bcap", "qcap", "pool_slots_per_node", "desc_cap",
 * "rec_cap", "ring", "casper_votes", "casper_blocks", "stage_words" (node-sharded GSF / Handel: staging area for pooled payloads that
 * cross shards, 64-bit words per sending shard and pass parity); test hooks "force_shuffle_serial" (SanFermin family, Slush,
 * Snowflake: the serial re-derivation of draw indices) and "force_pick_serial" (Handel: checkSigs' level draws walked serially, locally and across shards).  Exceeding a capacity makes wtg_run_ms fail loudly; it never drops events. */
int wtg_set_tunable(wtg_net* net, const char* key, long long value);

/* new PingPong(params).init() — protocols/PingPong.java:52-57, 82-87 */
int wtg_pingpong_init(wtg_net* net, int node_ct);

/* new GSFSignature(params).init() — protocols/GSFSignature.java:59-84, 611-635.
 * params7 = { nodeCount, threshold, pairingTime, timeoutPerLevelMs, periodDurationMs,
 *             acceleratedCallsCount, nodesDown }  (the fields of GSFSignatureParameters) */
int wtg_gsf_init(wtg_net* net, const int* params7);

/* new SanFerminSignature(params) — protocols/SanFerminSignature.java:112-129 (the constructor builds the nodes on
 * network.rd, so a later wtg_set_seed does not change them) and .init() — :136-138.
 * params6 = { nodeCount, threshold, pairingTime, signatureSize, replyTimeout, candidateCount } (:41-110;
 * shuffledLists / verbose are unused by the reference).  Device engine: power-of-two nodeCount, candidateCount <= 63. */
int wtg_sanfermin_construct(wtg_net* net, const int* params6);
int wtg_sanfermin_init(wtg_net* net);

/* new SanFerminCappos(params).init() — protocols/SanFerminCappos.java:106-134.
 * params6 = { nodeCount, threshold, pairingTime, signatureSize, timeout, candidateCount } (SanFerminParameters :86-103).
 * Device engine: power-of-two nodeCount, candidateCount <= 63. */
int wtg_cappos_init(wtg_net* net, const int* params6);

/* new Slush(new SlushParameters(nodes, M, K, A, ...)).init() — protocols/Slush.java:36-74, and
 * new Snowflake(new SnowflakeParameters(nodes, M, K, A, B, ...)).init() — protocols/Snowflake.java:38-88.
 * AK = K * A is compared in double (onAnswer, Slush.java:161-176, Snowflake.java:170-188).  The sample of every query
 * (randomRemotes, Slush.java:126-137, Snowflake.java:136-147) is drawn from network.rd at its exact position in the draw
 * order.  1 <= K <= min(63, nodes - 1): with K >= nodes the reference never returns, with K = 0 it sends nothing.
 * Not available on a node-sharded network. */
int wtg_slush_init(wtg_net* net, int nodes, int M, int K, double A);
int wtg_snowflake_init(wtg_net* net, int nodes, int M, int K, double A, int B);

/* new Handel(params).init() — protocols/Handel.java:96-141, 957-1014.
 * params11 = { nodeCount, threshold, pairingTime, levelWaitTime, extraCycle, disseminationPeriodMs, fastPath, nodesDown,
 *              desynchronizedStart, byzantineSuicide, hiddenByzantine } (HandelParameters; window = WindowParameters()).
 * HiddenByzantine (:840-917) is supported; badNodes is always drawn with Network.chooseBadNodes. */
int wtg_handel_init(wtg_net* net, const int* params11);

/* new CasperIMD(params) — protocols/CasperIMD.java:81-88 (the constructor builds the observer node on network.rd) and
 * .init(new ByzBlockProducerWF(byz_delay, genesis)) — :472-508 (init() itself uses byz_delay 0).
 * params6 = { cycleLength, randomOnTies, blockProducersCount, attestersPerRound, blockConstructionTime,
 *             attestationConstructionTime } (CasperParemeters :18-71).  Node ids: 0 observer, 1 the Byzantine producer,
 * 2.. the other producers, then the attesters.  randomOnTies: a vote tie between two branches draws network.rd.nextBoolean()
 * inside the handler (:250-253) at its exact position in the draw order (the node is suspended in the parallel pass and run
 * by a tie pass in processing order); blocks created in the same millisecond get their ids in processing order.  Both are
 * reported as errors on a node-sharded network only. */
int wtg_casper_construct(wtg_net* net, const int* params6);
int wtg_casper_init(wtg_net* net, int byz_delay);
/* .init(new ByzBlockProducer / SF / NS / WF (byz_delay, genesis)) — kind 3 / 4 / 5 / 6 (CasperIMD.java:511-707) */
int wtg_casper_init_byz(wtg_net* net, int kind, int byz_delay);

/* network.send(msg, from, to) / send(msg, from, dests) / sendAll(msg, from) called by the host between two runMs windows —
 * Network.java:341-366: one rd.nextInt() per call, send time = time + 1.  `type` / `payload` name a message of the running
 * protocol: PingPong 1 = Ping, 2 = Pong (payload unused); CasperIMD 2 = SendBlock(block id).  Any number of
 * destinations per wtg_send; wtg_send_all needs the sendAll path (CasperIMD).  Other protocols' messages carry device-resident payloads and are
 * not offered. */
int wtg_send(wtg_net* net, int type, unsigned long long payload, int from, const int* to, int n);
int wtg_send_all(wtg_net* net, int type, unsigned long long payload, int from);
/* network.send(msg, sendTime, from, to) and send(msg, sendTime, from, dests, delaysBetweenMessage) — Network.java:369-382, 420-447:
 * explicit send time (> time) and, for several destinations, `delay_between` ms between the sends (MultipleDestWithDelayEnvelope) */
int wtg_send_at(wtg_net* net, int type, unsigned long long payload, int from, const int* to, int n, int send_time, int delay_between);

/* network.runMs(ms) — Network.java:318-338.  Returns 1/0 like the reference's boolean. */
int wtg_run_ms(wtg_net* net, int ms);
/* network.time — Network.java:49 */
int wtg_time(wtg_net* net);
/* network.allNodes.size() — Network.java:29 */
int wtg_node_count(wtg_net* net);
/* network.msgs.size() / network.msgs.sizeAt(t) — Network.java:204-220 */
int wtg_msgs_size(wtg_net* net);
int wtg_msgs_size_at(wtg_net* net, int t);
/* network.msgs.peekMessages() — Network.java:279-286 (EnvelopeInfo.java:8-14; the call behind the REST façade's
 * GET /w/network/messages, wserver/.../ws/WServer.java:71-75): one row per pending arrival — every remaining destination of a
 * multi-destination envelope is a row — sorted by arrival time.  from/to: node ids; sent_at: Envelope.sendTime (-1 when the
 * engine did not record it: tasks registered by init()); kind: 0 message, 2 Task, 3 PeriodicTask; msg_type: the protocol's
 * message type code (GSF/Handel: payload kind and level).  Returns the number of pending arrivals; at most `cap` rows are
 * written (any output pointer may be NULL).  On a node-sharded network every pending
 * arrival is reported by exactly one shard (single-destination envelopes by the destination's shard). */
int wtg_peek_messages(wtg_net* net, int* from, int* to, int* sent_at, int* arriving_at, int* kind, int* msg_type, int cap);

/* node.stop() / node.start() — Node.java:120-127 */
int wtg_stop_node(wtg_net* net, int node_id);
int wtg_start_node(wtg_net* net, int node_id);
/* network.partition(part) / network.endPartition() — Network.java:693-707.  For CasperIMD endPartition is
 * BlockChainNetwork.endPartition (BlockChainNetwork.java:46-54): every node re-sends its head to all (needs rec_cap >= nodes + 64). */
int wtg_partition(wtg_net* net, float part);
int wtg_end_partition(wtg_net* net);

/* the 48-bit state of network.rd (for parity checks of the consumed stream position) */
unsigned long long wtg_rng_state(wtg_net* net);

/* Node.msgReceived / msgSent / bytesSent / bytesReceived / doneAt — Node.java:72-79.
 * out5N = 5 arrays of N int64, in that order. */
int wtg_node_counters(wtg_net* net, long long* out5N);
/* Node.x / y / extraLatency / city (AWS region index, -1 otherwise) / speedRatio / isDown() — Node.java:36-69.
 * Any pointer may be NULL. */
int wtg_node_attrs(wtg_net* net, int* x, int* y, int* extra, int* city, double* speed, unsigned char* down);

/* PingPongNode.pong — protocols/PingPong.java:61 */
int wtg_pingpong_pongs(wtg_net* net, int* out);

/* SanFerminNode.aggValue, currentPrefixLength, done, thresholdDone, sentRequests, receivedRequests, isSwapping,
 * thresholdAt — protocols/SanFerminSignature.java:157-208 */
int wtg_sanfermin_node_scalars(wtg_net* net, int* agg, int* cpl, int* done, int* thr_done, int* sent_req, int* recv_req,
                               int* swapping, long long* threshold_at);

/* CasperIMD read-backs.  Blocks are numbered in creation order (Block.id, core/Block.java:10,49; genesis = 0).
 * wtg_casper_blocks: per block height, parent id (-1), producer node id (-1), proposalTime, number of attestations it
 * includes (CasperBlock.attestationsByHeight, CasperIMD.java:152); returns the block count.
 * wtg_casper_block_attestations: those attestations as (attester node id, attestation height); returns their number.
 * wtg_casper_node_state: per node head id (BlockChainNode.head), attestations received and distinct heads among them
 * (attestationsByHead, CasperIMD.java:197), blocks received incl. genesis (blocksReceivedByBlockId), |blocksToReevaluate|,
 * and an order-free 64-bit hash over (attester, height, head id) of the received attestations.
 * wtg_casper_byz: { toSend, h, late, onTime, delay, onDirectFather, onOlderAncestor, incNotTheBestFather, skipped } of the
 * Byzantine producer (:512-518, 615, 648-649). */
int wtg_casper_block_count(wtg_net* net);
int wtg_casper_blocks(wtg_net* net, int* height, int* parent, int* producer, int* proposal_time, int* included);
int wtg_casper_block_attestations(wtg_net* net, int block, int* attester, int* height, int cap);
int wtg_casper_node_state(wtg_net* net, int* head, int* atts_received, int* heads_with_atts, int* blocks_received,
                          int* to_reevaluate, unsigned long long* att_hash);
int wtg_casper_heads(wtg_net* net, int* head); /* BlockChainNode.head of every node (block id) */
int wtg_casper_byz(wtg_net* net, int* out9);

/* SanFerminCappos.SanFerminNode: currentPrefixLength, totalNumberOfSigs(-1), done, thresholdDone, isSwapping, the levels
 * present in signatureCache (bit mask), thresholdAt — protocols/SanFerminCappos.java:155-180, 351-358 */
int wtg_cappos_node_scalars(wtg_net* net, int* cpl, int* sigs, int* done, int* thr_done, int* swapping, int* cache_mask,
                            long long* threshold_at);
/* java.util.Collections.shuffle(list, rnd) with rnd in 48-bit state `state` (JDK: for i = size; i > 1; i-- swap(i-1,
 * rnd.nextInt(i))); runs on the host the code the emit kernel uses; returns the number of values drawn from the stream */
int wtg_java_shuffle(unsigned long long state, int n, int* inout);

/* SlushNode / SnowflakeNode: myColor, myQueryNonce, round (Slush) or cnt (Snowflake), whether answerIP holds the Answer of
 * the last query, and that Answer's colorsFound[1] / colorsFound[2] (0 when none is pending) — protocols/Slush.java:117-120,
 * 217-231; protocols/Snowflake.java:127-130, 217-232 (Answer.round is never read by the reference and is not kept) */
int wtg_avalanche_node_scalars(wtg_net* net, int* color, int* nonce, int* round_or_cnt, int* pending, int* found1, int* found2);
/* pipeline passes whose rd draw indices were re-derived serially because a shuffle's nextInt rejected a value or a sample
 * (randomRemotes) discarded an attempt (no reference counterpart; -1 on failure) */
long long wtg_serial_passes(wtg_net* net);

/* new P2PFlood(new P2PFloodParameters(nodeCount, deadNodeCount, delayBeforeResent, msgCount, msgToReceive, peersCount,
 * delayBetweenSends, ...)).init() — protocols/P2PFlood.java:146-165 on core/P2PNetwork.java (setPeers, minimum = true) and
 * core/messages/FloodMessage.java (msgToReceive is never read by the protocol).  Refused: negative arguments,
 * peersCount >= nodeCount (the reference throws), msgCount above the live nodes (the reference never returns),
 * delayBetweenSends >= 2^20, a peer graph with a degree above 256, record arenas beyond 2^31 entries, a node-sharded network. */
int wtg_p2pflood_init(wtg_net* net, int nodeCount, int deadNodeCount, int delayBeforeResent, int msgCount, int peersCount,
                      int delayBetweenSends);
/* P2PNode.peers of `node` in the reference's order (link creation): its size; wtg_p2p_peers writes up to cap ids */
int wtg_p2p_peer_count(wtg_net* net, int node);
int wtg_p2p_peers(wtg_net* net, int node, int* out, int cap);
/* P2PNetwork.avgPeers() (P2PNetwork.java:115-125) */
int wtg_p2p_avg_peers(wtg_net* net);
/* getMsgReceived(-1).size() of every node into count[N]; with bits != NULL also which originating messages (init's draw
 * order) `node` holds, ceil(msgCount / 64) words (at least one).  Returns the number of words. */
int wtg_p2pflood_received(wtg_net* net, int* count, int node, unsigned long long* bits);

/* Handel read-backs on a node-sharded network: node_scalars, rows and level_scalars cover the shard's own ids (nLoc in place of
 * N); peers and ranks fail with "node belongs to another shard" for a node of another shard. */
/* HNode fields — protocols/Handel.java:280-298: 9 int arrays of N: startAt, nodePairingTime, sigsChecked, sigQueueSize,
 * msgFiltered, currWindowSize, addedCycle, totalSigSize(), total length of the toVerifyAgg lists */
int wtg_handel_node_scalars(wtg_net* net, int* out9N);
/* HLevel bitsets as unions over levels, N rows of N/64 uint64 — :373-394; which: 0 totalIncoming, 1 lastAggVerified,
 * 2 verifiedIndSignatures, 3 toVerifyInd, 4 finishedPeers, 5 HNode.blacklist (:287) */
int wtg_handel_rows(wtg_net* net, int which, unsigned long long* outNW);
/* HLevel.posInLevel, outgoingFinished, suicideBizAfter as N*L arrays — :397-406 */
int wtg_handel_level_scalars(wtg_net* net, int* pos, int* outgoing_finished, int* suicide_biz_after);
/* HLevel.peers (emission order) — :370 ; HNode.receptionRanks — :285 ; HNode.levels.size() */
int wtg_handel_peers(wtg_net* net, int node, int level, int* out, int cap);
int wtg_handel_ranks(wtg_net* net, int node, int* outN);
int wtg_handel_levels(wtg_net* net);

/* GSFNode.levels.size() — protocols/GSFSignature.java:168 */
int wtg_gsf_levels(wtg_net* net);
/* GSFNode.verifiedSignatures of every node as N rows of N/64 uint64 (bit i = word i/64, bit i%64) — :169 */
int wtg_gsf_verified(wtg_net* net, unsigned long long* outNW);
/* which: 0 verifiedSignatures, 1 union over levels of SFLevel.individualSignatures, 2 of SFLevel.indivVerifiedSig — :242-244 */
int wtg_gsf_rows(wtg_net* net, int which, unsigned long long* outNW);
/* nodePairingTime, sigChecked, sigQueueSize, toVerify.size(), verifiedSignatures.cardinality() — :167-174 */
int wtg_gsf_node_scalars(wtg_net* net, int* pairing, int* sig_checked, int* sig_queue_size, int* to_verify_size, int* card);
/* SFLevel.posInLevel, remainingCalls, verifiedSignatures.cardinality() as N*L arrays — :251-254 */
int wtg_gsf_level_scalars(wtg_net* net, int* pos, int* remaining, int* card);
/* SFLevel.peers of one node / level — :239 ; returns the list length */
int wtg_gsf_peers(wtg_net* net, int node, int level, int* out, int cap);

/* engine statistics (26 int64), see wittgenstein_b200/network.py:Network.stats for the keys */
int wtg_stats(wtg_net* net, long long* out26);

/* measurement hooks (no reference counterpart): a CUDA-event stopwatch on the engine's stream, and
 * per-kernel event timing of the tick pipeline (names[i] are static strings; on = 2 reports the delivery dispatch's
 * scan A under names of its own instead of adding it into scan B's) */
int wtg_timer_start(wtg_net* net);
double wtg_timer_stop_ms(wtg_net* net);
int wtg_profile_enable(wtg_net* net, int on);
int wtg_profile_read(wtg_net* net, double* ms, long long* launches, const char** names, int cap);

#ifdef __cplusplus
}
#endif
#endif /* WTG_H */
