// TEST INFRASTRUCTURE ONLY — C interface (ctypes) over the CPU restatement of P2PFlood (p2pflood.hpp).
// Loaded by tests/p2p_oracle_lib.py; the product package never loads it.
#include <chrono>
#include <cstring>
#include <string>
#include <unordered_map>

#include "p2pflood.hpp"

using namespace wo;

static thread_local std::string g_err;

namespace {
template <class F>
int guarded(F f) {
  try {
    return f();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}
P2PFlood& P(void* h) { return *static_cast<P2PFlood*>(h); }
}  // namespace

extern "C" {

const char* wpf_last_error() { return g_err.c_str(); }

void* wpf_create(int nodeCount, int deadNodeCount, int delayBeforeResent, int msgCount, int msgToReceive, int peersCount,
                 int delayBetweenSends, const char* nodeBuilderName, const char* networkLatencyName) {
  try {
    P2PFlood::Params p;
    p.nodeCount = nodeCount;
    p.deadNodeCount = deadNodeCount;
    p.delayBeforeResent = delayBeforeResent;
    p.msgCount = msgCount;
    p.msgToReceive = msgToReceive;
    p.peersCount = peersCount;
    p.delayBetweenSends = delayBetweenSends;
    p.nodeBuilderName = nodeBuilderName ? nodeBuilderName : "";
    p.latencyNull = networkLatencyName == nullptr;
    p.networkLatencyName = networkLatencyName ? networkLatencyName : "";
    return new P2PFlood(p);
  } catch (const std::exception& e) {
    g_err = e.what();
    return nullptr;
  }
}
void wpf_destroy(void* h) { delete static_cast<P2PFlood*>(h); }
void wpf_set_seed(void* h, int64_t s) { P(h).network.rd.setSeed(s); }
int wpf_init(void* h) {
  return guarded([&] {
    P(h).init();
    return 0;
  });
}
int wpf_run_ms(void* h, int ms) {
  return guarded([&] { return P(h).network.runMs(ms) ? 1 : 0; });
}
// runMs(ms) timed on the host clock, in milliseconds (-1 on failure)
double wpf_run_timed(void* h, int ms) {
  auto t0 = std::chrono::steady_clock::now();
  if (wpf_run_ms(h, ms) < 0) return -1.0;
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}
int wpf_time(void* h) { return P(h).network.time; }
int wpf_msgs_size(void* h) { return P(h).network.msgs.size(); }
uint64_t wpf_rng_state(void* h) { return P(h).network.rd.seed; }
int64_t wpf_deliveries(void* h) { return P(h).network.statDeliveries; }
void wpf_node_counters(void* h, int64_t* out5N) {
  const std::vector<Node*>& nodes = P(h).network.allNodes;
  size_t n = nodes.size();
  for (size_t i = 0; i < n; ++i) {
    out5N[0 * n + i] = nodes[i]->msgReceived;
    out5N[1 * n + i] = nodes[i]->msgSent;
    out5N[2 * n + i] = nodes[i]->bytesSent;
    out5N[3 * n + i] = nodes[i]->bytesReceived;
    out5N[4 * n + i] = nodes[i]->doneAt;
  }
}
// per node: getMsgReceived(-1).size() and isDown(); bits[N][words]: which originating messages (init's draw order) it holds
void wpf_received(void* h, int32_t* count, uint8_t* down, uint64_t* bits, int words) {
  P2PFlood& p = P(h);
  std::unordered_map<const FloodMessage*, int> idx;
  for (size_t i = 0; i < p.msgs.size(); ++i) idx[p.msgs[i].get()] = static_cast<int>(i);
  for (size_t i = 0; i < p.nodes.size(); ++i) {
    const auto& n = *p.nodes[i];
    count[i] = static_cast<int32_t>(n.received.size());
    down[i] = n.isDown() ? 1 : 0;
    if (!bits) continue;
    uint64_t* row = bits + i * static_cast<size_t>(words);
    for (int w = 0; w < words; ++w) row[w] = 0;
    for (const FloodMessage* m : n.received) {
      int k = idx.at(m);
      row[k >> 6] |= 1ULL << (k & 63);
    }
  }
}
int wpf_peer_count(void* h, int node) { return static_cast<int>(P(h).nodes.at(static_cast<size_t>(node))->peers.size()); }
void wpf_peers(void* h, int node, int32_t* out) {
  const auto& pe = P(h).nodes.at(static_cast<size_t>(node))->peers;
  for (size_t i = 0; i < pe.size(); ++i) out[i] = pe[i]->nodeId;
}
int wpf_avg_peers(void* h) { return P(h).network.avgPeers(); }
int wpf_node_xy(void* h, int32_t* x, int32_t* y) {
  for (size_t i = 0; i < P(h).nodes.size(); ++i) {
    x[i] = P(h).nodes[i]->x;
    y[i] = P(h).nodes[i]->y;
  }
  return 0;
}
// network.msgs.peekMessages() rows (from, to, sentAt, arrivingAt), sorted like the engine's read-back; returns the total
int wpf_peek_messages(void* h, int32_t* from, int32_t* to, int32_t* sentAt, int32_t* arrivingAt, int cap) {
  std::vector<EnvelopeInfo> rows = P(h).network.msgs.peekMessages();
  for (size_t i = 0; i < rows.size() && static_cast<int>(i) < cap; ++i) {
    from[i] = rows[i].from;
    to[i] = rows[i].to;
    sentAt[i] = rows[i].sentAt;
    arrivingAt[i] = rows[i].arrivingAt;
  }
  return static_cast<int>(rows.size());
}
// op: 0 stop(arg), 1 start(arg), 2 partition(arg / 10000.f), 3 endPartition
int wpf_net_ctl(void* h, int op, int arg) {
  return guarded([&] {
    Network& net = P(h).network;
    switch (op) {
      case 0: net.getNodeById(arg).stop(); break;
      case 1: net.getNodeById(arg).start(); break;
      case 2: net.partition(static_cast<float>(arg) / 10000.f); break;
      case 3: net.endPartition(); break;
      default: throw IllegalArgument("op");
    }
    return 0;
  });
}

}  // extern "C"
