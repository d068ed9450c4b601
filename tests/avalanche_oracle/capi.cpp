// TEST INFRASTRUCTURE ONLY — C interface (ctypes) over the CPU restatement of Slush / Snowflake (avalanche.hpp).
// Loaded by tests/avalanche_oracle_lib.py; the product package never loads it.
#include <chrono>
#include <cstring>
#include <string>

#include "avalanche.hpp"

using namespace wo;

static thread_local std::string g_err;

namespace {
// one handle type for both protocols: kind 0 Slush, 1 Snowflake
struct Handle {
  std::unique_ptr<Slush> slush;
  std::unique_ptr<Snowflake> snow;
  Network& net() { return slush ? slush->network : snow->network; }
};
template <class F>
int guarded(F f) {
  try {
    return f();
  } catch (const std::exception& e) {
    g_err = e.what();
    return -1;
  }
}
template <class P, class F>
void eachNode(P& p, F f) {
  for (size_t i = 0; i < p.nodes.size(); ++i) {
    auto& n = *p.nodes[i];
    int f1 = 0, f2 = 0;
    bool pending = !n.answerIP.empty();
    if (pending) {
      auto it = n.answerIP.find(n.myQueryNonce);
      if (it != n.answerIP.end()) {
        f1 = it->second.colorsFound[1];
        f2 = it->second.colorsFound[2];
      }
    }
    f(i, n, pending, f1, f2, (int)n.answerIP.size());
  }
}
}  // namespace

extern "C" {

const char* wav_last_error() { return g_err.c_str(); }

// B < 0: Slush
void* wav_create(int nodes, int M, int K, double A, int B, const char* nodeBuilderName, const char* networkLatencyName) {
  try {
    auto* h = new Handle();
    if (B < 0) {
      Slush::Params p;
      p.NODES_AV = nodes;
      p.M = M;
      p.K = K;
      p.A = A;
      p.nodeBuilderName = nodeBuilderName ? nodeBuilderName : "";
      p.latencyNull = networkLatencyName == nullptr;
      p.networkLatencyName = networkLatencyName ? networkLatencyName : "";
      h->slush = std::make_unique<Slush>(p);
    } else {
      Snowflake::Params p;
      p.NODES_AV = nodes;
      p.M = M;
      p.K = K;
      p.A = A;
      p.B = B;
      p.nodeBuilderName = nodeBuilderName ? nodeBuilderName : "";
      p.latencyNull = networkLatencyName == nullptr;
      p.networkLatencyName = networkLatencyName ? networkLatencyName : "";
      h->snow = std::make_unique<Snowflake>(p);
    }
    return h;
  } catch (const std::exception& e) {
    g_err = e.what();
    return nullptr;
  }
}
void wav_destroy(void* h) { delete static_cast<Handle*>(h); }
void wav_set_seed(void* h, int64_t s) { static_cast<Handle*>(h)->net().rd.setSeed(s); }
int wav_init(void* h) {
  return guarded([&] {
    auto* x = static_cast<Handle*>(h);
    if (x->slush)
      x->slush->init();
    else
      x->snow->init();
    return 0;
  });
}
int wav_run_ms(void* h, int ms) {
  return guarded([&] { return static_cast<Handle*>(h)->net().runMs(ms) ? 1 : 0; });
}
// runMs(ms) timed on the host clock, in milliseconds (-1 on failure)
double wav_run_timed(void* h, int ms) {
  auto t0 = std::chrono::steady_clock::now();
  if (wav_run_ms(h, ms) < 0) return -1.0;
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}
int wav_time(void* h) { return static_cast<Handle*>(h)->net().time; }
int wav_msgs_size(void* h) { return static_cast<Handle*>(h)->net().msgs.size(); }
int64_t wav_msgs_live(void* h) { return static_cast<Handle*>(h)->net().msgs.live; }
uint64_t wav_rng_state(void* h) { return static_cast<Handle*>(h)->net().rd.seed; }
int64_t wav_deliveries(void* h) { return static_cast<Handle*>(h)->net().statDeliveries; }
void wav_node_counters(void* h, int64_t* out5N) {
  const std::vector<Node*>& nodes = static_cast<Handle*>(h)->net().allNodes;
  size_t n = nodes.size();
  for (size_t i = 0; i < n; ++i) {
    out5N[0 * n + i] = nodes[i]->msgReceived;
    out5N[1 * n + i] = nodes[i]->msgSent;
    out5N[2 * n + i] = nodes[i]->bytesSent;
    out5N[3 * n + i] = nodes[i]->bytesReceived;
    out5N[4 * n + i] = nodes[i]->doneAt;
  }
}
// per node: myColor, myQueryNonce, round / cnt, pending (answerIP not empty), colorsFound[1], colorsFound[2] of the pending
// Answer; returns the largest answerIP.size() seen (at most one query per node is ever pending)
int wav_node_scalars(void* h, int32_t* color, int32_t* nonce, int32_t* roundOrCnt, int32_t* pending, int32_t* f1, int32_t* f2) {
  auto* x = static_cast<Handle*>(h);
  int maxOpen = 0;
  auto put = [&](size_t i, auto& n, bool pend, int a, int b, int open) {
    color[i] = n.myColor;
    nonce[i] = n.myQueryNonce;
    pending[i] = pend ? 1 : 0;
    f1[i] = a;
    f2[i] = b;
    maxOpen = std::max(maxOpen, open);
  };
  if (x->slush)
    eachNode(*x->slush, [&](size_t i, Slush::SlushNode& n, bool pend, int a, int b, int open) {
      put(i, n, pend, a, b, open);
      roundOrCnt[i] = n.round;
    });
  else
    eachNode(*x->snow, [&](size_t i, Snowflake::SnowflakeNode& n, bool pend, int a, int b, int open) {
      put(i, n, pend, a, b, open);
      roundOrCnt[i] = n.cnt;
    });
  return maxOpen;
}
// op: 0 stop(arg), 1 start(arg), 2 partition(arg / 10000.f), 3 endPartition
int wav_net_ctl(void* h, int op, int arg) {
  return guarded([&] {
    Network& net = static_cast<Handle*>(h)->net();
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
