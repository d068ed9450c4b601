// TEST INFRASTRUCTURE.  C++ parity tests through the C++ mirror of the reference classes (include/wtg.hpp, over the C
// ABI) against the CPU oracle (oracle/*.hpp), written like the reference's own JUnit tests:
//   PT/PingPongTest.java:8-19, PT/GSFSignatureTest.java:95-124, PT/CasperByzantineTest.java:12-36, PT/HandelTest.java:36-49.
// Built and run by tests/test_cpp_mirror.py (the run needs a GPU: the product library has no CPU fallback).
#include <cstdio>
#include <cstdlib>

#include "../../include/wtg.hpp"
#include "../../oracle/casper.hpp"
#include "../../oracle/protocols.hpp"

using namespace wtg_b200;

static int g_fail = 0;
#define ASSERT_TRUE(c)                                                   \
  do {                                                                   \
    if (!(c)) {                                                          \
      std::printf("FAIL %s:%d  %s\n", __FILE__, __LINE__, #c);           \
      ++g_fail;                                                          \
      return;                                                            \
    }                                                                    \
  } while (0)
#define ASSERT_EQ(a, b)                                                                                    \
  do {                                                                                                     \
    long long _a = (long long)(a), _b = (long long)(b);                                                    \
    if (_a != _b) {                                                                                        \
      std::printf("FAIL %s:%d  %s == %s  (%lld vs %lld)\n", __FILE__, __LINE__, #a, #b, _a, _b);           \
      ++g_fail;                                                                                            \
      return;                                                                                              \
    }                                                                                                      \
  } while (0)

template <class Nodes>
static bool sameCounters(const NodeCounters& c, const Nodes& nodes) {
  for (size_t i = 0; i < nodes.size(); ++i) {
    const wo::Node& n = *nodes[i];
    if (c.msgReceived[i] != n.msgReceived || c.msgSent[i] != n.msgSent || c.bytesSent[i] != n.bytesSent ||
        c.bytesReceived[i] != n.bytesReceived || c.doneAt[i] != n.doneAt)
      return false;
  }
  return true;
}

// PT/PingPongTest.java: node 0 pings everybody; after the run it has all its pongs.
static void testPingPong() {
  PingPong p(PingPongParameters{1000, "", ""});
  wo::PingPong::Params op;
  op.nodeCt = 1000;
  wo::PingPong o(op);
  p.init();
  o.init();
  for (int i = 0; i < 10; ++i) {
    ASSERT_EQ(p.network().runMs(100), o.network.runMs(100));
    std::vector<int> pong = p.pong();
    for (int n = 0; n < 1000; ++n) ASSERT_EQ(pong[(size_t)n], o.nodes[(size_t)n]->pong);
    ASSERT_TRUE(sameCounters(p.network().counters(), o.nodes));
    ASSERT_EQ(p.network().msgs.size(), o.network.msgs.live);
  }
  ASSERT_EQ(p.pong()[0], 1000);
}

// PT/GSFSignatureTest.java:107-124 (threshold run), here at 256 nodes with AWS regions and Tor, compared with the oracle
// every 10 ms down to the bitmaps.
static void testGSFSignature() {
  const std::string nb = "AWS_SPEED=GAUSSIAN_TOR=0.33", nl = "AwsRegionNetworkLatency";
  GSFSignature p(GSFSignatureParameters{256, 204, 4, 50, 20, 10, 25, nb, nl});
  wo::GSFSignature o(wo::GSFSignature::makeParams(256, 204, 4, 50, 20, 10, 25, nb, nl));
  p.network().rd.setSeed(3);
  o.network.rd.setSeed(3);
  p.init();
  o.init();
  int steps = 0;
  while (p.continueIf()) {
    ASSERT_EQ(p.network().runMs(10), o.network.runMs(10));
    ASSERT_TRUE(++steps < 1000);
    ASSERT_EQ(p.network().rngState(), o.network.rd.seed);
    ASSERT_TRUE(sameCounters(p.network().counters(), o.nodes));
    std::vector<unsigned long long> v = p.verifiedSignatures();
    GSFSignature::Scalars s = p.scalars();
    for (int n = 0; n < 256; ++n) {
      const auto& on = *o.nodes[(size_t)n];
      ASSERT_EQ(s.sigChecked[(size_t)n], on.sigChecked);
      ASSERT_EQ(s.cardinality[(size_t)n], on.verifiedSignatures.cardinality());
      for (int b = 0; b < 256; ++b)
        ASSERT_EQ((v[(size_t)n * 4 + (size_t)(b >> 6)] >> (b & 63)) & 1ULL, on.verifiedSignatures.get(b) ? 1 : 0);
    }
  }
  NodeCounters c = p.network().counters();
  std::vector<unsigned char> down = p.network().down();
  for (int n = 0; n < 256; ++n)
    if (!down[(size_t)n]) ASSERT_TRUE(c.doneAt[(size_t)n] > 0);  // every live node reached the threshold
}

// PT/CasperByzantineTest.java:12-36
static void testCasperByzantineWF() {
  CasperParemeters prm;
  prm.cycleLength = 1;
  prm.randomOnTies = false;
  prm.blockProducersCount = 2;
  prm.attestersPerRound = 2;
  prm.networkLatencyName = "NetworkNoLatency";
  CasperIMD ci(prm);
  ci.init(CasperIMD::ByzBlockProducerWF, 0);
  const int byz = 1, observer = 0;
  ci.network().run(9);
  ASSERT_EQ(ci.heads()[observer], 0);  // genesis
  ci.network().run(1);
  CasperIMD::Blocks b = ci.blocks();
  int h = ci.heads()[observer];
  ASSERT_EQ(b.height[(size_t)h], 1);
  ASSERT_EQ(b.producer[(size_t)h], byz);
  ci.network().run(8);
  b = ci.blocks();
  h = ci.heads()[observer];
  ASSERT_EQ(b.height[(size_t)h], 2);
  ASSERT_TRUE(b.producer[(size_t)h] != byz);
  ci.network().run(8);
  b = ci.blocks();
  h = ci.heads()[observer];
  ASSERT_EQ(b.height[(size_t)h], 3);
  ASSERT_EQ(b.producer[(size_t)h], byz);
}

// CasperIMD with forks (Byzantine producer 9 s late), against the oracle slot by slot
static void testCasperForks() {
  CasperParemeters prm;
  prm.cycleLength = 3;
  prm.randomOnTies = false;
  prm.blockProducersCount = 3;
  prm.attestersPerRound = 20;
  CasperIMD ci(prm);
  ci.network().setTunable("casper_votes", 12);
  wo::CasperIMD o(wo::CasperIMD::makeParams(3, false, 3, 20, 1000, 1, "", "", true));
  ci.init(CasperIMD::ByzBlockProducerWF, 9000);
  o.init(o.newByzWF(9000));
  for (int slot = 0; slot < 25; ++slot) {
    ASSERT_EQ(ci.network().runMs(8000), o.network.runMs(8000));
    std::vector<int> heads = ci.heads();
    for (size_t n = 0; n < heads.size(); ++n)
      ASSERT_EQ(heads[n], static_cast<wo::CasperIMD::CasperNode*>(o.network.allNodes[n])->head->id);
    CasperIMD::Blocks b = ci.blocks();
    ASSERT_EQ(b.height.size(), o.blocks.size() + 1);
    for (size_t i = 0; i < o.blocks.size(); ++i) {
      ASSERT_EQ(b.height[i + 1], o.blocks[i]->height);
      ASSERT_EQ(b.parent[i + 1], o.blocks[i]->parent->id);
      ASSERT_EQ(b.producer[i + 1], o.blocks[i]->producer->nodeId);
    }
  }
}

// PT/HandelTest.java:36-49 parameters: the run terminates and every live node holds the threshold
static void testHandel() {
  const std::string nb = "RANDOM_SPEED=CONSTANT_TOR=0.00", nl = "NetworkLatencyByDistanceWJitter";
  HandelParameters hp{64, 60, 6, 10, 5, 5, 10, 2, nb, nl, 100, false, false};
  Handel p(hp);
  p.init();
  for (int i = 0; i < 300; ++i) p.network().runMs(10);
  NodeCounters c = p.network().counters();
  std::vector<unsigned char> down = p.network().down();
  int live = 0;
  for (int n = 0; n < 64; ++n)
    if (!down[(size_t)n]) {
      ++live;
      ASSERT_TRUE(c.doneAt[(size_t)n] > 0);
    }
  ASSERT_EQ(live, 62);
}

// SanFerminCappos.sigsPerTime scaled down (SanFerminCappos.java:465-471), every 10 ms against the oracle
static void testCappos() {
  SanFerminCappos p(SanFerminCapposParameters{512, 256, 2, 48, 150, 50, "", ""});
  wo::SanFerminCappos::Params op;
  op.nodeCount = 512;
  op.threshold = 256;
  op.candidateCount = 50;
  wo::SanFerminCappos o(op);
  p.init();
  o.init();
  for (int i = 0; i < 400; ++i) {
    ASSERT_EQ(p.network().runMs(10), o.network.runMs(10));
    ASSERT_EQ(p.network().rngState(), o.network.rd.seed);
    ASSERT_TRUE(sameCounters(p.network().counters(), o.nodes));
  }
  NodeCounters c = p.network().counters();
  int done = 0;
  for (int n = 0; n < 512; ++n) done += c.doneAt[(size_t)n] > 0;
  ASSERT_TRUE(done > 500);
}

// CT/StatsTest.java:10-22 and RunMultipleTimes: concurrent seeds give the sequential result
static void testStatsAndRunMultipleTimes() {
  SimpleStats a = avg({SimpleStats{10, 20, 30}, SimpleStats{16, 26, 36}});
  ASSERT_EQ(a.min, 13);
  ASSERT_EQ(a.max, 23);
  ASSERT_EQ(a.avg, 33);
  GSFSignatureParameters prm{128, 100, 3, 20, 10, 10, 8, "RANDOM_SPEED=CONSTANT_TOR=0.00", "NetworkLatencyByDistanceWJitter"};
  RunMultipleTimes<GSFSignature, GSFSignatureParameters> seq{prm, 4, 0, {}}, con{prm, 4, 0, {}};
  auto cont = [](GSFSignature& p) { return p.continueIf(); };
  auto r1 = seq.run(cont, 1);
  auto r2 = con.run(cont, 4);
  ASSERT_EQ(r1.doneAt.avg, r2.doneAt.avg);
  ASSERT_EQ(r1.doneAt.max, r2.doneAt.max);
  ASSERT_EQ(r1.msgReceived.avg, r2.msgReceived.avg);
  for (int i = 0; i < 4; ++i) ASSERT_EQ(seq.endTimes[(size_t)i], con.endTimes[(size_t)i]);
  ASSERT_TRUE(r1.doneAt.min > 0);
}

// error behaviour: the reference's unchecked exceptions surface as WtgError
static void testErrors() {
  bool thrown = false;
  try {
    GSFSignature p(GSFSignatureParameters{100, 90, 3, 20, 10, 10, 0, "", ""});
    p.init();  // not a power of two
  } catch (const WtgError&) {
    thrown = true;
  }
  ASSERT_TRUE(thrown);
  thrown = false;
  try {
    PingPong p(PingPongParameters{10, "", ""});
    p.init();
    p.network().runMs(0);  // Network.java:319-321
  } catch (const WtgError&) {
    thrown = true;
  }
  ASSERT_TRUE(thrown);
}

int main() {
  testPingPong();
  testGSFSignature();
  testCasperByzantineWF();
  testCasperForks();
  testHandel();
  testCappos();
  testStatsAndRunMultipleTimes();
  testErrors();
  if (g_fail) {
    std::printf("MIRROR PARITY FAILED: %d\n", g_fail);
    return 1;
  }
  std::printf("MIRROR PARITY OK\n");
  return 0;
}
