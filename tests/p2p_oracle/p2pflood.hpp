// TEST INFRASTRUCTURE ONLY — CPU restatement of core/P2PNetwork.java, core/P2PNode.java, core/messages/FloodMessage.java and
// protocols/P2PFlood.java on the oracle's core (oracle/core.hpp: Network, Node, Message, java.util.Random), line by line.
// Line references are to those files.
#pragma once
#include <algorithm>
#include <memory>
#include <string>
#include <unordered_set>
#include <vector>

#include "../../oracle/core.hpp"

namespace wo {

struct FloodMessage;

// P2PNode :8-28
struct P2PNode : Node {
  std::vector<P2PNode*> peers;                          // :11
  std::unordered_set<const FloodMessage*> received;     // received.get(-1) (:13-17): FloodMessage.msgId() is always -1
  P2PNode(JavaRandom& rd, NodeBuilder& nb) : Node(rd, nb) {}
  virtual void onFlood(P2PNode& /*from*/, const FloodMessage& /*m*/) {}  // :27
};

// FloodMessage :15-61
struct FloodMessage : Message, std::enable_shared_from_this<FloodMessage> {
  int size_, localDelay, delayBetweenPeers;
  FloodMessage(int size, int ld, int dbp) : size_(size), localDelay(ld), delayBetweenPeers(dbp) {}
  bool addToReceived(P2PNode& to) const { return to.received.insert(this).second; }  // :43-45
  void action(Network& network, Node& from, Node& to) override;                       // :47-55
  int size() const override { return size_; }
};

// P2PNetwork :11-133 (minimum = true: the only mode P2PFlood uses)
struct P2PNetwork : Network {
  int connectionCount;
  std::unordered_set<int64_t> existingLinks;
  explicit P2PNetwork(int cc) : connectionCount(cc) {}
  P2PNode& peer(int id) { return static_cast<P2PNode&>(getNodeById(id)); }

  void setPeers() {  // :26-55
    if (connectionCount >= static_cast<int>(allNodes.size()))
      throw IllegalArgument("Wrong configuration: #nodes=" + std::to_string(allNodes.size()) + ", connection target=" +
                            std::to_string(connectionCount));
    std::vector<Node*> an(allNodes);
    javaShuffle(an, rd);
    for (Node* n : an) {
      while (static_cast<int>(static_cast<P2PNode*>(n)->peers.size()) < connectionCount) {
        int pp2 = rd.nextInt(static_cast<int>(allNodes.size()));
        createLink(n->nodeId, pp2);
      }
    }
  }
  void createLink(int pp1, int pp2) {  // :71-92
    if (pp1 == pp2) return;
    int64_t l1 = std::min(pp1, pp2), l2 = std::max(pp1, pp2);
    int64_t link = (l1 << 32) + l2;
    if (!existingLinks.insert(link).second) return;
    P2PNode& p1 = peer(pp1);
    P2PNode& p2 = peer(pp2);
    p1.peers.push_back(&p2);
    p2.peers.push_back(&p1);
  }
  int avgPeers() const {  // :115-125
    if (allNodes.empty()) return 0;
    int64_t tot = 0;
    for (Node* n : allNodes) tot += static_cast<int64_t>(static_cast<P2PNode*>(n)->peers.size());
    return static_cast<int>(tot / static_cast<int64_t>(allNodes.size()));
  }
  void sendPeers(const std::shared_ptr<FloodMessage>& msg, P2PNode& from) {  // :127-132
    msg->addToReceived(from);
    std::vector<Node*> dest(from.peers.begin(), from.peers.end());
    javaShuffle(dest, rd);
    send(msg, time + 1 + msg->localDelay, from, dest, msg->delayBetweenPeers);
  }
};

inline void FloodMessage::action(Network& network, Node& fromN, Node& toN) {
  P2PNode& from = static_cast<P2PNode&>(fromN);
  P2PNode& to = static_cast<P2PNode&>(toN);
  if (addToReceived(to)) {
    to.onFlood(from, *this);
    std::vector<Node*> dest;
    for (P2PNode* n : to.peers)
      if (n != &from) dest.push_back(n);
    javaShuffle(dest, network.rd);
    network.send(shared_from_this(), network.time + 1 + localDelay, to, dest, delayBetweenPeers);
  }
}

// P2PFlood :20-281
struct P2PFlood {
  struct Params {  // P2PFloodParameters :46-109 (JSON defaults :77-87)
    int nodeCount = 100, deadNodeCount = 10, delayBeforeResent = 50, msgCount = 1, msgToReceive = 1, peersCount = 10,
        delayBetweenSends = 30;
    std::string nodeBuilderName, networkLatencyName;
    bool latencyNull = true;
  };
  struct P2PFloodNode : P2PNode {  // :25-44
    P2PFlood* p;
    P2PFloodNode(P2PFlood* pp, bool down) : P2PNode(pp->network.rd, pp->nb), p(pp) {
      if (down) stop();
    }
    void onFlood(P2PNode&, const FloodMessage&) override {  // :39-43
      if (static_cast<int>(received.size()) == p->params.msgCount) doneAt = p->network.time;
    }
  };

  Params params;
  P2PNetwork network;
  NodeBuilder nb;
  std::vector<std::unique_ptr<P2PFloodNode>> nodes;
  std::vector<std::shared_ptr<FloodMessage>> msgs;  // the originating messages, in init's draw order (identity = index)

  explicit P2PFlood(const Params& pr) : params(pr), network(pr.peersCount) {  // :111-117
    nb = nodeBuilderByName(pr.nodeBuilderName);
    network.setNetworkLatency(networkLatencyByName(pr.networkLatencyName, pr.latencyNull));
  }
  void init() {  // :146-165
    for (int i = 0; i < params.nodeCount; i++) {
      nodes.push_back(std::make_unique<P2PFloodNode>(this, i < params.deadNodeCount));
      network.addNode(nodes.back().get());
    }
    network.setPeers();
    std::unordered_set<int> senders;
    while (static_cast<int>(senders.size()) < params.msgCount) {
      int nodeId = network.rd.nextInt(params.nodeCount);
      P2PFloodNode& from = *nodes[static_cast<size_t>(nodeId)];
      if (!from.isDown() && senders.insert(nodeId).second) {
        auto m = std::make_shared<FloodMessage>(1, params.delayBeforeResent, params.delayBetweenSends);
        msgs.push_back(m);
        network.sendPeers(m, from);
        if (params.msgCount == 1) from.doneAt = 1;
      }
    }
  }
};

}  // namespace wo
