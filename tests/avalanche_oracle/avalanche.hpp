// TEST INFRASTRUCTURE ONLY — CPU restatement of protocols/Slush.java and protocols/Snowflake.java on the oracle's core
// (oracle/core.hpp: Network, Node, Message, java.util.Random), line by line.  Line references are to those two files.
#pragma once
#include <algorithm>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../oracle/core.hpp"

namespace wo {

// ----------------------------------------------------------------------------------------
// Slush  (protocols/Slush.java)
// ----------------------------------------------------------------------------------------
struct Slush {
  struct Params {  // SlushParameters :14-52
    int NODES_AV = 100, M = 4, K = 7;
    double A = 4;
    double AK = 28;
    std::string nodeBuilderName, networkLatencyName;
    bool latencyNull = true;
  };
  struct Answer {  // :200-214
    int round;
    int colorsFound[3] = {0, 0, 0};
    explicit Answer(int r) : round(r) {}
    int answerCount() const { return colorsFound[0] + colorsFound[1] + colorsFound[2]; }
  };
  struct SlushNode;
  struct Query : Message {  // :86-99
    int id, color;
    Query(int i, int c) : id(i), color(c) {}
    void action(Network&, Node& from, Node& to) override;
  };
  struct AnswerQuery : Message {  // :101-114
    int originalQueryId, color;
    AnswerQuery(int q, int c) : originalQueryId(q), color(c) {}
    void action(Network&, Node& from, Node& to) override;
  };
  struct SlushNode : Node {  // :116-198
    Slush* p;
    int myColor = 0;
    int myQueryNonce = 0;
    int round = 0;
    std::unordered_map<int, Answer> answerIP;  // HashMap<Integer, Answer>
    explicit SlushNode(Slush* pp) : Node(pp->network.rd, pp->nb), p(pp) {}

    std::vector<Node*> randomRemotes() {  // :126-137
      std::vector<Node*> res;
      while (static_cast<int>(res.size()) != p->params.K) {
        int r = p->network.rd.nextInt(p->params.NODES_AV);
        Node* n = &p->network.getNodeById(r);
        if (r != nodeId && std::find(res.begin(), res.end(), n) == res.end()) res.push_back(n);  // ArrayList.contains
      }
      return res;
    }
    int otherColor() const { return myColor == 1 ? 2 : 1; }  // :139-141
    void onQuery(const Query& qa, Node& from) {  // :148-154
      if (myColor == 0) {
        myColor = qa.color;
        sendQuery(1);
      }
      p->network.send(std::make_shared<AnswerQuery>(qa.id, myColor), *this, from);
    }
    void onAnswer(int queryId, int color) {  // :161-176
      auto it = answerIP.find(queryId);
      if (it == answerIP.end()) throw IllegalState("answerIP.get(queryId) is null");  // NullPointerException
      Answer asw = it->second;
      asw.colorsFound[color]++;
      it->second = asw;
      if (asw.answerCount() == p->params.K) {
        answerIP.erase(it);
        if (asw.colorsFound[otherColor()] > p->params.AK) myColor = otherColor();
        if (round < p->params.M) {
          round++;
          sendQuery(asw.round + 1);
        }
      }
    }
    void sendQuery(int countInM) {  // :178-182
      int id = ++myQueryNonce;
      answerIP.erase(id);
      answerIP.emplace(id, Answer(countInM));
      p->network.send(std::make_shared<Query>(id, myColor), *this, randomRemotes());
    }
  };

  Params params;
  Network network;
  NodeBuilder nb;
  std::vector<std::unique_ptr<SlushNode>> nodes;

  explicit Slush(const Params& pr) : params(pr) {  // :54-60
    params.AK = params.K * params.A;  // :42
    nb = nodeBuilderByName(pr.nodeBuilderName);
    network.setNetworkLatency(networkLatencyByName(pr.networkLatencyName, pr.latencyNull));
  }
  void init() {  // :63-74
    for (int i = 0; i < params.NODES_AV; i++) {
      nodes.push_back(std::make_unique<SlushNode>(this));
      network.addNode(nodes.back().get());
    }
    SlushNode& uncolored1 = *nodes[0];
    SlushNode& uncolored2 = *nodes[1];
    uncolored1.myColor = 1;
    uncolored1.sendQuery(1);
    uncolored2.myColor = 2;
    uncolored2.sendQuery(1);
  }
};
inline void Slush::Query::action(Network&, Node& from, Node& to) { static_cast<SlushNode&>(to).onQuery(*this, from); }
inline void Slush::AnswerQuery::action(Network&, Node&, Node& to) { static_cast<SlushNode&>(to).onAnswer(originalQueryId, color); }

// ----------------------------------------------------------------------------------------
// Snowflake  (protocols/Snowflake.java)
// ----------------------------------------------------------------------------------------
struct Snowflake {
  struct Params {  // SnowflakeParameters :18-61
    int NODES_AV = 100, M = 4, K = 7;
    double A = 4;
    double AK = 28;
    int B = 7;
    std::string nodeBuilderName, networkLatencyName;
    bool latencyNull = true;
  };
  struct Answer {  // :217-232
    int round;
    int colorsFound[3] = {0, 0, 0};
    explicit Answer(int r) : round(r) {}
    int answerCount() const { return colorsFound[0] + colorsFound[1] + colorsFound[2]; }
  };
  struct SnowflakeNode;
  struct Query : Message {  // :95-108
    int id, color;
    Query(int i, int c) : id(i), color(c) {}
    void action(Network&, Node& from, Node& to) override;
  };
  struct AnswerQuery : Message {  // :110-123
    int originalQueryId, color;
    AnswerQuery(int q, int c) : originalQueryId(q), color(c) {}
    void action(Network&, Node& from, Node& to) override;
  };
  struct SnowflakeNode : Node {  // :125-215
    Snowflake* p;
    int myColor = 0;
    int myQueryNonce = 0;
    int cnt = 0;
    std::unordered_map<int, Answer> answerIP;  // HashMap<Integer, Answer>
    explicit SnowflakeNode(Snowflake* pp) : Node(pp->network.rd, pp->nb), p(pp) {}

    std::vector<Node*> randomRemotes() {  // :136-147
      std::vector<Node*> res;
      while (static_cast<int>(res.size()) != p->params.K) {
        int r = p->network.rd.nextInt(p->params.NODES_AV);
        Node* n = &p->network.getNodeById(r);
        if (r != nodeId && std::find(res.begin(), res.end(), n) == res.end()) res.push_back(n);  // ArrayList.contains
      }
      return res;
    }
    int otherColor() const { return myColor == 1 ? 2 : 1; }  // :149-151
    void onQuery(const Query& qa, Node& from) {  // :153-159
      if (myColor == 0) {
        myColor = qa.color;
        sendQuery(1);
      }
      p->network.send(std::make_shared<AnswerQuery>(qa.id, myColor), *this, from);
    }
    void onAnswer(int queryId, int color) {  // :170-188
      auto it = answerIP.find(queryId);
      if (it == answerIP.end()) throw IllegalState("answerIP.get(queryId) is null");  // NullPointerException
      Answer asw = it->second;
      asw.colorsFound[color]++;
      it->second = asw;
      if (asw.answerCount() == p->params.K) {
        answerIP.erase(it);
        if (asw.colorsFound[otherColor()] > p->params.AK) {
          myColor = otherColor();
          cnt = 0;
        } else {
          if (asw.colorsFound[myColor] > p->params.AK) cnt++;
        }
        if (cnt <= p->params.B) sendQuery(asw.round + 1);
      }
    }
    void sendQuery(int countInM) {  // :190-194
      int id = ++myQueryNonce;
      answerIP.erase(id);
      answerIP.emplace(id, Answer(countInM));
      p->network.send(std::make_shared<Query>(id, myColor), *this, randomRemotes());
    }
  };

  Params params;
  Network network;
  NodeBuilder nb;
  std::vector<std::unique_ptr<SnowflakeNode>> nodes;

  explicit Snowflake(const Params& pr) : params(pr) {  // :63-69
    params.AK = params.A * params.K;  // :51
    nb = nodeBuilderByName(pr.nodeBuilderName);
    network.setNetworkLatency(networkLatencyByName(pr.networkLatencyName, pr.latencyNull));
  }
  void init() {  // :77-88
    for (int i = 0; i < params.NODES_AV; i++) {
      nodes.push_back(std::make_unique<SnowflakeNode>(this));
      network.addNode(nodes.back().get());
    }
    SnowflakeNode& uncolored1 = *nodes[0];
    SnowflakeNode& uncolored2 = *nodes[1];
    uncolored1.myColor = 1;
    uncolored1.sendQuery(1);
    uncolored2.myColor = 2;
    uncolored2.sendQuery(1);
  }
};
inline void Snowflake::Query::action(Network&, Node& from, Node& to) { static_cast<SnowflakeNode&>(to).onQuery(*this, from); }
inline void Snowflake::AnswerQuery::action(Network&, Node&, Node& to) {
  static_cast<SnowflakeNode&>(to).onAnswer(originalQueryId, color);
}

}  // namespace wo
