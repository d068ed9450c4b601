"""REST façade over the C ABI: the reference's `wserver` surface for the accelerated protocols.

Reference: wserver/src/main/java/net/consensys/wittgenstein/server/IServer.java:9-34 (the interface),
Server.java:20-172 (its implementation over a `Protocol`), ws/WServer.java:19-125 (the Spring REST controller under `/w`),
core/EnvelopeInfo.java:8-14, core/messages/SendMessage.java:5-25, core/WParameters.java:9-15 (JSON objects carry their
simple class name in the property `type`), core/External.java.

`Server` mirrors `Server.java` method by method on top of the Python mirror of the protocol classes (one C-ABI call per
method); `create_app()` exposes it with the same routes, verbs and JSON field names as `WServer.java`, so that the
reference's web UI (wserver/src/main/resources/static) and HTTP clients can drive the device engine.  Differences, all
reported as HTTP errors instead of being guessed:
  * `POST /w/network/nodes/{id}/external` (Server.setExternal): a per-delivery HTTP callback cannot run inside a device
    handler -> 501 (SURVEY.md §8b: host-defined `Message.action` bodies are not part of the accelerated ABI);
  * `POST /w/network/send` accepts the message types the engine can inject from the host (PingPong: Ping / Pong;
    CasperIMD: SendBlock / Attestation with their block / attestation index as `payload`); other types -> 400.
"""
import threading

import numpy as np

from . import protocols as P
from ._lib import WtgError

PKG = "net.consensys.wittgenstein.protocols."

# Java field name -> attribute of the Python parameter mirror, in constructor order
_PARAMS = {
    "PingPong": (P.PingPong, P.PingPongParameters, "PingPongParameters",
                 [("nodeCt", "node_ct"), ("nodeBuilderName", "node_builder_name"), ("networkLatencyName", "network_latency_name")]),
    "GSFSignature": (P.GSFSignature, P.GSFSignatureParameters, "GSFSignatureParameters",
                     [("nodeCount", "node_count"), ("threshold", "threshold"), ("pairingTime", "pairing_time"),
                      ("timeoutPerLevelMs", "timeout_per_level_ms"), ("periodDurationMs", "period_duration_ms"),
                      ("acceleratedCallsCount", "accelerated_calls_count"), ("nodesDown", "nodes_down"),
                      ("nodeBuilderName", "node_builder_name"), ("networkLatencyName", "network_latency_name")]),
    "SanFerminSignature": (P.SanFerminSignature, P.SanFerminSignatureParameters, "SanFerminSignatureParameters",
                           [("nodeCount", "node_count"), ("threshold", "threshold"), ("pairingTime", "pairing_time"),
                            ("signatureSize", "signature_size"), ("replyTimeout", "reply_timeout"), ("candidateCount", "candidate_count"),
                            ("shuffledLists", "shuffled_lists"), ("nodeBuilderName", "node_builder_name"),
                            ("networkLatencyName", "network_latency_name")]),
    "CasperIMD": (P.CasperIMD, P.CasperParemeters, "CasperParemeters",
                  [("cycleLength", "cycle_length"), ("randomOnTies", "random_on_ties"), ("blockProducersCount", "block_producers_count"),
                   ("attestersPerRound", "attesters_per_round"), ("blockConstructionTime", "block_construction_time"),
                   ("attestationConstructionTime", "attestation_construction_time"), ("nodeBuilderName", "node_builder_name"),
                   ("networkLatencyName", "network_latency_name")]),
    "SanFerminCappos": (P.SanFerminCappos, P.SanFerminCapposParameters, "SanFerminParameters",
                        [("nodeCount", "node_count"), ("threshold", "threshold"), ("pairingTime", "pairing_time"),
                         ("signatureSize", "signature_size"), ("timeout", "timeout"), ("candidateCount", "candidate_count"),
                         ("nodeBuilderName", "node_builder_name"), ("networkLatencyName", "network_latency_name")]),
    "Handel": (P.Handel, P.HandelParameters, "HandelParameters",
               [("nodeCount", "node_count"), ("threshold", "threshold"), ("pairingTime", "pairing_time"),
                ("levelWaitTime", "level_wait_time"), ("extraCycle", "extra_cycle"), ("disseminationPeriodMs", "dissemination_period_ms"),
                ("fastPath", "fast_path"), ("nodesDown", "nodes_down"), ("nodeBuilderName", "node_builder_name"),
                ("networkLatencyName", "network_latency_name"), ("desynchronizedStart", "desynchronized_start"),
                ("byzantineSuicide", "byzantine_suicide"), ("hiddenByzantine", "hidden_byzantine")]),
}

# message type names (simple class names, the `type` property of the JSON) <-> the engine's type codes (csrc/wtg_types.h)
_MSG_TYPES = {
    "PingPong": {"Ping": 1, "Pong": 2},
    "CasperIMD": {"Attestation": 1, "SendBlock": 2},
    "SanFerminSignature": {"SwapRequest": 1, "SwapReply": 2},
    "SanFerminCappos": {"SwapReply": 1, "Swap": 2},
}
_AWS_CITIES = None


def _simple(full_class_name):
    name = full_class_name[len(PKG):] if full_class_name.startswith(PKG) else full_class_name
    if name not in _PARAMS:
        raise KeyError("Class not found: " + full_class_name)  # Server.java:31-33
    return name


class Server:
    """Server.java: holds one protocol instance; every method maps onto the C ABI through the Python mirror."""

    def __init__(self, _api=None):
        self._api = _api
        self.protocol = None
        self.name = None
        self._lock = threading.Lock()  # the reference's engine is single-threaded (Network.java:10); so is a wtg_net handle

    # ---- protocols and their parameters (Server.java:53-108) ----
    def get_protocols(self):
        return [PKG + n for n in _PARAMS]

    def get_protocol_parameters(self, full_class_name):
        """The parameter object built by its no-argument constructor (Server.java:73-108), as its JSON form."""
        name = _simple(full_class_name)
        _, pcls, ptype, fields = _PARAMS[name]
        prm = pcls()
        out = {"type": ptype}
        for java, py in fields:
            out[java] = getattr(prm, py)
        return out

    def init(self, full_class_name, parameters):
        """Server.init (:47-51): protocol = new <class>(parameters); protocol.init()."""
        name = _simple(full_class_name)
        cls, pcls, _, fields = _PARAMS[name]
        parameters = dict(parameters or {})
        kwargs = {py: parameters[java] for java, py in fields if java in parameters}  # unknown properties are ignored (ObjectMapperFactory.java:16)
        with self._lock:
            if self.protocol is not None:
                self.protocol.network().close()
            prm = pcls(**kwargs)
            self.protocol = cls(prm, _api=self._api) if self._api is not None else cls(prm)
            self.name = name
            self.protocol.init()

    def _net(self):
        if self.protocol is None:
            raise WtgError("no protocol initialised: POST /w/network/init/{fullClassName} first")
        return self.protocol.network()

    # ---- network (Server.java:24-29, 130-172) ----
    def get_time(self):
        with self._lock:
            return self._net().time

    def run_ms(self, ms):
        with self._lock:
            self._net().run_ms(int(ms))

    def start_node(self, node_id):
        with self._lock:
            self._net().start_node(int(node_id))

    def stop_node(self, node_id):
        with self._lock:
            self._net().stop_node(int(node_id))

    def set_external(self, node_id, address):
        raise NotImplementedError("Node.setExternal: an external (HTTP) handler cannot run inside a device-side Message.action")

    def _nodes(self):
        net = self._net()
        a = net.attrs()
        c = net.counters()
        n = net.node_count
        extra = {}
        if self.name == "PingPong":
            extra["pong"] = self.protocol.pongs()
        out = []
        for i in range(n):
            d = {"nodeId": i, "x": int(a["x"][i]), "y": int(a["y"][i]), "extraLatency": int(a["extra"][i]), "byzantine": False,
                 "speedRatio": float(a["speed"][i]), "cityIndex": int(a["city"][i]), "down": bool(a["down"][i]),
                 "msgReceived": int(c[0][i]), "msgSent": int(c[1][i]), "bytesSent": int(c[2][i]), "bytesReceived": int(c[3][i]),
                 "doneAt": int(c[4][i]), "external": None}
            for k, v in extra.items():
                d[k] = int(v[i])
            out.append(d)
        return out

    def get_node_info(self, node_id=None):
        """Server.getNodeInfo() / getNodeInfo(nodeId): the public fields of core/Node.java:22-79."""
        with self._lock:
            nodes = self._nodes()
        if node_id is None:
            return nodes
        if node_id < 0 or node_id >= len(nodes):
            raise IndexError(f"node {node_id}")
        return nodes[node_id]

    def get_messages(self, cap=1 << 16):
        """Server.getMessages (:169-172) = network.msgs.peekMessages(): EnvelopeInfo rows sorted by arrival."""
        with self._lock:
            _, r = self._net().peek_messages(cap)
        names = {v: k for k, v in _MSG_TYPES.get(self.name, {}).items()}
        out = []
        for i in range(len(r["from"])):
            kind = int(r["kind"][i])
            t = int(r["msg_type"][i])
            if kind == 2:
                mtype = "Task"
            elif kind == 3:
                mtype = "PeriodicTask"
            elif self.name in ("GSFSignature", "Handel"):
                mtype = "SendSigs"
            else:
                mtype = names.get(t, str(t))
            out.append({"from": int(r["from"][i]), "to": int(r["to"][i]), "sentAt": int(r["sent_at"][i]),
                        "arrivingAt": int(r["arriving_at"][i]), "msg": {"type": mtype, "code": t}})
        return out

    def send_message(self, msg):
        """Server.sendMessage (:160-167): network.send(message, sendTime, from, dests, delayBetweenSend)."""
        m = msg.get("message") or {}
        mtype = m.get("type")
        codes = _MSG_TYPES.get(self.name, {})
        if isinstance(mtype, str) and mtype in codes:
            code = codes[mtype]
        elif isinstance(mtype, int):
            code = mtype
        else:
            raise WtgError(f"message type {mtype!r} cannot be sent from the host on {self.name}")
        to = [int(t) for t in (msg.get("to") or [])]
        if not to:
            raise WtgError("no destination")
        with self._lock:
            net = self._net()
            net.send(code, int(msg.get("from", 0)), to if len(to) > 1 else to[0], payload=int(m.get("payload", 0)),
                     send_time=int(msg.get("sendTime", net.time + 1)), delay_between=int(msg.get("delayBetweenSend", 0)))


def create_app(server=None):
    """The routes of ws/WServer.java:23-104 (same paths, verbs and JSON) as an ASGI application (FastAPI)."""
    from fastapi import Body, FastAPI, HTTPException
    from fastapi.responses import PlainTextResponse

    srv = server or Server()
    app = FastAPI(title="wittgenstein_b200 wserver")
    app.state.server = srv

    def guarded(fn, *a):
        try:
            return fn(*a)
        except NotImplementedError as e:
            raise HTTPException(status_code=501, detail=str(e))
        except (KeyError, IndexError) as e:
            raise HTTPException(status_code=404, detail=str(e))
        except (WtgError, ValueError, TypeError) as e:
            raise HTTPException(status_code=400, detail=str(e))

    @app.get("/w/network/nodes")  # WServer.java:26-30
    def nodes():
        return guarded(srv.get_node_info)

    @app.get("/w/network/time", response_class=PlainTextResponse)  # :32-36 (the body is the bare integer)
    def time():
        return str(guarded(srv.get_time))

    @app.get("/w/protocols")  # :38-42
    def protocols():
        return srv.get_protocols()

    @app.get("/w/protocols/{full_class_name}")  # :44-48
    def protocol_parameters(full_class_name: str):
        return guarded(srv.get_protocol_parameters, full_class_name)

    @app.post("/w/network/init/{full_class_name}")  # :50-54
    def init(full_class_name: str, parameters: dict = Body(default=None)):
        guarded(srv.init, full_class_name, parameters)

    @app.post("/w/network/runMs/{ms}")  # :56-60
    def run_ms(ms: int):
        guarded(srv.run_ms, ms)

    @app.get("/w/network/nodes/{node_id}")  # :62-66
    def node(node_id: int):
        return guarded(srv.get_node_info, node_id)

    @app.get("/w/network/messages")  # :68-72
    def messages():
        return guarded(srv.get_messages)

    @app.post("/w/nodes/{node_id}/start")  # :74-78 (the reference's path has no /network here)
    @app.post("/w/network/nodes/{node_id}/start")
    def start(node_id: int):
        guarded(srv.start_node, node_id)

    @app.post("/w/network/nodes/{node_id}/stop")  # :80-84
    def stop(node_id: int):
        guarded(srv.stop_node, node_id)

    @app.post("/w/network/nodes/{node_id}/external")  # :86-91
    def external(node_id: int, address: str = Body(default="")):
        guarded(srv.set_external, node_id, address)

    @app.post("/w/network/send")  # :93-97
    @app.post("/w/network/send/")
    def send(msg: dict = Body(...)):
        guarded(srv.send_message, msg)

    return app


def main(host="127.0.0.1", port=8080):
    """WServer.main (:121-123)."""
    import uvicorn

    uvicorn.run(create_app(), host=host, port=port)


if __name__ == "__main__":
    main()
