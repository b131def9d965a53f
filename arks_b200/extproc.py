"""ext_proc gRPC surface of arks-gateway-plugins over the batched engine (BASELINE config 1: loopback plumbing).

Host-side mirror of `Server.Process` and its four handlers (pkg/gateway/gateway.go:77-138,
handle_request.go:33-249, handle_response.go:37-268, util.go:40-77 of the reference): one bidi stream per HTTP
request, messages RequestHeaders -> RequestBody -> ResponseHeaders -> ResponseBody*, replies shaped like the Go
server's. What used to be Redis/informer calls inside the handlers is one enqueue into a micro-batcher whose worker
calls `engine.handle_request_body / handle_response_body` (the C ABI on a GPU; the parity tests plug the oracle in on
CPU boxes because the product has no CPU path).

No protoc / grpc_tools in this image: the handful of envoy.service.ext_proc.v3 / envoy.config.core.v3 messages used
on this path are declared programmatically below with the upstream field numbers (envoy API v3 as vendored by
go-control-plane v1.32.4). tools/verify_descriptors.py checks the envoy.config.core.v3 / envoy.type.v3 ones against the
descriptors grpcio's C core embeds (tests/test_descriptors.py); the ext_proc service messages are in no package of this
image and stay hand-typed from the published .proto layout — re-check those before pointing a real Envoy at it.
Enum-typed upstream fields (HttpStatus.code, CommonResponse.status) are declared int32 here: same wire encoding.
"""
from __future__ import annotations

import json
import queue
import threading
import time
from concurrent import futures

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

from . import abi, replies
from .abi import RequestBatch, ResponseBatch

# --------------------------------------------------------------------------------------------------
# protobuf messages
# --------------------------------------------------------------------------------------------------
_T = descriptor_pb2.FieldDescriptorProto


def _build_messages():
    f = descriptor_pb2.FileDescriptorProto()
    f.name, f.package, f.syntax = "arks_extproc_subset.proto", "envoy.service.ext_proc.v3", "proto3"

    def msg(name, fields, oneof=None):
        m = f.message_type.add()
        m.name = name
        if oneof:
            m.oneof_decl.add().name = oneof
        for fname, num, ftype, tname, rep, in_oneof in fields:
            fd = m.field.add()
            fd.name, fd.number, fd.type = fname, num, ftype
            fd.label = _T.LABEL_REPEATED if rep else _T.LABEL_OPTIONAL
            if tname:
                fd.type_name = ".envoy.service.ext_proc.v3." + tname
            if in_oneof:
                fd.oneof_index = 0
        return m

    M, S, B, BY, I32 = _T.TYPE_MESSAGE, _T.TYPE_STRING, _T.TYPE_BOOL, _T.TYPE_BYTES, _T.TYPE_INT32
    # envoy.config.core.v3 (flattened into this package: only the wire format matters for the loopback)
    msg("HeaderValue", [("key", 1, S, None, 0, 0), ("value", 2, S, None, 0, 0), ("raw_value", 3, BY, None, 0, 0)])
    msg("HeaderMap", [("headers", 1, M, "HeaderValue", 1, 0)])
    msg("HeaderValueOption", [("header", 1, M, "HeaderValue", 0, 0)])
    msg("HttpStatus", [("code", 1, I32, None, 0, 0)])
    # envoy.service.ext_proc.v3
    msg("HttpHeaders", [("headers", 1, M, "HeaderMap", 0, 0), ("end_of_stream", 3, B, None, 0, 0)])
    msg("HttpBody", [("body", 1, BY, None, 0, 0), ("end_of_stream", 2, B, None, 0, 0)])
    msg("HeaderMutation", [("set_headers", 1, M, "HeaderValueOption", 1, 0), ("remove_headers", 2, S, None, 1, 0)])
    msg("CommonResponse", [("status", 1, I32, None, 0, 0), ("header_mutation", 2, M, "HeaderMutation", 0, 0),
                           ("clear_route_cache", 5, B, None, 0, 0)])
    msg("HeadersResponse", [("response", 1, M, "CommonResponse", 0, 0)])
    msg("BodyResponse", [("response", 1, M, "CommonResponse", 0, 0)])
    msg("ImmediateResponse", [("status", 1, M, "HttpStatus", 0, 0), ("headers", 2, M, "HeaderMutation", 0, 0),
                              ("body", 3, BY, None, 0, 0), ("details", 5, S, None, 0, 0)])
    msg("ProcessingRequest", [("request_headers", 2, M, "HttpHeaders", 0, 1), ("response_headers", 3, M, "HttpHeaders", 0, 1),
                              ("request_body", 4, M, "HttpBody", 0, 1), ("response_body", 5, M, "HttpBody", 0, 1)],
        oneof="request")
    msg("ProcessingResponse", [("request_headers", 1, M, "HeadersResponse", 0, 1),
                               ("response_headers", 2, M, "HeadersResponse", 0, 1),
                               ("request_body", 3, M, "BodyResponse", 0, 1), ("response_body", 4, M, "BodyResponse", 0, 1),
                               ("immediate_response", 7, M, "ImmediateResponse", 0, 1)], oneof="response")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(f)
    get = lambda n: message_factory.GetMessageClass(pool.FindMessageTypeByName("envoy.service.ext_proc.v3." + n))
    return {n: get(n) for n in ("HeaderValue", "HeaderMap", "HeaderValueOption", "HttpStatus", "HttpHeaders", "HttpBody",
                                "HeaderMutation", "CommonResponse", "HeadersResponse", "BodyResponse",
                                "ImmediateResponse", "ProcessingRequest", "ProcessingResponse")}


PB = _build_messages()
SERVICE = "envoy.service.ext_proc.v3.ExternalProcessor"


def _build_health_messages():
    """grpc.health.v1 (grpc/health/v1/health.proto): the four messages of Check / List / Watch"""
    f = descriptor_pb2.FileDescriptorProto()
    f.name, f.package, f.syntax = "arks_health_subset.proto", "grpc.health.v1", "proto3"
    m = f.message_type.add()
    m.name = "HealthCheckRequest"
    fd = m.field.add()
    fd.name, fd.number, fd.type, fd.label = "service", 1, _T.TYPE_STRING, _T.LABEL_OPTIONAL
    m = f.message_type.add()
    m.name = "HealthCheckResponse"
    e = m.enum_type.add()
    e.name = "ServingStatus"
    for i, n in enumerate(("UNKNOWN", "SERVING", "NOT_SERVING", "SERVICE_UNKNOWN")):
        v = e.value.add()
        v.name, v.number = n, i
    fd = m.field.add()
    fd.name, fd.number, fd.type, fd.label = "status", 1, _T.TYPE_ENUM, _T.LABEL_OPTIONAL
    fd.type_name = ".grpc.health.v1.HealthCheckResponse.ServingStatus"
    f.message_type.add().name = "HealthListRequest"
    m = f.message_type.add()
    m.name = "HealthListResponse"
    ent = m.nested_type.add()  # map<string, HealthCheckResponse> statuses = 1
    ent.name = "StatusesEntry"
    ent.options.map_entry = True
    k = ent.field.add()
    k.name, k.number, k.type, k.label = "key", 1, _T.TYPE_STRING, _T.LABEL_OPTIONAL
    v = ent.field.add()
    v.name, v.number, v.type, v.label, v.type_name = "value", 2, _T.TYPE_MESSAGE, _T.LABEL_OPTIONAL, ".grpc.health.v1.HealthCheckResponse"
    fd = m.field.add()
    fd.name, fd.number, fd.type, fd.label = "statuses", 1, _T.TYPE_MESSAGE, _T.LABEL_REPEATED
    fd.type_name = ".grpc.health.v1.HealthListResponse.StatusesEntry"
    pool = descriptor_pool.DescriptorPool()
    pool.Add(f)
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName("grpc.health.v1." + n))
            for n in ("HealthCheckRequest", "HealthCheckResponse", "HealthListRequest", "HealthListResponse")}


HEALTH_PB = _build_health_messages()
HEALTH_SERVICE = "grpc.health.v1.Health"
SERVING = 1


class HealthServer:
    """HealthServer of the reference (pkg/gateway/gateway.go:261-279): always SERVING, empty List, Watch unimplemented"""

    def Check(self, request, context):
        return HEALTH_PB["HealthCheckResponse"](status=SERVING)

    def List(self, request, context):
        return HEALTH_PB["HealthListResponse"]()

    def Watch(self, request, context):
        import grpc
        context.abort(grpc.StatusCode.UNIMPLEMENTED, "watch is not implemented")


# ---- GET /v1/models (pkg/gateway/http_handler.go:18-60; the plain HTTP listener of gateway.go:140-157) ----------------
def models_reply(tables, authorization):
    """-> (status, content type, body) of handleGetModels. GetModelsByToken (qosconfig/arks_impl.go:378-397): the qos
    entries' endpoint names of the FIRST ArksToken object with that spec.token; an unknown token is a 500, like there.
    Model objects are openai-go v0.1.0-beta.3's `Model` marshalled by encoding/json (a go.mod dependency that is not
    vendored: its published struct has id, created, object, owned_by, all emitted); no models -> "data":null (nil slice)."""
    text = "text/plain; charset=utf-8"
    if authorization is None or not authorization.startswith("Bearer "):
        return 401, text, b"Unauthorized\n"
    token = authorization[len("Bearer "):]
    if token == "":
        return 401, text, b"Unauthorized\n"
    try:
        t = tables.token_string.index(token)
    except ValueError:
        return 500, text, b"error in getting model list\n"
    lo, hi = int(tables.tok_qos_off[t]), int(tables.tok_qos_off[t + 1])
    data = [{"id": tables.qos_model_name[q], "created": 0, "object": "model", "owned_by": ""} for q in range(lo, hi)] or None
    return 200, "application/json", json.dumps({"object": "list", "data": data}, separators=(",", ":"), ensure_ascii=False).encode()


def serve_http(get_tables, port: int = 8080, host: str = "127.0.0.1"):
    """the /v1/models listener; get_tables() returns the current arks_b200.tables.Tables (it changes with the config plane)"""
    from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer

    class H(BaseHTTPRequestHandler):
        def _any(self):
            if self.path.split("?", 1)[0] != "/v1/models":  # http.ServeMux: 404 page not found
                st, ct, body = 404, "text/plain; charset=utf-8", b"404 page not found\n"
            else:
                st, ct, body = models_reply(get_tables(), self.headers.get("Authorization"))
            self.send_response(st)
            self.send_header("Content-Type", ct)
            if st != 200:
                self.send_header("X-Content-Type-Options", "nosniff")  # http.Error
            self.send_header("Content-Length", str(len(body)))
            self.end_headers()
            if self.command != "HEAD":
                self.wfile.write(body)

        do_GET = do_POST = do_HEAD = do_PUT = do_DELETE = _any  # the mux pattern has no method: every verb is served

        def log_message(self, *a):
            pass

    httpd = ThreadingHTTPServer((host, port), H)
    th = threading.Thread(target=httpd.serve_forever, daemon=True)
    th.start()
    return httpd, httpd.server_address[1]

# header names, pkg/gateway/types.go:24-56
H_WENT_REQ, H_WENT_RESP = "x-went-into-req-headers", "x-went-into-resp-headers"


def _set_headers(pairs):
    mut = PB["HeaderMutation"]()
    for k, v in pairs:
        o = mut.set_headers.add()
        o.header.key = k
        o.header.raw_value = v if isinstance(v, bytes) else str(v).encode("utf-8", "surrogateescape")  # Go strings are bytes
    return mut


def error_response(status: int, header: str, header_value, message: str):
    """generateErrorResponse, pkg/gateway/util.go:40-77: status + x-error-* header + Content-Type + JSON body."""
    r = PB["ProcessingResponse"]()
    im = r.immediate_response
    im.status.code = status
    im.headers.CopyFrom(_set_headers([(header, header_value)]))
    ct = im.headers.set_headers.add()
    ct.header.key, ct.header.value = "Content-Type", "application/json"
    im.body = replies.error_body(message, status)
    return r


def passthrough_error(status: int, headers, message: str):
    """responseErrorProcessing, gateway.go:281-294: the headers of the reply built so far (none in the body phase)"""
    r = PB["ProcessingResponse"]()
    im = r.immediate_response
    im.status.code = status
    im.headers.CopyFrom(_set_headers(headers))
    ct = im.headers.set_headers.add()
    ct.header.key, ct.header.value = "Content-Type", "application/json"
    im.body = replies.error_body(message, status)
    return r


# --------------------------------------------------------------------------------------------------
# micro-batcher (the Python twin of host/cpp Batcher)
# --------------------------------------------------------------------------------------------------
class Batcher:
    """Stream handlers enqueue; one worker thread cuts batches by deadline (max_wait_s) or size and makes one engine
    call per batch. `clock()` stamps each batch (the engine never reads a clock)."""

    def __init__(self, engine, max_batch=4096, max_wait_s=200e-6, clock=time.time):
        self.engine, self.max_batch, self.max_wait, self.clock = engine, max_batch, max_wait_s, clock
        self.q: queue.Queue = queue.Queue()
        self.batches = 0
        self._stop = False
        self._now = -1 << 62
        self.t = threading.Thread(target=self._run, daemon=True)
        self.t.start()

    def close(self):
        self._stop = True
        self.q.put(None)
        self.t.join(timeout=5)

    def _answer(self, item):
        """enqueue and wait for the worker; a row that arrives after close() (or that the worker left behind when it stopped)
        is answered like an engine failure instead of holding its stream forever"""
        ev = item["ev"] = threading.Event()
        self.q.put(item)
        while not ev.wait(0.1):
            if self._stop and not self.t.is_alive():
                return dict(self._FAILED, error="the batcher is closed")
        return item["out"]

    def request(self, body: bytes, token: bytes):
        return self._answer({"kind": "req", "body": body, "token": token})

    def response(self, body: bytes, qos: int, flags: int, gen: int = None):
        return self._answer({"kind": "resp", "body": body, "qos": qos, "flags": flags, "gen": gen})

    def between_batches(self, fn):
        """run fn() on the worker thread between two engine calls (a table generation swap: arks_commit_tables belongs to the
        batch thread); what was enqueued before is decided first. Returns fn's result, re-raises its exception."""
        ev = threading.Event()
        item = {"kind": "call", "fn": fn, "ev": ev}
        self.q.put(item)
        while not ev.wait(0.1):
            if self._stop and not self.t.is_alive():  # closed before the call's turn came
                raise RuntimeError("the batcher is closed")
        if "error" in item:
            raise item["error"]
        return item["out"]

    _FAILED = {"reason": 255, "detail": 0, "flags": 0, "qos": -1, "token": -1, "pick": -1, "cur_usage": 0, "limit_max": 0,
               "counted": 0, "usage": [0, 0, 0], "now": 0, "gen": 0, "model_off": 0, "model_len": 0}

    def _run(self):
        while not self._stop:
            items = self._collect()
            if not items:
                continue
            run = []
            for it in items + [None]:
                if it is not None and it["kind"] != "call":
                    run.append(it)
                    continue
                if run:
                    try:
                        self._decide(run)
                    except Exception as e:  # an engine error must neither kill the worker nor strand the handlers of this cycle
                        for i in run:
                            if "out" not in i:
                                i["out"] = dict(self._FAILED, error=repr(e))
                                i["ev"].set()
                    run = []
                if it is not None:
                    try:
                        it["out"] = it["fn"]()
                    except Exception as e:
                        it["error"] = e
                    it["ev"].set()

    def _collect(self):
        first = self.q.get()
        if first is None:
            self._stop = True
            return []
        items = [first]
        deadline = time.perf_counter() + self.max_wait
        while len(items) < self.max_batch:
            left = deadline - time.perf_counter()
            if left <= 0:
                break
            try:
                it = self.q.get(timeout=left)
            except queue.Empty:
                break
            if it is None:
                self._stop = True
                break
            items.append(it)
        return items

    def _decide(self, items):
        now = self._now = max(int(self.clock()), self._now)  # a wall clock that steps back must not fail the batch
        gen = getattr(self.engine, "generation", 0)
        reqs = [i for i in items if i["kind"] == "req"]
        resps = [i for i in items if i["kind"] == "resp"]
        if reqs:  # arrival order inside the batch == index order == the linearisation the decisions follow
            rnd = np.random.default_rng(self.batches).integers(0, 1 << 63, len(reqs), dtype=np.uint64)
            r = self.engine.handle_request_body(
                RequestBatch.from_lists([i["body"] for i in reqs], [i["token"] for i in reqs], now, pick_rand=rnd))
            for k, i in enumerate(reqs):
                i["out"] = {f: v[k] for f, v in r.fields().items()}
                i["out"].update({f: tuple(v[k]) if v.ndim > 1 else int(v[k]) for f, v in r.report().items()})  # report on
                i["out"].update(now=now, gen=gen)
                i["ev"].set()
        if resps:
            r = self.engine.handle_response_body(
                ResponseBatch.from_lists([i["body"] for i in resps], [i["qos"] for i in resps], [i["flags"] for i in resps], now,
                                         gen=[gen if i["gen"] is None else i["gen"] for i in resps]))
            for k, i in enumerate(resps):
                i["out"] = {"reason": r.reason[k], "counted": r.counted[k], "usage": r.usage[k]}
                i["ev"].set()
        self.batches += 1


# --------------------------------------------------------------------------------------------------
# the ext_proc server
# --------------------------------------------------------------------------------------------------
class CompiledBatcher:
    """The same interface as Batcher, served by the compiled micro-batcher (host/cpp arks_host::Batcher through
    arks_b200/cpphost.py): gRPC handler threads block inside C++ (ctypes releases the GIL) and are batched there."""

    def __init__(self, cpp_batcher, clock=None):
        """clock=None (a production server): the C++ batcher reads the wall clock for every batch, so the rate-limit windows
        roll. A test passes a callable and the batcher is pinned to its reading."""
        self.b = cpp_batcher
        self._clock = clock
        if clock is not None:
            self.b.set_fixed_clock(int(clock()))

    @property
    def clock(self):
        return self._clock

    @clock.setter
    def clock(self, fn):  # the loopback tests move time
        self._clock = fn
        self.b.set_fixed_clock(int(fn()))

    def request(self, body: bytes, token: bytes):
        d = self.b.request(token, body, 0)
        return {"reason": d.reason, "detail": d.detail, "flags": d.flags, "qos": d.qos, "token": d.token, "pick": d.pick,
                "cur_usage": d.cur_usage, "limit_max": d.limit_max, "now": d.now_unix, "gen": d.gen,
                "model_off": d.model_off, "model_len": d.model_len, "rl_entry": tuple(d.rl_entry), "rl_limit": tuple(d.rl_limit),
                "rl_remaining": tuple(d.rl_remaining), **({"rl_reset": tuple(d.rl_reset), "rl_retry": d.rl_retry} if d.rl_sliding else {})}

    def response(self, body: bytes, qos: int, flags: int, gen: int = None):
        d = self.b.response(qos, body, flags, gen)
        return {"reason": d.reason, "counted": d.counted, "usage": list(d.usage)}

    def close(self):
        self.b.close()


class ExtProcServer:
    def __init__(self, engine, tables, extract_bearer, max_wait_s=200e-6, clock=time.time, batcher=None):
        """engine: handle_request_body / handle_response_body; tables: arks_b200.tables.Tables (names for the routing
        headers); extract_bearer: HandleRequestHeaders' scan (the C ABI's host function); batcher: a CompiledBatcher to
        batch in C++ instead of the Python twin."""
        self.tables = tables
        self._names = {int(getattr(engine, "generation", 0) or 0): tables}  # generation -> names; a stream keeps its request's
        self.extract_bearer = extract_bearer
        self.batcher = batcher or Batcher(engine, max_wait_s=max_wait_s, clock=clock)
        from .metrics import HostMetrics
        self.metrics = HostMetrics()  # the wall-clock series (durations, non-200 statuses); the rest is counted on the device
        self.monotonic = time.monotonic

    # ---- Server.Process, gateway.go:77-138
    def Process(self, request_iterator, context):
        token, qos, stream, status, rl = b"", (-1, None), False, 0, []
        buffered = bytearray()
        start, completed, resp_spent = self.monotonic(), False, 0.0
        for req in request_iterator:
            kind = req.WhichOneof("request")
            if kind == "request_headers":
                start = self.monotonic()  # requestStart, gateway.go:108
                resp, token = self.handle_request_headers(req)
            elif kind == "request_body":
                resp, qos, stream, rl = self.handle_request_body(req, token)
            elif kind == "response_headers":
                resp, status = self.handle_response_headers(req, rl)
                if status == 500:  # gateway.go:115-121 -> responseErrorProcessing keeps the reply's headers, empty message
                    self._record_request(qos, start, status)
                    hs = [(o.header.key, o.header.raw_value) for o in resp.response_headers.response.header_mutation.set_headers]
                    resp = passthrough_error(500, hs, "")
            elif kind == "response_body":
                if status != 200:  # gateway.go:122-126: pass the upstream error through
                    resp = passthrough_error(status, [], req.response_body.body.decode("utf-8", "surrogateescape"))
                else:
                    t0 = self.monotonic()
                    resp, counted = self.handle_response_body(req, qos, stream, buffered)
                    resp_spent += self.monotonic() - t0
                    # handle_response.go:100-106: once per stream, on the end-of-stream message that completed it
                    if not completed and counted and req.response_body.end_of_stream and qos[0] >= 0:
                        self.metrics.record_resp_processing(*self._labels(qos), resp_spent)
                    completed = completed or counted
                self._record_request(qos, start, status)  # gateway.go:129: every response-body message
            else:
                resp = PB["ProcessingResponse"]()
            yield resp

    # ---- live configuration: the names (routing headers, error bodies, metric labels) follow the table generations
    def names_of(self, gen):
        """the name tables of the generation a decision was made on (qos / token indices are positional in ITS tables)"""
        return self._names.get(int(gen), self.tables) if gen is not None else self.tables

    def publish_names(self, gen: int, tables):
        self._names[int(gen)] = tables
        self.tables = tables
        for g in sorted(self._names)[:-abi.GEN_HISTORY]:  # as many as the library re-maps responses for
            del self._names[g]

    def publisher(self, gateway):
        """`publish` for arks_b200.provider.ArksProvider: the generation is built on the provider's thread
        (arks_config_prepare), swapped in on the batch thread between two batches, and the names change with it"""
        if isinstance(self.batcher, CompiledBatcher):
            def publish(names):
                self.batcher.b.apply_config(names)  # Batcher::ApplyConfig: build here, swap between two cycles
                self.publish_names(gateway.generation, names)
            return publish

        def publish(names):
            prepared = gateway.config_prepare()

            def swap():
                gateway.commit_tables((prepared[0], names))
                self.publish_names(gateway.generation, names)
            self.batcher.between_batches(swap)
        return publish

    def _labels(self, qos):
        t = self.names_of(qos[1])
        q = qos[0]
        tok = int(t.qos_token[q])
        return t.token_namespace[tok], t.token_user[tok], t.qos_model_name[q]

    def _record_request(self, qos, start, status):
        if qos[0] >= 0:  # the reference dereferences a nil qos here when the request phase never resolved one
            self.metrics.record_request(*self._labels(qos), self.monotonic() - start, status)

    # ---- HandleRequestHeaders, handle_request.go:33-81
    def handle_request_headers(self, req):
        hs = [(h.key, h.raw_value or h.value.encode()) for h in req.request_headers.headers.headers]
        token = self.extract_bearer(hs)
        if not token:
            st, h, v, m = replies.request_error_reply(abi.R_NO_TOKEN, 0, 0, 0, 0, self.tables, -1, b"", "")
            return error_response(st, h, v, m), b""
        r = PB["ProcessingResponse"]()
        r.request_headers.response.header_mutation.CopyFrom(_set_headers([(H_WENT_REQ, "true")]))
        r.request_headers.response.clear_route_cache = True
        return r, token

    # ---- HandleRequestBody, handle_request.go:83-249 (decision comes from the engine)
    def handle_request_body(self, req, token):
        """-> (reply, (qos, gen), RESP_* flags of the stream's chunks, rate-limit headers for the response headers)"""
        body = bytes(req.request_body.body)
        out = self.batcher.request(body, token)
        reason = int(out["reason"])
        rl = replies.ratelimit_headers(reason, int(out["detail"]), int(out["qos"]), int(out.get("now", 0)), out.get("rl_entry"),
                                       out.get("rl_limit"), out.get("rl_remaining"), self.names_of(out.get("gen")),
                                       out.get("rl_reset"), out.get("rl_retry"))
        if reason != abi.R_OK:
            ml = int(out.get("model_len", 0))
            raw = body[int(out.get("model_off", 0)):int(out.get("model_off", 0)) + (ml & 0x7FFFFFFF)]
            st, h, v, m = replies.request_error_reply(reason, int(out["detail"]), int(out["cur_usage"]), int(out["limit_max"]),
                                                      int(out.get("now", 0)), self.names_of(out.get("gen")), int(out["qos"]), token,
                                                      replies.decode_model(raw, bool(ml >> 31)), out.get("rl_retry"))
            r = error_response(st, h, v, m)
            r.immediate_response.headers.MergeFrom(_set_headers(rl))  # behind x-error-* and Content-Type
            return r, (-1, None), False, []
        t = self.names_of(out.get("gen"))
        q, tok = int(out["qos"]), int(out["token"])
        r = PB["ProcessingResponse"]()
        r.request_body.response.header_mutation.CopyFrom(_set_headers([
            ("model", t.qos_model_name[q]), ("namespace", t.token_namespace[tok]), ("username", t.token_user[tok])]))
        # a stream's response flags: RESP_METERED rides on every chunk of a stream admitted with FLAG_METERED (N5)
        fl = int(out["flags"])
        return r, (q, out.get("gen")), (abi.RESP_STREAM | (abi.RESP_METERED if fl & abi.FLAG_METERED else 0)) if fl & 1 else 0, rl

    # ---- HandleResponseHeaders, handle_response.go:37-78
    def handle_response_headers(self, req, rl=()):
        """`rl`: the stream's rate-limit headers (handle_request_body). They replace any upstream header of the same name,
        except on an upstream 500, whose reply keeps the reference's headers"""
        pairs, status = [(H_WENT_RESP, "true")], 0
        for h in req.response_headers.headers.headers:
            v = h.raw_value or h.value.encode()
            if h.key == ":status":
                try:
                    status = int(v)
                except ValueError:
                    status = 0
            pairs.append((h.key, v))
        if rl and status != 500:
            ours = {k for k, _ in rl}
            pairs = [(k, v) for k, v in pairs if k.lower() not in ours] + list(rl)
        r = PB["ProcessingResponse"]()
        r.response_headers.response.header_mutation.CopyFrom(_set_headers(pairs))
        r.response_headers.response.clear_route_cache = True
        return r, status

    # ---- HandleResponseBody, handle_response.go:80-268
    def handle_response_body(self, req, qos, stream, buffered):
        """`stream`: 0, or the RESP_* flags of the stream's chunks (handle_request_body)"""
        body, eos = bytes(req.response_body.body), req.response_body.end_of_stream
        qos, gen = qos
        if stream:
            out = self.batcher.response(body, qos, stream, gen)
        else:
            buffered += body  # requestBuffers, handle_response.go:134-155
            if not eos:
                r = PB["ProcessingResponse"]()
                r.response_body.response.SetInParent()
                return r, False
            out = self.batcher.response(bytes(buffered), qos, abi.RESP_END_OF_STREAM, gen)
        reason = int(out["reason"])
        if reason not in (abi.R_OK, abi.R_PENDING, abi.R_QOS_GONE):
            return error_response(*replies.response_error_reply(reason, self.names_of(gen), qos, body)), False
        r = PB["ProcessingResponse"]()
        r.response_body.response.header_mutation.SetInParent()
        return r, bool(out.get("counted", 0))


def serve(server: ExtProcServer, port: int = 50052, max_workers: int = 64, host: str = "127.0.0.1"):
    """grpc.NewServer() + RegisterExternalProcessorServer (gateway.go:175-192); plaintext, default options."""
    import grpc
    handler = grpc.method_handlers_generic_handler(SERVICE, {
        "Process": grpc.stream_stream_rpc_method_handler(
            server.Process, request_deserializer=PB["ProcessingRequest"].FromString,
            response_serializer=PB["ProcessingResponse"].SerializeToString)})
    hs = HealthServer()  # healthPb.RegisterHealthServer, gateway.go:179
    HP = HEALTH_PB
    health = grpc.method_handlers_generic_handler(HEALTH_SERVICE, {
        "Check": grpc.unary_unary_rpc_method_handler(hs.Check, request_deserializer=HP["HealthCheckRequest"].FromString,
                                                     response_serializer=HP["HealthCheckResponse"].SerializeToString),
        "List": grpc.unary_unary_rpc_method_handler(hs.List, request_deserializer=HP["HealthListRequest"].FromString,
                                                    response_serializer=HP["HealthListResponse"].SerializeToString),
        "Watch": grpc.unary_stream_rpc_method_handler(hs.Watch, request_deserializer=HP["HealthCheckRequest"].FromString,
                                                      response_serializer=HP["HealthCheckResponse"].SerializeToString)})
    s = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers))
    s.add_generic_rpc_handlers((handler, health))
    bound = s.add_insecure_port(f"{host}:{port}")
    s.start()
    return s, bound


def serve_metrics(render, port: int = 9110, host: str = "127.0.0.1"):
    """the /metrics listener (gateway.go:158-173): `render()` returns the Prometheus text exposition (metrics.exposition of
    the device rows + HostMetrics.exposition of the wall-clock series)"""
    from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer

    class H(BaseHTTPRequestHandler):
        def do_GET(self):
            ok = self.path.split("?", 1)[0] == "/metrics"
            body = render().encode() if ok else b"404 page not found\n"
            self.send_response(200 if ok else 404)
            self.send_header("Content-Type", "text/plain; version=0.0.4; charset=utf-8" if ok else "text/plain; charset=utf-8")
            self.send_header("Content-Length", str(len(body)))
            self.end_headers()
            self.wfile.write(body)

        def log_message(self, *a):
            pass

    httpd = ThreadingHTTPServer((host, port), H)
    threading.Thread(target=httpd.serve_forever, daemon=True).start()
    return httpd, httpd.server_address[1]


def gracefully_shutdown(grpc_server=None, http_server=None, metrics_server=None, timeout_s: float = 5.0):
    """Server.GracefullyShutdown (gateway.go:194-259): the three listeners stop in parallel; the gRPC server stops accepting
    streams and lets the ones in flight finish, and is cut off when the deadline passes. Returns the list of errors (empty:
    "All servers shutdown successfully")."""
    errors, threads = [], []

    def stop_http(srv, what):
        try:
            srv.shutdown()
            srv.server_close()
        except Exception as e:  # noqa: BLE001
            errors.append(f"{what} server shutdown error: {e}")

    for srv, what in ((http_server, "HTTP"), (metrics_server, "Metrics")):
        if srv is not None:
            threads.append(threading.Thread(target=stop_http, args=(srv, what)))
    if grpc_server is not None:
        def stop_grpc():
            done = grpc_server.stop(timeout_s)  # GracefulStop with the context's deadline: then Stop()
            if not done.wait(timeout_s + 1.0):
                errors.append("gRPC server shutdown timeout")
        threads.append(threading.Thread(target=stop_grpc))
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    return errors


def client_stub(port: int):
    import grpc
    ch = grpc.insecure_channel(f"127.0.0.1:{port}")
    return ch, ch.stream_stream(f"/{SERVICE}/Process", request_serializer=PB["ProcessingRequest"].SerializeToString,
                                response_deserializer=PB["ProcessingResponse"].FromString)
