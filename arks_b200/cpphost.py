"""ctypes view of the C++ host library (host/cpp/arks_host.{h,cc}): the compiled micro-batcher and ext_proc stream state
machine that sit above the C ABI where the reference has its Go server. Python only drives it (tests, bench load
generation); the batching, threading and waiting all happen in C++.

`build(against=...)` links the host against a given provider of the C ABI: arks_b200/libarksgw.so (the product) or, in
CPU-only tests, tests/_build/libarksgw_shim.so (the oracle behind the same three entry points)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "host", "cpp", "arks_host.cc")
HDR = os.path.join(ROOT, "host", "cpp", "arks_host.h")
LIB = os.path.join(ROOT, "host", "cpp", "libarkshost.so")


class RequestDecision(C.Structure):
    _fields_ = [("reason", C.c_uint8), ("detail", C.c_uint8), ("flags", C.c_uint8), ("qos", C.c_int32), ("token", C.c_int32),
                ("pick", C.c_int32), ("cur_usage", C.c_int64), ("limit_max", C.c_int64), ("cycle", C.c_uint64),
                ("index", C.c_uint32), ("now_unix", C.c_int64), ("gen", C.c_uint32), ("model_off", C.c_uint32),
                ("model_len", C.c_uint32), ("bpe_count", C.c_uint32),
                # rate-limit report: [0] requests, [1] tokens (rl_entry 0xFF: no such figure)
                ("rl_entry", C.c_uint8 * 2), ("rl_limit", C.c_int64 * 2), ("rl_remaining", C.c_int64 * 2),
                # sliding window with the report: rl_sliding 1, the projected reset [requests, tokens] and retry seconds
                ("rl_reset", C.c_uint32 * 2), ("rl_retry", C.c_uint32), ("rl_sliding", C.c_uint8)]


class ResponseDecision(C.Structure):
    _fields_ = [("reason", C.c_uint8), ("counted", C.c_uint8), ("usage", C.c_int64 * 3), ("cycle", C.c_uint64),
                ("index", C.c_uint32), ("now_unix", C.c_int64)]


class BatcherStats(C.Structure):
    _fields_ = [(k, C.c_uint64) for k in ("cycles", "request_batches", "response_batches", "requests", "responses",
                                          "max_request_batch", "max_response_batch", "ns_submit", "ns_device", "ns_deliver",
                                          "max_ns_submit", "max_ns_device", "max_ns_deliver", "max_ns_gap",
                                          "slow_submit", "slow_device", "slow_deliver", "slow_gap", "ns_fill", "max_ns_fill", "slow_fill", "late_rows")]


REQ_DTYPE = np.dtype(RequestDecision)
RESP_DTYPE = np.dtype(ResponseDecision)
EXPORTED = ["arks_host_create", "arks_host_destroy", "arks_host_set_fixed_clock", "arks_host_request", "arks_host_response",
            "arks_host_stats", "arks_host_run_requests", "arks_host_run_responses", "arks_host_open_loop_requests",
            "arks_host_stream_transcript", "arks_host_load_tables", "arks_host_apply_config", "arks_host_set_precharge", "arks_host_set_ratelimit_report", "arks_host_set_sliding_window", "arks_host_ratelimit_headers", "arks_host_response_pre", "arks_host_set_names", "arks_host_request_error_reply",
            "arks_host_response_error_reply", "arks_host_load_tables_named", "arks_host_apply_config_named",
            "arks_host_response_error_reply_gen"]


def build(out: str = LIB, against: str = None, force: bool = False) -> str:
    """g++ the host library, linked against `against` (default arks_b200/libarksgw.so)."""
    against = against or os.path.join(ROOT, "arks_b200", "libarksgw.so")
    srcs = [SRC, HDR, os.path.join(ROOT, "include", "arks_gateway.h"), against]
    if force or not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        d, f = os.path.split(against)
        assert f.startswith("lib") and f.endswith(".so")
        subprocess.check_call(["g++", "-O2", "-std=c++20", "-shared", "-fPIC", "-pthread", "-Wall", "-o", out, SRC,
                               "-L" + d, "-l" + f[3:-3],
                               "-Wl,-rpath,$ORIGIN/" + os.path.relpath(d, os.path.dirname(out))])  # relocatable with the tree
    return out


def load(path: str = LIB):
    L = C.CDLL(path)
    vp, u8p, u32p = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)
    L.arks_host_create.argtypes = [vp, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(vp)]
    L.arks_host_destroy.argtypes = [vp]
    L.arks_host_destroy.restype = None
    L.arks_host_set_fixed_clock.argtypes = [vp, C.c_int64]
    L.arks_host_set_fixed_clock.restype = None
    L.arks_host_request.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint64, C.POINTER(RequestDecision)]
    L.arks_host_response.argtypes = [vp, C.c_int32, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint8, C.POINTER(ResponseDecision)]
    L.arks_host_load_tables.argtypes = [vp, vp]
    L.arks_host_apply_config.argtypes = [vp]
    L.arks_host_load_tables_named.argtypes = [vp, vp, C.c_char_p, C.c_uint32]
    L.arks_host_apply_config_named.argtypes = [vp, C.c_char_p, C.c_uint32]
    L.arks_host_set_precharge.argtypes = [vp, C.c_int]
    L.arks_host_set_ratelimit_report.argtypes = [vp, C.c_int]
    L.arks_host_set_sliding_window.argtypes = [vp, C.c_int]
    L.arks_host_ratelimit_headers.argtypes = [vp, C.POINTER(RequestDecision), C.c_char_p, C.c_uint32]
    L.arks_host_response_pre.argtypes = [vp, C.c_int32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_uint32, C.c_uint8, C.POINTER(ResponseDecision)]
    L.arks_host_reset_tail.argtypes = [vp]
    L.arks_host_reset_tail.restype = None
    L.arks_host_open_loop_lateness.restype = None
    L.arks_host_open_loop_call_latency.restype = None
    L.arks_host_open_loop_call_latency.argtypes = [vp]
    L.arks_host_set_names.argtypes = [vp, C.c_char_p, C.c_uint32]
    L.arks_host_request_error_reply.argtypes = [vp, C.POINTER(RequestDecision), C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32,
                                                C.c_char_p, C.c_uint32]
    L.arks_host_response_error_reply.argtypes = [vp, C.POINTER(ResponseDecision), C.c_int32, C.c_char_p, C.c_uint32, C.c_char_p,
                                                 C.c_uint32]
    L.arks_host_response_error_reply_gen.argtypes = [vp, C.POINTER(ResponseDecision), C.c_int32, C.c_uint32, C.c_char_p, C.c_uint32,
                                                     C.c_char_p, C.c_uint32]
    L.arks_host_stats.argtypes = [vp, C.POINTER(BatcherStats)]
    L.arks_host_stats.restype = None
    L.arks_host_run_requests.argtypes = [vp, C.c_uint32, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.arks_host_run_requests.restype = C.c_int64
    L.arks_host_run_responses.argtypes = [vp, C.c_uint32, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.arks_host_run_responses.restype = C.c_int64
    L.arks_host_open_loop_requests.argtypes = [vp, C.c_uint32, C.c_double, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]
    L.arks_host_open_loop_requests.restype = C.c_int64
    cpp = C.POINTER(C.c_char_p)
    L.arks_host_stream_transcript.argtypes = [vp, cpp, cpp, C.c_uint32, C.c_char_p,
                                              C.c_uint32, cpp, cpp, C.c_uint32, C.POINTER(C.c_char_p), u32p, C.c_uint32,
                                              C.c_uint64, C.c_char_p, C.c_uint32]
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


class Batcher:
    """arks_host::Batcher over an arks_ctx handle (Gateway._h, or the CPU shim's context in tests)."""

    def __init__(self, lib, ctx_handle, max_batch=4096, max_bytes=16 << 20, linger_us=0, max_inflight=1):
        self.L = lib
        h = C.c_void_p()
        rc = lib.arks_host_create(ctx_handle, max_batch, max_bytes, linger_us, max_inflight, C.byref(h))
        if rc:
            raise RuntimeError(f"arks_host_create: {rc}")
        self._h = h

    def close(self):
        if self._h:
            self.L.arks_host_destroy(self._h)
            self._h = None

    def set_fixed_clock(self, now: int):
        self.L.arks_host_set_fixed_clock(self._h, int(now))

    def request(self, token: bytes, body: bytes, pick_rand: int = 0) -> RequestDecision:
        d = RequestDecision()
        self.L.arks_host_request(self._h, token, len(token), body, len(body), pick_rand, C.byref(d))
        return d

    def response(self, qos: int, body: bytes, flags: int, gen: int = None, precharged: int = 0) -> ResponseDecision:
        """`gen`: RequestDecision.gen of the stream's request; None = the tables have not changed since. `precharged`: its
        RequestDecision.bpe_count while set_precharge(True) is in force (N4)"""
        d = ResponseDecision()
        self.L.arks_host_response_pre(self._h, qos, 0xFFFFFFFF if gen is None else gen, precharged, body, len(body), flags, C.byref(d))
        return d

    def set_precharge(self, on: bool):
        if self.L.arks_host_set_precharge(self._h, int(bool(on))):
            raise RuntimeError("arks_host_set_precharge failed")

    def set_ratelimit_report(self, on: bool):
        """request decisions carry the rate-limit figures and the stream state machine sends x-ratelimit-* / retry-after"""
        if self.L.arks_host_set_ratelimit_report(self._h, int(bool(on))):
            raise RuntimeError("arks_host_set_ratelimit_report failed")

    def set_sliding_window(self, on: bool):
        """the limiter's sliding window (arks_set_sliding_window); with the report on, decisions carry reset / retry times"""
        if self.L.arks_host_set_sliding_window(self._h, int(bool(on))):
            raise RuntimeError("arks_host_set_sliding_window failed")

    def ratelimit_headers(self, d: RequestDecision):
        """[(key, value)] the stream state machine adds for decision `d` (names of its generation)"""
        buf = C.create_string_buffer(4096)
        n = self.L.arks_host_ratelimit_headers(self._h, C.byref(d), buf, len(buf))
        if n < 0:
            raise RuntimeError("reply buffer too small")
        return [tuple(line.split(": ", 1)) for line in buf.raw[:n].decode().splitlines()]

    def load_tables(self, tables):
        """config reload between two cycles (Batcher::LoadTables); the reply-shaping names of the new generation enter the
        host's NameBook under its number before the swap (streams decided earlier keep theirs)"""
        ts = tables.c_struct()
        blob = tables.names_blob()
        rc = self.L.arks_host_load_tables_named(self._h, C.byref(ts), blob, len(blob))
        if rc:
            raise RuntimeError(f"arks_host_load_tables: {rc}")

    def apply_config(self, tables=None):
        """publish the arks_upsert_* / arks_delete_* calls made on the context (Batcher::ApplyConfig); `tables`: the same
        objects as an arks_b200.tables.Tables in (namespace, name) order, for the reply-shaping names"""
        if tables is not None:
            blob = tables.names_blob()
            rc = self.L.arks_host_apply_config_named(self._h, blob, len(blob))
        else:
            rc = self.L.arks_host_apply_config(self._h)
        if rc:
            raise RuntimeError(f"arks_host_apply_config: {rc}")

    def set_names(self, tables):
        blob = tables.names_blob()
        if self.L.arks_host_set_names(self._h, blob, len(blob)):
            raise RuntimeError("arks_host_set_names: malformed name table")

    def _reply(self, n, buf):
        if n < 0:
            raise RuntimeError("reply buffer too small")
        status, header, value, message = buf.raw[:n].decode("utf-8", "surrogateescape").split("\n", 3)
        return int(status), header, value, message

    def request_error_reply(self, d: RequestDecision, token: bytes, body: bytes):
        """(status, x-error header, header value, error message) the reference sends for a failed request decision"""
        buf = C.create_string_buffer(len(body) + len(token) + 4096)
        return self._reply(self.L.arks_host_request_error_reply(self._h, C.byref(d), token, len(token), body, len(body), buf, len(buf)), buf)

    def response_error_reply(self, d: ResponseDecision, qos: int, chunk: bytes, gen: int = None):
        """`gen`: RequestDecision.gen of the stream's request (the generation `qos` is an index of); None: the latest"""
        buf = C.create_string_buffer(len(chunk) + 4096)
        if gen is None:
            return self._reply(self.L.arks_host_response_error_reply(self._h, C.byref(d), qos, chunk, len(chunk), buf, len(buf)), buf)
        return self._reply(self.L.arks_host_response_error_reply_gen(self._h, C.byref(d), qos, gen, chunk, len(chunk), buf, len(buf)), buf)

    def reset_tail(self):
        self.L.arks_host_reset_tail(self._h)

    def open_loop_lateness(self) -> dict:
        """the load generator's own lateness in the last open_loop_requests run (ns)"""
        a = (C.c_int64 * 3)()
        self.L.arks_host_open_loop_lateness(a)
        return {"producer_late_max_us": a[0] / 1e3, "producer_rows_late_100us": int(a[1]), "submit_call_max_us": a[2] / 1e3}

    def stats(self) -> dict:
        s = BatcherStats()
        self.L.arks_host_stats(self._h, C.byref(s))
        return {k: int(getattr(s, k)) for k, _ in BatcherStats._fields_}

    def run_requests(self, batch, threads: int):
        """every row of an abi.RequestBatch as one blocking HandleRequestBody call, issued by `threads` C++ threads.
        Returns (decisions as a structured array in row order, latency_ns per call, wall seconds)."""
        out = np.zeros(batch.n, REQ_DTYPE)
        lat = np.zeros(batch.n, np.int64)
        bodies = np.ascontiguousarray(batch.bodies)
        ns = self.L.arks_host_run_requests(self._h, batch.n, threads, _ptr(bodies), _ptr(batch.body_off), _ptr(batch.body_len),
                                           _ptr(batch.tokens), _ptr(batch.token_off), _ptr(batch.pick_rand), _ptr(out), _ptr(lat))
        return out, lat, ns * 1e-9

    def open_loop_requests(self, batch, rate_per_s: float, producers: int = 4):
        """rows of `batch` ARRIVE at rate_per_s (exponential gaps) through the asynchronous SubmitRequest, whether or not
        earlier ones are answered; latency = decision handed over - scheduled arrival (no coordinated omission)."""
        out = np.zeros(batch.n, REQ_DTYPE)
        lat = np.zeros(batch.n, np.int64)
        # second clock: decision - the moment the generator made the call (a generator thread that the OS kept off its
        # core for milliseconds is late on its own; `lat` still charges that to the request, this array does not)
        self.last_call_latency = np.zeros(batch.n, np.int64)
        # np.zeros hands out untouched pages: the first write to each (from the completion path, inside the timed region,
        # 2 MiB at a time under transparent huge pages) would be charged to the requests that happen to land there
        for a in (out, lat, self.last_call_latency):
            a.view(np.uint8)[:] = 0
        self.L.arks_host_open_loop_call_latency(_ptr(self.last_call_latency))
        bodies = np.ascontiguousarray(batch.bodies)
        ns = self.L.arks_host_open_loop_requests(self._h, batch.n, float(rate_per_s), producers, _ptr(bodies), _ptr(batch.body_off),
                                                 _ptr(batch.body_len), _ptr(batch.tokens), _ptr(batch.token_off),
                                                 _ptr(batch.pick_rand), _ptr(out), _ptr(lat))
        return out, lat, ns * 1e-9

    def run_responses(self, batch, threads: int):
        out = np.zeros(batch.n, RESP_DTYPE)
        lat = np.zeros(batch.n, np.int64)
        bodies = np.ascontiguousarray(batch.bodies)
        ns = self.L.arks_host_run_responses(self._h, batch.n, threads, _ptr(bodies), _ptr(batch.body_off), _ptr(batch.body_len),
                                            _ptr(batch.qos), _ptr(getattr(batch, "gen", None)), _ptr(batch.flags), _ptr(out), _ptr(lat))
        return out, lat, ns * 1e-9

    def stream_transcript(self, req_headers, req_body: bytes, resp_headers, resp_chunks, pick_rand: int = 0) -> str:
        """drive one ext_proc stream through arks_host::StreamProcessor (names: set_names / load_tables)"""
        def arr(strs):
            a = (C.c_char_p * max(len(strs), 1))()
            for i, s in enumerate(strs):
                a[i] = s if isinstance(s, bytes) else s.encode()
            return a
        rk, rv = arr([k for k, _ in req_headers]), arr([v for _, v in req_headers])
        pk, pv = arr([k for k, _ in resp_headers]), arr([v for _, v in resp_headers])
        chunks = (C.c_char_p * max(len(resp_chunks), 1))()
        lens = (C.c_uint32 * max(len(resp_chunks), 1))()
        for i, c in enumerate(resp_chunks):
            chunks[i], lens[i] = c, len(c)
        buf = C.create_string_buffer(1 << 20)
        n = self.L.arks_host_stream_transcript(self._h, rk, rv, len(req_headers),
                                               req_body, len(req_body), pk, pv, len(resp_headers), chunks, lens,
                                               len(resp_chunks), pick_rand, buf, len(buf))
        if n < 0:
            raise RuntimeError("transcript buffer too small")
        return buf.raw[:n].decode("latin1")
