"""ctypes mirror of include/arks_gateway.h (structs, enums) plus numpy packers for the flat SoA buffers.

Shared by the product wrapper (arks_b200.gateway) and the test-only oracle wrapper (tests/orklib.py).
Nothing here computes decisions; it only lays bytes out the way the C ABI documents.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

# enum arks_rule / arks_quota_type  (rate_limiter.go:31-68, arksquota_types.go:28-33 of the reference; "cost" is this
# project's: spend at the endpoints' prices, include/arks_gateway.h ARKS_QT_COST)
RULES = {"rpm": 0, "rpd": 1, "tpm": 2, "tpd": 3}
RULE_NAMES = ["rpm", "rpd", "tpm", "tpd"]
QUOTA_TYPES = {"prompt": 0, "response": 1, "total": 2, "cost": 3}
QT_COST = QUOTA_TYPES["cost"]
QUOTA_NONE, QUOTA_MISSING = -1, -2
GEN_HISTORY = 16  # ARKS_GEN_HISTORY: generations a response row can be re-mapped from

# enum arks_reason
(R_OK, R_NO_TOKEN, R_REQUEST_BODY, R_NO_MODEL, R_TOKEN_NOT_FOUND, R_MODEL_NOT_IN_TOKEN, R_NO_MODEL_BACKENDS,
 R_STREAM_OPTIONS, R_RATE_LIMIT, R_QUOTA, R_QUOTA_CONFIG, R_STREAMING, R_RESPONSE_UNMARSHAL, R_RESPONSE_UNKNOWN,
 R_QUOTA_CONFIG_RESP, R_PENDING, R_QOS_GONE) = range(17)

# (http status, x-error-* header) per reason — pkg/gateway/types.go:24-56 and the status map of SURVEY.md §8a
REASON_HTTP = {
    R_OK: (200, None),
    R_NO_TOKEN: (401, "x-error-token"),
    R_REQUEST_BODY: (400, "x-error-request-body-processing"),
    R_NO_MODEL: (400, "x-error-no-model-in-request"),
    R_TOKEN_NOT_FOUND: (500, "x-error-token"),
    R_MODEL_NOT_IN_TOKEN: (500, "x-error-token"),
    R_NO_MODEL_BACKENDS: (400, "x-error-no-model-backends"),
    R_STREAM_OPTIONS: (400, "x-error-no-stream-options-include-usage"),
    R_RATE_LIMIT: (429, "x-error-rate-limit"),
    R_QUOTA: (429, "x-error-quota"),
    R_QUOTA_CONFIG: (500, "x-error-quota"),
    R_STREAMING: (500, "x-error-streaming"),
    R_RESPONSE_UNMARSHAL: (500, "x-error-response-unmarshal"),
    R_RESPONSE_UNKNOWN: (500, "x-error-response-unknown"),
    R_QUOTA_CONFIG_RESP: (500, "x-error-quota"),
    R_PENDING: (200, None),
    R_QOS_GONE: (200, None),  # nothing billed; the stream continues (include/arks_gateway.h)
}

RESP_STREAM, RESP_END_OF_STREAM, RESP_COMPLETED = 1, 2, 4
RESP_METERED = 8    # a chunk of a metered stream (N5, arks_set_stream_metering); with RESP_STREAM
FLAG_METERED = 2    # arks_request_result.flags: admitted and metered; the host sets RESP_METERED on its chunks
# metric row layout (include/arks_gateway.h ARKS_METRIC_*)
METRIC_COLS, METRIC_HITS, METRIC_USAGE, METRIC_HIST_IN, METRIC_HIST_OUT, METRIC_HIST_BUCKETS, METRIC_MESSAGES = 44, 0, 4, 6, 24, 18, 42

E_INVALID_ARG, E_NO_DEVICE, E_CUDA, E_TIME_WENT_BACK, E_BAD_TABLE, E_CAPACITY, E_NOT_LOADED = -1, -2, -3, -4, -5, -6, -7

u8p, u32p, i32p, i64p, u64p = (C.POINTER(t) for t in (C.c_uint8, C.c_uint32, C.c_int32, C.c_int64, C.c_uint64))


class ArksTables(C.Structure):
    _fields_ = [
        ("str_bytes", u8p), ("str_off", u32p), ("n_str", C.c_uint32),
        ("n_tokens", C.c_uint32), ("tok_token_str", u32p), ("tok_ns_str", u32p), ("tok_name_str", u32p),
        ("tok_qos_off", u32p),
        ("n_qos", C.c_uint32), ("qos_model_str", u32p), ("qos_quota", i32p), ("qos_rl_off", u32p),
        ("n_rl", C.c_uint32), ("rl_rule", u8p), ("rl_value", i64p),
        ("n_quotas", C.c_uint32), ("quota_ns_str", u32p), ("quota_name_str", u32p), ("quota_item_off", u32p),
        ("n_qitems", C.c_uint32), ("qitem_type", u8p), ("qitem_value", i64p),
        ("n_endpoints", C.c_uint32), ("ep_ns_str", u32p), ("ep_name_str", u32p), ("ep_backend_off", u32p),
        ("n_backends", C.c_uint32), ("backend_weight", i32p),
    ]


class ArksQosSpec(C.Structure):  # arks_qos_spec: one spec.qos[] entry of arks_upsert_token
    _fields_ = [("model", C.c_char_p), ("model_len", C.c_uint32), ("quota", C.c_char_p), ("quota_len", C.c_uint32),
                ("n_rl", C.c_uint32), ("rl_rule", u8p), ("rl_value", i64p)]


class ArksRequestBatch(C.Structure):
    _fields_ = [("n", C.c_uint32), ("bodies", u8p), ("body_off", u32p), ("body_len", u32p),
                ("bodies_bytes", C.c_uint64), ("tokens", u8p), ("token_off", u32p), ("pick_rand", u64p),
                ("now_unix", C.c_int64)]


class ArksRequestResult(C.Structure):
    _fields_ = [("reason", u8p), ("detail", u8p), ("flags", u8p), ("qos", i32p), ("token", i32p), ("pick", i32p),
                ("cur_usage", i64p), ("limit_max", i64p), ("model_off", u32p), ("model_len", u32p), ("bpe_count", u32p),
                ("rl_entry", u8p), ("rl_limit", i64p), ("rl_remaining", i64p), ("rl_reset", u32p), ("rl_retry", u32p)]


RL_NONE = 0xFF  # ARKS_RL_NONE: no rate-limit figure of that kind (arks_set_ratelimit_report)


class ArksResponseBatch(C.Structure):
    _fields_ = [("n", C.c_uint32), ("bodies", u8p), ("body_off", u32p), ("body_len", u32p),
                ("bodies_bytes", C.c_uint64), ("qos", i32p), ("flags", u8p), ("now_unix", C.c_int64), ("gen", u32p),
                ("precharged", u32p)]


class ArksResponseResult(C.Structure):
    _fields_ = [("reason", u8p), ("counted", u8p), ("usage", i64p), ("bpe_count", u32p)]


def ptr(a: np.ndarray, ty):
    """ctypes pointer into a C-contiguous numpy array (the array must outlive the call)."""
    if a is None:
        return C.cast(None, ty)
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ty)


def pack_blobs(blobs, align: int = 32):
    """Concatenate byte strings with every start aligned to `align`; returns (buf, off, len). The ABI requires 16; bodies that
    start on 32-byte boundaries are read a whole 32-byte sector at a time by the fast path (tests also pack with 16)."""
    n = len(blobs)
    lens = np.fromiter((len(b) for b in blobs), dtype=np.uint32, count=n)
    padded = (lens.astype(np.uint64) + (align - 1)) // align * align
    off = np.zeros(n, dtype=np.uint64)
    if n:
        off[1:] = np.cumsum(padded)[:-1]
    total = int(padded.sum()) if n else 0
    buf = np.zeros(max(total, align), dtype=np.uint8)
    mv = memoryview(buf)
    for i, b in enumerate(blobs):
        o = int(off[i])
        mv[o:o + len(b)] = b
    return buf, off.astype(np.uint32), lens


def pack_concat(blobs):
    """Plain concatenation with n+1 offsets (bearer tokens)."""
    n = len(blobs)
    off = np.zeros(n + 1, dtype=np.uint32)
    if n:
        off[1:] = np.cumsum(np.fromiter((len(b) for b in blobs), dtype=np.uint64, count=n))
    buf = np.frombuffer(b"".join(blobs) + b"\0", dtype=np.uint8).copy()
    return buf, off


@dataclass
class RequestBatch:
    """Host-side request micro-batch: what the Go batcher goroutine would assemble (INTEGRATION.md §2)."""
    bodies: np.ndarray
    body_off: np.ndarray
    body_len: np.ndarray
    tokens: np.ndarray
    token_off: np.ndarray
    now_unix: int
    pick_rand: np.ndarray | None = None

    @property
    def n(self) -> int:
        return int(self.body_len.shape[0])

    @classmethod
    def from_lists(cls, bodies, tokens, now_unix, pick_rand=None):
        bb, bo, bl = pack_blobs(bodies)
        tb, to = pack_concat(tokens)
        pr = None if pick_rand is None else np.ascontiguousarray(pick_rand, dtype=np.uint64)
        return cls(bb, bo, bl, tb, to, int(now_unix), pr)

    def c_struct(self) -> ArksRequestBatch:
        return ArksRequestBatch(self.n, ptr(self.bodies, u8p), ptr(self.body_off, u32p), ptr(self.body_len, u32p),
                                int(self.bodies.shape[0]), ptr(self.tokens, u8p), ptr(self.token_off, u32p),
                                ptr(self.pick_rand, u64p), self.now_unix)


@dataclass
class RequestResult:
    reason: np.ndarray
    detail: np.ndarray
    flags: np.ndarray
    qos: np.ndarray
    token: np.ndarray
    pick: np.ndarray
    cur_usage: np.ndarray
    limit_max: np.ndarray
    model_off: np.ndarray = None
    model_len: np.ndarray = None
    bpe_count: np.ndarray = None
    # rate-limit report (arks_set_ratelimit_report): [n, 2] each, column 0 the requests figure, 1 the tokens figure
    rl_entry: np.ndarray = None
    rl_limit: np.ndarray = None
    rl_remaining: np.ndarray = None
    # sliding window with the report (arks_set_sliding_window): rl_reset [n, 2] like the figures, rl_retry [n]
    rl_reset: np.ndarray = None
    rl_retry: np.ndarray = None

    @classmethod
    def empty(cls, n, report: bool = False, sliding: bool = False):
        r = cls(np.full(n, 255, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.full(n, -9, np.int32),
                np.full(n, -9, np.int32), np.full(n, -9, np.int32), np.zeros(n, np.int64), np.zeros(n, np.int64),
                np.full(n, 0xEEEEEEEE, np.uint32), np.full(n, 0xEEEEEEEE, np.uint32), np.full(n, 0xEEEEEEEE, np.uint32))
        if report:
            r.rl_entry = np.full((n, 2), 0xEE, np.uint8)
            r.rl_limit = np.full((n, 2), -9, np.int64)
            r.rl_remaining = np.full((n, 2), -9, np.int64)
            if sliding:
                r.rl_reset = np.full((n, 2), 0xEEEEEEEE, np.uint32)
                r.rl_retry = np.full(n, 0xEEEEEEEE, np.uint32)
        return r

    def c_struct(self) -> ArksRequestResult:
        return ArksRequestResult(ptr(self.reason, u8p), ptr(self.detail, u8p), ptr(self.flags, u8p),
                                 ptr(self.qos, i32p), ptr(self.token, i32p), ptr(self.pick, i32p),
                                 ptr(self.cur_usage, i64p), ptr(self.limit_max, i64p), ptr(self.model_off, u32p),
                                 ptr(self.model_len, u32p), ptr(self.bpe_count, u32p), ptr(self.rl_entry, u8p),
                                 ptr(self.rl_limit, i64p), ptr(self.rl_remaining, i64p), ptr(self.rl_reset, u32p),
                                 ptr(self.rl_retry, u32p))

    def report(self):
        """the rate-limit report columns, or {} when the result was not asked for them"""
        if self.rl_entry is None:
            return {}
        out = {"rl_entry": self.rl_entry, "rl_limit": self.rl_limit, "rl_remaining": self.rl_remaining}
        if self.rl_reset is not None:
            out.update(rl_reset=self.rl_reset, rl_retry=self.rl_retry)
        return out

    def fields(self):
        """the arrays the reference's decision determines (bpe_count has its own oracle: tests/test_bpe.py)"""
        return {k: getattr(self, k) for k in
                ("reason", "detail", "flags", "qos", "token", "pick", "cur_usage", "limit_max", "model_off", "model_len")}

    def model_bytes(self, batch, i: int) -> bytes:
        """raw bytes of request i's `model` string inside its body (escapes not decoded)"""
        o = int(batch.body_off[i]) + int(self.model_off[i])
        return bytes(batch.bodies[o:o + (int(self.model_len[i]) & 0x7FFFFFFF)])


@dataclass
class ResponseBatch:
    bodies: np.ndarray
    body_off: np.ndarray
    body_len: np.ndarray
    qos: np.ndarray
    flags: np.ndarray
    now_unix: int
    gen: np.ndarray | None = None  # table generation of each row's request (None: the current one)
    precharged: np.ndarray | None = None  # N4: what the request phase charged the token-type rules for each row's stream

    @property
    def n(self) -> int:
        return int(self.body_len.shape[0])

    @classmethod
    def from_lists(cls, bodies, qos, flags, now_unix, gen=None):
        bb, bo, bl = pack_blobs(bodies)
        return cls(bb, bo, bl, np.ascontiguousarray(qos, dtype=np.int32), np.ascontiguousarray(flags, dtype=np.uint8),
                   int(now_unix), None if gen is None else np.ascontiguousarray(gen, dtype=np.uint32))

    def c_struct(self) -> ArksResponseBatch:
        return ArksResponseBatch(self.n, ptr(self.bodies, u8p), ptr(self.body_off, u32p), ptr(self.body_len, u32p),
                                 int(self.bodies.shape[0]), ptr(self.qos, i32p), ptr(self.flags, u8p), self.now_unix,
                                 ptr(self.gen, u32p), ptr(self.precharged, u32p))


@dataclass
class ResponseResult:
    reason: np.ndarray
    counted: np.ndarray
    usage: np.ndarray
    bpe_count: np.ndarray = None

    @classmethod
    def empty(cls, n):
        return cls(np.full(n, 255, np.uint8), np.full(n, 255, np.uint8), np.full((n, 3), -7, np.int64),
                   np.full(n, 0xEEEEEEEE, np.uint32))

    def c_struct(self) -> ArksResponseResult:
        return ArksResponseResult(ptr(self.reason, u8p), ptr(self.counted, u8p), ptr(self.usage, i64p), ptr(self.bpe_count, u32p))

    def fields(self):
        return {"reason": self.reason, "counted": self.counted, "usage": self.usage}
