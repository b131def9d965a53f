"""ctypes wrapper around the TEST-ONLY host build of the device state machines (tests/host_machine.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_machine.cpp")
HDRS = [os.path.join(ROOT, "arks_b200", "csrc", f) for f in ("json_common.cuh", "json_engine.cuh", "json_tables.h", "mask_scan.cuh", "warp_scan.cuh", "bpe.cuh", "config_store.h")] + [os.path.join(ROOT, "include", "arks_gateway.h")]
OUT = os.path.join(ROOT, "tests", "_build", "libhost_machine.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        os.makedirs(os.path.dirname(OUT), exist_ok=True)
        if not os.path.exists(OUT) or max([os.path.getmtime(SRC)] + [os.path.getmtime(h) for h in HDRS]) > os.path.getmtime(OUT):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", OUT, SRC])
        L = C.CDLL(OUT)
        i64p = C.POINTER(C.c_int64)
        L.hm_parse_request.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t),
                                       C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
        L.hm_parse_response.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), i64p]
        L.hm_parse_sse.argtypes = [C.c_char_p, C.c_size_t, i64p]
        L.hm_parse_sse_split.argtypes = [C.c_char_p, C.c_size_t, i64p]
        u32p = C.POINTER(C.c_uint32)
        ip = C.POINTER(C.c_int)
        L.hm_fast_request.argtypes = [C.c_char_p, C.c_size_t, u32p, ip, ip, ip]
        L.hm_engine_request_span.argtypes = [C.c_char_p, C.c_size_t, u32p, ip, ip, ip]
        L.hm_fast_response.argtypes = [C.c_char_p, C.c_size_t, u32p, i64p]
        L.hm_engine_response_span.argtypes = [C.c_char_p, C.c_size_t, u32p, i64p]
        L.hm_warp_request.argtypes = [C.c_char_p, C.c_size_t, u32p, ip, ip, ip]
        L.hm_warp_response.argtypes = [C.c_char_p, C.c_size_t, u32p, i64p]
        L.hm_bpe_load.argtypes = [u32p, C.c_uint32, u32p, u32p, u32p, C.POINTER(C.c_uint8), C.c_uint32]
        L.hm_bpe_count.argtypes = [C.c_char_p, C.c_size_t]
        L.hm_bpe_count.restype = C.c_uint32
        L.hm_bpe_pretokenize.argtypes = [C.c_char_p, C.c_size_t, u32p, C.c_int]
        L.hm_set_past_end.argtypes = [C.c_size_t]
        L.hm_work_profile.argtypes = [C.c_int, C.c_char_p, C.c_size_t, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_size_t]
        vp, cp, u32 = C.c_void_p, C.c_char_p, C.c_uint32
        L.hm_store_new.restype = vp
        L.hm_store_free.argtypes = [vp]
        L.hm_store_upsert_token.argtypes = [vp, cp, u32, cp, u32, cp, u32, vp, u32]
        L.hm_store_upsert_quota.argtypes = [vp, cp, u32, cp, u32, C.POINTER(C.c_uint8), i64p, u32]
        L.hm_store_upsert_endpoint.argtypes = [vp, cp, u32, cp, u32, C.POINTER(C.c_int32), u32]
        L.hm_store_erase.argtypes = [vp, C.c_int, cp, u32, cp, u32]
        L.hm_store_flatten.argtypes = [vp]
        L.hm_store_flatten.restype = vp
        L.hm_tables_shape_error.argtypes = [vp]
        L.hm_tables_shape_error.restype = C.c_char_p
        _lib = L
    return _lib


def _past(body: bytes, past: bytes) -> bytes:
    """the buffer a host driver is handed: the document, then `past`, the bytes it finds behind the document's end (the
    device reads the padding, the next body or stale staging memory there); without `past`, the drivers' fixed fills"""
    lib().hm_set_past_end(len(past))
    return body + past


def parse_request_body(body: bytes, past: bytes = b""):
    buf = C.create_string_buffer(4096)
    ml, st, so, iu = C.c_size_t(), C.c_int(), C.c_int(), C.c_int()
    rc = lib().hm_parse_request(_past(body, past), len(body), buf, 4096, C.byref(ml), C.byref(st), C.byref(so), C.byref(iu))
    return rc, buf.raw[:min(ml.value, 4096)], st.value, so.value, iu.value


def parse_response_body(body: bytes, past: bytes = b""):
    ne = C.c_size_t()
    u = np.zeros(3, np.int64)
    rc = lib().hm_parse_response(_past(body, past), len(body), C.byref(ne), u.ctypes.data_as(C.POINTER(C.c_int64)))
    return rc, ne.value, tuple(int(x) for x in u)


def parse_sse_chunk(body: bytes, past: bytes = b""):
    u = np.zeros(3, np.int64)
    rc = lib().hm_parse_sse(_past(body, past), len(body), u.ctypes.data_as(C.POINTER(C.c_int64)))
    return rc, tuple(int(x) for x in u)


def parse_sse_chunk_split(body: bytes, past: bytes = b""):
    """the event-parallel path of the SSE kernel (SseSplit + one JsonT per event); third item: fell back to SseT"""
    u = np.zeros(3, np.int64)
    rc = lib().hm_parse_sse_split(_past(body, past), len(body), u.ctypes.data_as(C.POINTER(C.c_int64)))
    return rc & 1, tuple(int(x) for x in u), bool(rc & 2)


def set_evsync(mode):
    """schedule for JsonT documents: 0 / False consume_t, 1 / True consume_evsync, 4 or 8 consume_rounds<R>"""
    lib().hm_set_evsync(int(mode))


def work_profile(body: bytes, kind: int = 0):
    """(advances, events) per 128-byte window of one request (kind 0) / response (kind 1) body, as the schedules count them"""
    n = (len(body) + 127) // 128
    a = np.zeros(max(n, 1), np.uint32)
    e = np.zeros(max(n, 1), np.uint32)
    u32p = C.POINTER(C.c_uint32)
    rc = lib().hm_work_profile(kind, body, len(body), a.ctypes.data_as(u32p), e.ctypes.data_as(u32p), len(a))
    assert rc >= 0
    return a[:n], e[:n]


def _req(fn, body, past):
    span = (C.c_uint32 * 3)()
    st, so, iu = C.c_int(), C.c_int(), C.c_int()
    ok = fn(_past(body, past), len(body), span, C.byref(st), C.byref(so), C.byref(iu))
    return (tuple(span), st.value, so.value, iu.value) if ok else None


def _resp(fn, body, past):
    span = (C.c_uint32 * 3)()
    u = (C.c_int64 * 3)()
    ok = fn(_past(body, past), len(body), span, u)
    return (tuple(span), tuple(u)) if ok else None


def fast_request(body: bytes, past: bytes = b""):
    """the fast path (host driver of mask_scan.cuh = one lane's work): ((start, rawlen, esc), stream3, so_present, iu3) or
    None when the document is left to the exact engine"""
    return _req(lib().hm_fast_request, body, past)


def engine_request(body: bytes, past: bytes = b""):
    """the exact engine in the same terms, None when it rejects the document"""
    return _req(lib().hm_engine_request_span, body, past)


def fast_response(body: bytes, past: bytes = b""):
    return _resp(lib().hm_fast_response, body, past)


def engine_response(body: bytes, past: bytes = b""):
    return _resp(lib().hm_engine_response_span, body, past)


def bpe_load(tables):
    """tables: arks_b200.bpe.BpeTables"""
    t = tables.c_struct()
    lib().hm_bpe_load(t.byte_id, t.n_merges, t.left, t.right, t.merged, t.cp_class, t.flags)
    lib()._bpe_keep = tables


def tables_shape_error(c_tables):
    """c_tables: a ctypes arks_tables (arks_b200.tables.Tables.c_struct()); None when well formed, else the complaint"""
    e = lib().hm_tables_shape_error(C.cast(C.pointer(c_tables), C.c_void_p))
    return e.decode() if e else None


def bpe_probes():
    """since the last call: slots read in the hot (shared-memory) table, in the full table, pieces, decoded text bytes"""
    out = (C.c_ulonglong * 4)()
    lib().hm_bpe_probes(out)
    return [int(x) for x in out]


def bpe_count(body: bytes, past: bytes = b"") -> int:
    return int(lib().hm_bpe_count(_past(body, past), len(body)))


def bpe_pretokenize(text: bytes):
    cap = len(text) + 1
    ends = (C.c_uint32 * cap)()
    n = lib().hm_bpe_pretokenize(text, len(text), ends, cap)
    return list(ends[:n])


def warp_request(body: bytes, past: bytes = b""):
    """the warp-per-document latency path (host driver of warp_scan.cuh), same convention as fast_request"""
    return _req(lib().hm_warp_request, body, past)


def warp_response(body: bytes, past: bytes = b""):
    return _resp(lib().hm_warp_response, body, past)


class ConfigStore:
    """arks::ConfigStore (csrc/config_store.h) driven with CRD-shaped dicts; flatten() -> an object with c_struct() the oracle takes"""

    def __init__(self):
        self.h = lib().hm_store_new()

    def __del__(self):
        if getattr(self, "h", None):
            lib().hm_store_free(self.h)
            self.h = None

    @staticmethod
    def _k(obj):
        md = obj["metadata"]
        return md.get("namespace", "default").encode(), md["name"].encode()

    def upsert(self, kind, obj):
        from arks_b200 import abi
        ns, nm = self._k(obj)
        if kind == "token":
            qos = obj["spec"].get("qos") or []
            specs = (abi.ArksQosSpec * max(1, len(qos)))()
            keep = []
            for i, q in enumerate(qos):
                m = q["arksEndpoint"]["name"].encode()
                qn = ((q.get("quota") or {}).get("name", "") or "").encode()
                rls = q.get("rateLimits") or []
                rr = np.array([abi.RULES[r["type"]] for r in rls], np.uint8)
                rv = np.array([int(r["value"]) for r in rls], np.int64)
                keep += [m, qn, rr, rv]
                specs[i] = abi.ArksQosSpec(m, len(m), qn, len(qn), len(rls), abi.ptr(rr, abi.u8p), abi.ptr(rv, abi.i64p))
            tk = obj["spec"]["token"].encode()
            lib().hm_store_upsert_token(self.h, ns, len(ns), nm, len(nm), tk, len(tk), C.cast(specs, C.c_void_p), len(qos))
        elif kind == "quota":
            items = obj["spec"]["quotas"]
            t = np.array([abi.QUOTA_TYPES[i["type"]] for i in items], np.uint8)
            v = np.array([int(i["value"]) for i in items], np.int64)
            lib().hm_store_upsert_quota(self.h, ns, len(ns), nm, len(nm), abi.ptr(t, abi.u8p), abi.ptr(v, abi.i64p), len(items))
        else:
            w = np.array(obj["weights"], np.int32)
            lib().hm_store_upsert_endpoint(self.h, ns, len(ns), nm, len(nm), abi.ptr(w, abi.i32p), len(w))

    def erase(self, kind, obj) -> bool:
        ns, nm = self._k(obj)
        return bool(lib().hm_store_erase(self.h, {"token": 0, "quota": 1, "endpoint": 2}[kind], ns, len(ns), nm, len(nm)))

    def flatten(self):
        from arks_b200 import abi
        p = lib().hm_store_flatten(self.h)
        ts = C.cast(p, C.POINTER(abi.ArksTables)).contents
        store = self

        class View:
            _keep = store

            def c_struct(self):
                return ts
        return View()
