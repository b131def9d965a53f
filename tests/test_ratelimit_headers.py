"""Opt-in rate-limit report (include/arks_gateway.h: arks_set_ratelimit_report): x-ratelimit-{limit,remaining,reset}-{requests,
tokens} on every decided request and retry-after on rate-limit 429s, the figures OpenAI-style clients pace themselves by.

CPU: the oracle's report mode (tests/ratelimit_oracle.c, read from its serial state) on hand-made scenarios with the numbers
written out; the header shaping of both hosts (Go duration strings, window edges); ext_proc transcripts of the C++ stream state
machine over tests/ratelimit_shim.c against the Python server; the switch off adds nothing anywhere.
GPU: limit_admit's closed form (arrival rank, admitted count, duplicate entries) against the oracle's report mode on every scan
path, around the hot-group threshold, across windows, with N4 / N5 on and across a generation swap; the report changes no
decision, counter, metric or launch; the compiled host on the GPU against the Python mirror."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from arks_b200 import abi, cpphost, extproc, replies
from arks_b200.abi import ArksRequestBatch, ArksRequestResult, ArksResponseBatch, ArksResponseResult, ArksTables
from arks_b200.abi import RequestBatch, RequestResult, ResponseBatch, ResponseResult
from arks_b200.extproc import PB
from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
FX = json.load(open(os.path.join(HERE, "golden", "quickstart.json")))
NOW = 1_700_000_000  # 2023-11-14T22:13:20Z: 20 s into its minute, 80 000 s into its day
RESP = FX["response_body"].encode()  # usage total_tokens 45
NONE = abi.RL_NONE


# ---- the oracle with its report mode -------------------------------------------------------------------------------------
def _stale(out, srcs):
    return not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs)


def rl_oracle_path() -> str:
    os.makedirs(BUILD, exist_ok=True)
    out = os.path.join(BUILD, "libarks_oracle_rl.so")
    od = os.path.join(ROOT, "oracle")
    srcs = [os.path.join(HERE, "ratelimit_oracle.c"), os.path.join(ROOT, "include", "arks_gateway.h")] + \
        [os.path.join(od, f) for f in os.listdir(od) if f.endswith((".c", ".h"))]
    if _stale(out, srcs):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-Wl,-Bsymbolic", "-o", out,
                               os.path.join(HERE, "ratelimit_oracle.c"), os.path.join(od, "ork_json.c")])
    return out


_L = None


def rl_lib():
    global _L
    if _L is None:
        L = C.CDLL(rl_oracle_path())
        L.ork_create.restype = C.c_void_p
        L.ork_create.argtypes = [C.POINTER(ArksTables)]
        L.ork_destroy.argtypes = [C.c_void_p]
        L.ork_reload.argtypes = [C.c_void_p, C.POINTER(ArksTables)]
        L.ork_set_ratelimit_report.argtypes = [C.c_void_p, C.c_int]
        L.ork_set_ratelimit_report.restype = None
        L.ork_set_precharge.argtypes = [C.c_void_p, C.c_int]
        L.ork_set_precharge.restype = None
        L.ork_set_estimates.argtypes = [C.c_void_p, abi.u32p, C.c_uint32]
        L.ork_set_estimates.restype = None
        L.ork_request_batch.argtypes = [C.c_void_p, C.POINTER(ArksRequestBatch), C.POINTER(ArksRequestResult)]
        L.ork_response_batch.argtypes = [C.c_void_p, C.POINTER(ArksResponseBatch), C.POINTER(ArksResponseResult)]
        L.ork_snapshot_rate.argtypes = [C.c_void_p, C.c_int64, abi.i64p]
        L.ork_snapshot_metrics.argtypes = [C.c_void_p, abi.i64p]
        _L = L
    return _L


class RlOracle:
    """the oracle with arks_set_ratelimit_report's mode (on unless report=False)"""

    def __init__(self, tables, report=True):
        self.tables, self._ts = tables, tables.c_struct()
        self.h = rl_lib().ork_create(C.byref(self._ts))
        assert self.h
        self.report = report
        rl_lib().ork_set_ratelimit_report(self.h, int(report))

    def __del__(self):
        if getattr(self, "h", None):
            rl_lib().ork_destroy(self.h)
            self.h = None

    def reload(self, tables):
        ts = tables.c_struct()
        assert rl_lib().ork_reload(self.h, C.byref(ts)) == 0
        self.tables, self._ts = tables, ts

    def set_precharge(self, on):
        rl_lib().ork_set_precharge(self.h, int(bool(on)))

    def set_estimates(self, est):
        self._est = np.ascontiguousarray(est, np.uint32)
        rl_lib().ork_set_estimates(self.h, abi.ptr(self._est, abi.u32p), len(self._est))

    def request_batch(self, b):
        r = RequestResult.empty(b.n, report=self.report)
        bs, rs = b.c_struct(), r.c_struct()
        assert rl_lib().ork_request_batch(self.h, C.byref(bs), C.byref(rs)) == 0
        return r

    def response_batch(self, b):
        r = ResponseResult.empty(b.n)
        bs, rs = b.c_struct(), r.c_struct()
        assert rl_lib().ork_response_batch(self.h, C.byref(bs), C.byref(rs)) == 0
        return r

    def snapshot_rate(self, now):
        out = np.zeros((self.tables.n_qos, 4), np.int64)
        rl_lib().ork_snapshot_rate(self.h, int(now), abi.ptr(out, abi.i64p))
        return out

    # the engine surface of extproc.Batcher
    handle_request_body = request_batch
    handle_response_body = response_batch


def reqs(token, n, now, model="qwen-7b", body=None):
    b = body or ('{"model":"%s","messages":[{"role":"user","content":"hi"}]}' % model).encode()
    return RequestBatch.from_lists([b] * n, [token.encode()] * n, now)


def responses(n, now, qos=0):
    return ResponseBatch.from_lists([RESP] * n, [qos] * n, [abi.RESP_END_OF_STREAM] * n, now)


def figs(r, i):
    """(requests figure, tokens figure) of row i as (entry, limit, remaining)"""
    return tuple((int(r.rl_entry[i, t]), int(r.rl_limit[i, t]), int(r.rl_remaining[i, t])) for t in (0, 1))


def quickstart():
    return Tables(FX["tokens"], FX["quotas"], FX["endpoints"])


# ---- 1. the oracle's report mode, numbers by hand ---------------------------------------------------------------------------
def test_oracle_report_quickstart_token():
    """rpm 5, tpm 40 000, rpd 100, tpd 1 000 000 (entries 0..3 in that order)"""
    t = quickstart()
    o = RlOracle(t)
    a = o.request_batch(reqs("sk-test123456", 7, NOW))
    assert a.reason.tolist() == [0] * 5 + [abi.R_RATE_LIMIT] * 2
    # rpm is tighter than rpd: 4 3 2 1 0 on rpm, then the two 429s see the five admissions
    assert [figs(a, i)[0] for i in range(7)] == [(0, 5, 4), (0, 5, 3), (0, 5, 2), (0, 5, 1), (0, 5, 0), (0, 5, 0), (0, 5, 0)]
    assert all(figs(a, i)[1] == (1, 40000, 40000) for i in range(7))
    hs = replies.ratelimit_headers(int(a.reason[5]), int(a.detail[5]), 0, NOW, a.rl_entry[5], a.rl_limit[5], a.rl_remaining[5], t)
    assert hs == [("retry-after", "40"), ("x-ratelimit-limit-requests", "5"), ("x-ratelimit-remaining-requests", "0"),
                  ("x-ratelimit-reset-requests", "40s"), ("x-ratelimit-limit-tokens", "40000"),
                  ("x-ratelimit-remaining-tokens", "40000"), ("x-ratelimit-reset-tokens", "40s")]
    o.response_batch(responses(1, NOW + 1))  # total_tokens 45 on tpm and tpd
    b = o.request_batch(reqs("sk-test123456", 1, NOW + 2))
    assert int(b.reason[0]) == abi.R_RATE_LIMIT and figs(b, 0) == ((0, 5, 0), (1, 40000, 39955))
    # the next minute: rpm starts over (rpd keeps its 5, tpd its 45; tpm is back at 40 000, tighter than tpd's 999 955)
    c = o.request_batch(reqs("sk-test123456", 2, NOW + 40))
    assert c.reason.tolist() == [0, 0]
    assert [figs(c, i) for i in range(2)] == [((0, 5, 4), (1, 40000, 40000)), ((0, 5, 3), (1, 40000, 40000))]
    hs = replies.ratelimit_headers(0, 0, 0, NOW + 40, c.rl_entry[0], c.rl_limit[0], c.rl_remaining[0], t)
    assert ("x-ratelimit-reset-requests", "1m0s") in hs  # NOW + 40 is the first second of its minute


def small(rules, quota="", quotas=(), extra_tokens=()):
    toks = [simple_token("u", "ns", "tk", "m", rules, quota)] + list(extra_tokens)
    return Tables(toks, list(quotas), [simple_endpoint("m", "ns")])


def test_oracle_report_duplicate_rules_and_ties():
    # two rpm entries: every admission adds 2 to the one counter; the 7 entry is the tighter one
    o = RlOracle(small([("rpm", 10), ("rpm", 7)]))
    a = o.request_batch(reqs("tk", 6, NOW, "m"))
    assert a.reason.tolist() == [0, 0, 0, 0, abi.R_RATE_LIMIT, abi.R_RATE_LIMIT] and a.detail.tolist()[4:] == [1, 1]
    assert [figs(a, i)[0] for i in range(6)] == [(1, 7, 5), (1, 7, 3), (1, 7, 1), (1, 7, 0), (1, 7, 0), (1, 7, 0)]
    assert all(figs(a, i)[1] == (NONE, 0, 0) for i in range(6))  # no token-type rule: no tokens figure
    # a tie goes to the first entry of its kind in qos.RateLimits order
    o = RlOracle(small([("rpd", 3), ("rpm", 3), ("tpd", 100), ("tpm", 100)]))
    a = o.request_batch(reqs("tk", 1, NOW, "m"))
    assert figs(a, 0) == ((0, 3, 2), (2, 100, 100))


def test_oracle_report_token_counter_over_its_limit_and_quota_denial():
    o = RlOracle(small([("rpm", 10), ("tpm", 50)]))
    assert o.request_batch(reqs("tk", 2, NOW, "m")).reason.tolist() == [0, 0]
    o.response_batch(responses(2, NOW))  # tpm 90 > 50
    a = o.request_batch(reqs("tk", 1, NOW + 1, "m"))
    assert (int(a.reason[0]), int(a.detail[0])) == (abi.R_RATE_LIMIT, 1)
    assert figs(a, 0) == ((0, 10, 8), (1, 50, 0))
    # quota denial: the figures are reported (the row reached the limiter), nothing is admitted
    o = RlOracle(small([("rpm", 10), ("tpd", 1000)], "q", [simple_quota("q", "ns", [("total", 40)])]))
    assert o.request_batch(reqs("tk", 1, NOW, "m")).reason.tolist() == [0]
    o.response_batch(responses(1, NOW))  # quota total 45 > 40
    a = o.request_batch(reqs("tk", 2, NOW + 1, "m"))
    assert a.reason.tolist() == [abi.R_QUOTA] * 2
    assert figs(a, 0) == figs(a, 1) == ((0, 10, 9), (1, 1000, 955))
    hs = replies.ratelimit_headers(abi.R_QUOTA, 0, 0, NOW + 1, a.rl_entry[0], a.rl_limit[0], a.rl_remaining[0], o.tables)
    assert [k for k, _ in hs] == list(replies.RATELIMIT_HEADERS)  # no retry-after: quotas never reset


def test_oracle_report_rows_that_never_reached_the_limiter():
    t = small([("rpm", 10)], "", (), [simple_token("v", "ns", "tk2", "m", [("rpm", 5)], "gone")])
    o = RlOracle(t)
    bodies = [b"{", b"{}", b'{"model":"m"}', b'{"model":"other"}', b'{"model":"m","stream":true}', b'{"model":"m"}', b'{"model":"m"}']
    toks = [b"tk", b"tk", b"nope", b"tk", b"tk", b"tk2", b"tk"]
    a = o.request_batch(RequestBatch.from_lists(bodies, toks, NOW))
    assert a.reason.tolist() == [abi.R_REQUEST_BODY, abi.R_NO_MODEL, abi.R_TOKEN_NOT_FOUND, abi.R_MODEL_NOT_IN_TOKEN,
                                 abi.R_STREAM_OPTIONS, abi.R_QUOTA_CONFIG, abi.R_OK]
    assert a.rl_entry[:6].tolist() == [[NONE, NONE]] * 6 and figs(a, 6) == ((0, 10, 9), (NONE, 0, 0))


# ---- 2. header shaping --------------------------------------------------------------------------------------------------
GO = [(0, "0s"), (1, "1s"), (59, "59s"), (60, "1m0s"), (61, "1m1s"), (3599, "59m59s"), (3600, "1h0m0s"), (86399, "23h59m59s"),
      (86400, "24h0m0s")]


@pytest.mark.parametrize("s,want", GO)
def test_go_duration(s, want):
    assert replies.go_duration(s) == want


def test_reset_and_retry_after_at_window_edges():
    t = quickstart()
    day = NOW - NOW % 86400
    for now, rpm, rpd, retry in ((day, "1m0s", "24h0m0s", "60"), (day + 59, "1s", "23h59m1s", "1"), (day - 1, "1s", "1s", "1"),
                                 (day + 60, "1m0s", "23h59m0s", "60")):
        e = np.array([0, 1], np.uint8)
        hs = dict(replies.ratelimit_headers(abi.R_RATE_LIMIT, 0, 0, now, e, [5, 40000], [0, 1], t))
        assert (hs["x-ratelimit-reset-requests"], hs["x-ratelimit-reset-tokens"], hs["retry-after"]) == (rpm, rpm, retry)
        e = np.array([2, 3], np.uint8)  # the rpd / tpd entries
        hs = dict(replies.ratelimit_headers(abi.R_RATE_LIMIT, 2, 0, now, e, [100, 10**6], [0, 1], t))
        assert (hs["x-ratelimit-reset-requests"], hs["x-ratelimit-reset-tokens"]) == (rpd, rpd)
        assert int(hs["retry-after"]) == replies.window_end(now, "rpd") - now
        assert replies.window_end(now, "rpm") - now == int(retry)


# the compiled host over tests/ratelimit_shim.c, in a process of its own: a shim loaded earlier by another test module would
# otherwise answer the host's calls
def _rl_shim():
    out = os.path.join(BUILD, "libarksgw_rlshim.so")
    ork = rl_oracle_path()
    srcs = [os.path.join(HERE, f) for f in ("ratelimit_shim.c", "abi_shim.c")] + [ork]
    if _stale(out, srcs):
        d = os.path.dirname(ork)
        subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", out, os.path.join(HERE, "ratelimit_shim.c"), "-L" + d,
                               "-larks_oracle_rl", "-Wl,-rpath," + d])
    return out


class ShimHost:
    """host/cpp's Batcher over the oracle (report mode) behind tests/ratelimit_shim.c"""

    def __init__(self, tables, report=True, **kw):
        shim = _rl_shim()
        self.shim = C.CDLL(shim, mode=C.RTLD_GLOBAL)
        self.L = cpphost.load(cpphost.build(os.path.join(BUILD, "libarkshost_rlshim.so"), against=shim))
        self._ts = tables.c_struct()
        self.ctx = C.c_void_p()
        self.shim.arks_shim_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        assert self.shim.arks_shim_create(C.byref(self._ts), C.byref(self.ctx)) == 0
        self.b = cpphost.Batcher(self.L, self.ctx, **kw)
        self.b.set_names(tables)
        if report:
            self.b.set_ratelimit_report(True)

    def close(self):
        self.b.close()


def _in_subprocess(fn):
    code = f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_ratelimit_headers as T; T.{fn}()"
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT)


def test_cpp_and_python_shapers_agree():
    _in_subprocess("check_shapers_agree")


def check_shapers_agree():
    t = Tables(FX["tokens"] + [simple_token("v", "ns", "tk2", "qwen-7b", [("tpd", 9), ("rpd", 3), ("rpm", 1), ("tpm", 4)])],
               FX["quotas"], FX["endpoints"] + [simple_endpoint("qwen-7b", "ns")])
    h = ShimHost(t)
    try:
        gen = h.b.request(b"tk2", b'{"model":"qwen-7b"}').gen  # the generation the names were published under
        rng = np.random.default_rng(5)
        day = NOW - NOW % 86400
        table = [(0, 0, 0, day, (0, 1)), (8, 2, 1, day + 59, (2, 0)), (9, 0, 0, day - 1, (0, NONE)), (8, 0, 0, NOW, (NONE, 1)),
                 (4, 0, 0, NOW, (0, 1)), (10, 0, 0, NOW, (0, 1)), (255, 0, 0, NOW, (0, 1)), (0, 0, 1, NOW, (NONE, NONE))]
        for _ in range(300):
            q = int(rng.integers(0, 2))
            n_rl = 4
            table.append((int(rng.choice([0, 8, 9, 1, 7, 10])), int(rng.integers(0, n_rl)), q, int(NOW + rng.integers(-10**6, 10**6)),
                          tuple(int(x) if rng.random() < 0.8 else NONE for x in rng.integers(0, n_rl, 2))))
        for reason, detail, q, now, ent in table:
            d = cpphost.RequestDecision()
            d.reason, d.detail, d.qos, d.now_unix, d.gen = reason, detail, q, now, gen
            lim, rem = [int(x) for x in rng.integers(0, 10**9, 2)], [int(x) for x in rng.integers(0, 10**6, 2)]
            for k in range(2):
                d.rl_entry[k], d.rl_limit[k], d.rl_remaining[k] = ent[k], lim[k], rem[k]
            want = replies.ratelimit_headers(reason, detail, q, now, list(ent), lim, rem, t)
            assert h.b.ratelimit_headers(d) == want, (reason, detail, q, now, ent)
    finally:
        h.close()


# ---- 3. / 4. ext_proc transcripts: the C++ StreamProcessor against the Python server ---------------------------------------
def py_transcript(srv, req_headers, req_body, resp_headers, chunks):
    """the Python server's replies to one stream in arks_host_stream_transcript's text form"""
    msgs = []
    m = PB["ProcessingRequest"]()
    for k, v in req_headers:
        h = m.request_headers.headers.headers.add()
        h.key, h.raw_value = k, v.encode()
    msgs.append(m)
    m = PB["ProcessingRequest"]()
    m.request_body.body, m.request_body.end_of_stream = req_body, True
    msgs.append(m)
    m = PB["ProcessingRequest"]()
    for k, v in resp_headers:
        h = m.response_headers.headers.headers.add()
        h.key, h.raw_value = k, v.encode()
    msgs.append(m)
    for i, c in enumerate(chunks):
        m = PB["ProcessingRequest"]()
        m.response_body.body, m.response_body.end_of_stream = c, i + 1 == len(chunks)
        msgs.append(m)
    out = ""
    kinds = {"request_headers": 0, "request_body": 1, "response_headers": 2, "response_body": 3}
    for r in srv.Process(iter(msgs), None):
        w = r.WhichOneof("response")
        if w == "immediate_response":
            im = r.immediate_response
            hs = [(o.header.key, (o.header.raw_value or o.header.value.encode()).decode("latin1")) for o in im.headers.set_headers]
            out += f"4 {im.status.code} 0\n" + "".join(f"{k}: {v}\n" for k, v in hs) + "\n" + im.body.decode("latin1") + "\n--\n"
            break
        cr = getattr(r, w).response
        hs = [(o.header.key, (o.header.raw_value or o.header.value.encode()).decode("latin1")) for o in cr.header_mutation.set_headers]
        out += f"{kinds[w]} 0 {int(cr.clear_route_cache)}\n" + "".join(f"{k}: {v}\n" for k, v in hs) + "\n\n--\n"
    return out


REQ_H = [(":method", "POST"), ("authorization", "Bearer sk-test123456"), ("content-type", "application/json")]
SREQ = b'{"model":"qwen-7b","stream":true,"stream_options":{"include_usage":true},"messages":[]}'


def stream_cases():
    sse = json.load(open(os.path.join(HERE, "golden", "sse_stream.json")))
    body = FX["request_body"].encode()
    ok = [(":status", "200"), ("content-type", "application/json")]
    return [
        ("admitted non-stream", REQ_H, body, ok, [RESP[:100], RESP[100:]]),
        ("admitted stream", REQ_H, SREQ, [(":status", "200")], [c.encode() for c in sse["chunks"]]),
        ("upstream 500", REQ_H, body, [(":status", "500"), ("x-ratelimit-remaining-requests", "77")], [b"boom"]),
        ("upstream header replaced", REQ_H, body, ok + [("X-RateLimit-Remaining-Requests", "77"), ("x-ratelimit-limit-tokens", "1")],
         [RESP]),
        ("upstream 404", REQ_H, body, [(":status", "404")], [b'{"detail":"nope"}']),
        ("429 rate limit", REQ_H, body, ok, [RESP]),
        ("429 rate limit again", REQ_H, body, ok, [RESP]),
        ("no bearer", [("content-type", "application/json")], body, [], []),
    ]


def run_transcripts(host, tables, report, clock_now=NOW):
    """every case through both; returns the C++ transcripts"""
    host.b.set_fixed_clock(clock_now)
    eng = RlOracle(tables, report=report)
    from arks_b200 import gateway
    srv = extproc.ExtProcServer(eng, tables, gateway.extract_bearer, clock=lambda: clock_now)
    got = []
    try:
        for name, rh, rb, ph, chunks in stream_cases():
            a = host.b.stream_transcript(rh, rb, ph, chunks)
            b = py_transcript(srv, rh, rb, ph, chunks)
            assert a == b, (name, a, b)
            got.append((name, a))
    finally:
        srv.batcher.close()
    return got


def test_transcripts_cpp_equal_python_report_on():
    _in_subprocess("check_transcripts_on")


def check_transcripts_on():
    import __graft_entry__ as ge
    ge.build()  # arks_extract_bearer of the Python server
    t = quickstart()
    # the quota rows: a second token on the same model whose quota is already over
    t = Tables(FX["tokens"] + [simple_token("q", "default", "sk-quota", "qwen-7b", [("rpm", 9), ("tpd", 500)], "tiny")],
               FX["quotas"] + [simple_quota("tiny", "default", [("total", 0)])], FX["endpoints"])
    h = ShimHost(t, max_batch=64, max_bytes=1 << 20)
    try:
        got = dict(run_transcripts(h, t, report=True))
        adm = got["admitted non-stream"].split("--\n")
        assert adm[2] == ("2 0 1\nx-went-into-resp-headers: true\n:status: 200\ncontent-type: application/json\n"
                          "x-ratelimit-limit-requests: 5\nx-ratelimit-remaining-requests: 4\nx-ratelimit-reset-requests: 40s\n"
                          "x-ratelimit-limit-tokens: 40000\nx-ratelimit-remaining-tokens: 40000\nx-ratelimit-reset-tokens: 40s\n\n\n")
        assert "x-ratelimit" not in adm[1]  # the request-body reply keeps the reference's three routing headers
        assert "x-ratelimit" not in got["upstream 500"].split("--\n")[2].replace("x-ratelimit-remaining-requests: 77", "")
        rep = got["upstream header replaced"].split("--\n")[2]
        assert "77" not in rep and "x-ratelimit-limit-tokens: 1\n" not in rep and rep.count("x-ratelimit-remaining-requests") == 1
        blk = got["429 rate limit"].split("--\n")[1]
        assert blk.startswith("4 429 0\nx-error-rate-limit: true\nContent-Type: application/json\nretry-after: 40\n"
                              "x-ratelimit-limit-requests: 5\nx-ratelimit-remaining-requests: 0\n")
        assert "x-ratelimit" not in got["no bearer"]
        # quota 429: figures, no retry-after
        q = h.b.stream_transcript([("authorization", "Bearer sk-quota")], FX["request_body"].encode(), [(":status", "200")], [RESP])
        assert q.split("--\n")[1].startswith("1 0 0\n")  # admitted once: bills 45 > 0
        q = h.b.stream_transcript([("authorization", "Bearer sk-quota")], FX["request_body"].encode(), [(":status", "200")], [RESP])
        blk = q.split("--\n")[1]
        assert blk.startswith("4 429 0\nx-error-quota: true\nContent-Type: application/json\nx-ratelimit-limit-requests: 9\n"
                              "x-ratelimit-remaining-requests: 8\nx-ratelimit-reset-requests: 40s\nx-ratelimit-limit-tokens: 500\n"
                              "x-ratelimit-remaining-tokens: 455\nx-ratelimit-reset-tokens: 1h46m40s\n")
    finally:
        h.close()


def test_report_off_adds_no_header():
    _in_subprocess("check_transcripts_off")


def _ours(text):
    """rate-limit header lines in a transcript"""
    return [ln for ln in text.splitlines() if ln.lower().startswith(("x-ratelimit-", "retry-after:"))]


def check_transcripts_off():
    import __graft_entry__ as ge
    ge.build()
    t = quickstart()
    # only the upstream's own x-ratelimit-* headers, echoed as the reference echoes every response header
    echoed = {name: [f"{k}: {v}" for k, v in ph if k.lower().startswith("x-ratelimit-")] for name, _, _, ph, _ in stream_cases()}
    h = ShimHost(t, report=False, max_batch=64, max_bytes=1 << 20)
    try:
        for name, text in run_transcripts(h, t, report=False):
            assert _ours(text) == echoed[name], name
    finally:
        h.close()
    # switched on and off again: the same
    h = ShimHost(t, report=True, max_batch=64, max_bytes=1 << 20)
    try:
        h.b.set_ratelimit_report(False)
        for name, text in run_transcripts(h, t, report=False):
            assert _ours(text) == echoed[name], name
    finally:
        h.close()


def test_process_flag_is_the_library_switch():
    from arks_b200 import __main__ as M

    class Rec:
        def __init__(self):
            self.calls = []

        def set_ratelimit_report(self, on):
            self.calls.append(on)

    class Cb:
        def __init__(self):
            self.b = Rec()

    for argv, want in (([], []), (["--gateway.ratelimit-headers"], [True])):
        a = M.parse_args(argv)
        e, cb = Rec(), Cb()
        M.configure_ratelimit_headers(e, cb, a)
        assert e.calls == want and cb.b.calls == want
        e = Rec()
        M.configure_ratelimit_headers(e, None, a)  # the Python batcher: the engine's switch alone
        assert e.calls == want


# ---- GPU --------------------------------------------------------------------------------------------------------------------
def gpu_tables(n_small=400, seed=3, front=()):
    """`front`: tokens listed before the others. Small groups with room, straddling groups (rpm + rpd), duplicate rules, token-type rules that responses push over,
    quota denials and a missing quota, and four hot tokens for groups of 255..258 arrivals"""
    rng = np.random.default_rng(seed)
    toks, quotas = [], [simple_quota("qa", "ns", [("total", 2000)]), simple_quota("qz", "ns", [("total", 0), ("prompt", 10**9)])]
    for i in range(n_small):
        kind = i % 6
        if kind == 0:
            rl = [("rpm", 10**6)]
        elif kind == 1:
            rl = [("rpm", int(rng.integers(1, 6))), ("rpd", int(rng.integers(2, 9)))]
        elif kind == 2:
            rl = [("rpm", int(rng.integers(3, 12))), ("tpm", 100), ("rpm", int(rng.integers(2, 9))), ("tpd", 10**5)]
        elif kind == 3:
            rl = [("tpm", 90), ("rpm", 50), ("tpd", 200)]
        elif kind == 4:
            rl = [("rpd", 20), ("tpm", 1000)]
        else:
            rl = [("rpm", 30)]
        quota = ["", "qa", "qz", "missing"][int(rng.integers(0, 4))] if kind >= 4 else ""
        toks.append(simple_token(f"u{i}", "ns", f"t{i}", "m", rl, quota))
    for i, lim in enumerate((256, 255, 300, 257)):  # hot tokens: groups of 255..258 around kHotGroup, some straddling
        toks.append(simple_token(f"h{i}", "ns", f"hot{i}", "m", [("rpm", lim), ("tpm", 10**6), ("rpd", lim + 1)]))
    return Tables(list(front) + toks, quotas, [simple_endpoint("m", "ns")])


def gpu_traffic(t, n, now, seed):
    rng = np.random.default_rng(seed)
    n_small = len(t.token_string) - 4
    toks = []
    room = n // 2
    for i, size in enumerate((255, 256, 257, 258)):
        if size <= room:
            toks += [f"hot{i}"] * size
            room -= size
    while len(toks) < n:
        r = rng.random()
        toks.append("nope" if r < 0.02 else f"t{int(rng.integers(0, n_small))}")
    toks = [toks[i] for i in rng.permutation(n)]
    bodies = []
    for k in range(n):
        r = rng.random()
        if r < 0.02:
            bodies.append(b'{"model":')
        elif r < 0.04:
            bodies.append(b'{"model":"other","messages":[]}')
        else:
            bodies.append(b'{"model":"m","messages":[{"role":"user","content":"hello %d"}]}' % k)
    return RequestBatch.from_lists(bodies, [x.encode() for x in toks], now, pick_rand=rng.integers(0, 1 << 62, n, dtype=np.uint64))


def same_decisions(a, b, where):
    for k, v in a.fields().items():
        assert np.array_equal(v, b.fields()[k]), (where, k)


def same_report(a, b, where):
    for k in ("rl_entry", "rl_limit", "rl_remaining"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), (where, k, np.flatnonzero((getattr(a, k) != getattr(b, k)).any(1))[:8])


def day_edge():
    return (NOW // 86400 + 1) * 86400


def answer(g, o, a, now):
    """every admitted row of a token-type entry answers with usage 45: the token counters climb over their limits"""
    ok = np.flatnonzero(a.reason == abi.R_OK)
    if not len(ok):
        return
    rb = ResponseBatch.from_lists([RESP] * len(ok), a.qos[ok], [abi.RESP_END_OF_STREAM] * len(ok), now)
    c, d = g.handle_response_body(rb), o.response_batch(rb)
    assert np.array_equal(c.reason, d.reason) and np.array_equal(c.counted, d.counted)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1200, 3000, 8192])  # warp path (<= 2048), exact engine alone, two-stage fast path (>= 4096)
def test_gpu_report_equals_the_oracle(gwmod, n):
    t = gpu_tables()
    g = gwmod.Gateway(0, 16384, 32 << 20)
    g.load_tables(t)
    g.set_ratelimit_report(True)
    o = RlOracle(t)
    d = day_edge()
    seen_hot = set()
    for step, now in enumerate((d - 61, d - 30, d - 1, d, d + 59, d + 60)):  # minute and day windows crossed
        req = gpu_traffic(t, n, now, seed=100 * n + step)
        a, want = g.handle_request_body(req), o.request_batch(req)
        same_decisions(a, want, (n, step))
        same_report(a, want, (n, step))
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), (n, step)
        reasons = set(a.reason.tolist())
        assert {abi.R_OK, abi.R_RATE_LIMIT}.issubset(reasons) and (a.rl_entry == NONE).any() and (a.rl_entry != NONE).any()
        seen_hot |= set(np.unique(a.qos[a.qos >= len(t.token_string) - 4]).tolist())
        answer(g, o, a, now)
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), (n, step)
    assert seen_hot


@pytest.mark.gpu
def test_gpu_report_changes_nothing(gwmod):
    t = gpu_tables(seed=4)
    on, off, toggled = (gwmod.Gateway(0, 16384, 32 << 20) for _ in range(3))
    for g in (on, off, toggled):
        g.load_tables(t)
        g.enable_metrics(True)
    on.set_ratelimit_report(True)
    toggled.set_ratelimit_report(True)
    toggled.set_ratelimit_report(False)
    d = day_edge()
    for step, (n, now) in enumerate(((700, d - 5), (9000, d - 1), (3000, d + 2))):
        req = gpu_traffic(t, n, now, seed=7 + step)
        l0 = [g.launch_count for g in (on, off, toggled)]
        a, b = on.handle_request_body(req), off.handle_request_body(req)
        c = toggled.handle_request_body(req, RequestResult.empty(n, report=True))  # the off path leaves the columns alone
        launches = [g.launch_count - x for g, x in zip((on, off, toggled), l0)]
        assert launches[0] == launches[1] == launches[2], launches  # no kernel of its own
        for r in (b, c):
            same_decisions(a, r, step)
            assert np.array_equal(a.bpe_count, r.bpe_count)
        assert (c.rl_entry == 0xEE).all() and (c.rl_limit == -9).all() and b.rl_entry is None
        for g in (off, toggled):
            assert np.array_equal(on.snapshot_rate(now), g.snapshot_rate(now)) and np.array_equal(on.snapshot_metrics(), g.snapshot_metrics())
        ok = np.flatnonzero(a.reason == abi.R_OK)
        rb = ResponseBatch.from_lists([RESP] * len(ok), a.qos[ok], [abi.RESP_END_OF_STREAM] * len(ok), now)
        for g in (on, off, toggled):
            g.handle_response_body(rb)


@pytest.mark.gpu
def test_gpu_report_with_precharge_and_metering(gwmod):
    from arks_b200 import bpe
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    t = gpu_tables(seed=5)
    g = gwmod.Gateway(0, 16384, 32 << 20)
    g.load_tables(t)
    g.load_bpe(bpe.load_tokenizer(text))
    g.set_precharge(True)
    g.set_stream_metering(True)
    g.set_ratelimit_report(True)
    o = RlOracle(t)
    o.set_precharge(True)
    for step, n in enumerate((1500, 9000, 600)):
        now = NOW + step
        req = gpu_traffic(t, n, now, seed=50 + step)
        a = g.handle_request_body(req)
        o.set_estimates(a.bpe_count)
        want = o.request_batch(req)
        same_decisions(a, want, step)
        same_report(a, want, step)  # the tokens figure is the batch's start: this batch's pre-charges are not in it
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), step


@pytest.mark.gpu
def test_gpu_report_across_a_generation_swap(gwmod):
    t1 = gpu_tables(n_small=300, seed=6)
    # the next generation: one more token in front, so every qos index moves; the counters follow their keys
    t2 = gpu_tables(n_small=300, seed=6, front=[simple_token("new", "ns", "tnew", "m", [("rpm", 2)])])
    g = gwmod.Gateway(0, 16384, 32 << 20)
    g.load_tables(t1)
    g.set_ratelimit_report(True)
    o = RlOracle(t1)
    for step in range(4):
        now = NOW + 10 * step
        if step == 2:
            g.commit_tables(g.prepare_tables(t2))
            o.reload(t2)
        t = t2 if step >= 2 else t1
        req = gpu_traffic(t, 2500, now, seed=70 + step)
        a, want = g.handle_request_body(req), o.request_batch(req)
        same_decisions(a, want, step)
        same_report(a, want, step)
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), step
        answer(g, o, a, now)


@pytest.mark.gpu
@pytest.mark.parametrize("inflight", [1, 4])
def test_gpu_compiled_host_transcripts_equal_the_python_mirror(gwmod, inflight):
    t = Tables(FX["tokens"] + [simple_token("q", "default", "sk-quota", "qwen-7b", [("rpm", 9), ("tpd", 500)], "tiny")],
               FX["quotas"] + [simple_quota("tiny", "default", [("total", 0)])], FX["endpoints"])
    g = gwmod.Gateway(0, 4096, 8 << 20)
    g.load_tables(t)

    from types import SimpleNamespace
    Host = SimpleNamespace(b=cpphost.Batcher(cpphost.load(cpphost.build()), g._h, max_batch=256, max_bytes=1 << 20,
                                             max_inflight=inflight))
    try:
        Host.b.set_names(t)
        Host.b.set_ratelimit_report(True)
        got = dict(run_transcripts(Host, t, report=True))
        assert "x-ratelimit-remaining-requests: 4\n" in got["admitted non-stream"]
        assert "retry-after: 40\n" in got["429 rate limit"]
    finally:
        Host.b.close()
