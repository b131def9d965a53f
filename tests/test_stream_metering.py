"""N5, opt-in stream metering (include/arks_gateway.h: arks_set_stream_metering). The reference refuses every stream:true request
without stream_options.include_usage:true (handle_request.go:156-171) because it cannot bill it; with metering on such a
request is decided like any other and billed by the on-device BPE counts of its prompt (when its micro-batch commits) and of
its SSE chunks (the upstream's `usage`, if any, is reported but not billed).

CPU: the metering oracle (tests/meter_model.py, on the reference oracle) on hand-made scenarios, the wide key set of the host
build (tests/bpe_keys_host.cpp) against HF `tokenizers`, the C++ StreamProcessor carrying the metered bit over
tests/meter_shim.c. GPU: the CUDA path against the metering oracle fed with `tokenizers` counts, on the warp, exact and fast
request paths."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import orklib
from arks_b200 import abi, bpe, cpphost, traffic
from arks_b200.abi import RequestBatch, ResponseBatch
from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token
from meter_model import METERED_CHUNK, MeteredOracle, is_metered_request

NOW = 1_700_000_000
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
UNC = bpe.UNCOUNTED


def small_tables():
    return Tables([simple_token("u", "ns", "tk", "m", [("tpm", 1000), ("rpm", 50), ("tpd", 10**6), ("tpm", 10**6)], "q")],
                  [simple_quota("q", "ns", [("prompt", 10**6), ("response", 10**6), ("total", 10**6)])], [simple_endpoint("m", "ns")])


METERED = b'{"model":"m","stream":true,"messages":[{"role":"user","content":"hello there"}]}'
WITH_USAGE = b'{"model":"m","stream":true,"stream_options":{"include_usage":true},"messages":[{"role":"user","content":"hi"}]}'
PLAIN = b'{"model":"m","messages":[{"role":"user","content":"hi"}]}'
CHUNK = b'data: {"choices":[{"delta":{"content":"abc"}}],"usage":null}\n\n'
USAGE_CHUNK = b'data: {"choices":[],"usage":{"prompt_tokens":7,"completion_tokens":5,"total_tokens":12}}\n\ndata: [DONE]\n\n'


def test_oracle_stream_metering_mode():
    t = small_tables()
    o = MeteredOracle(t)
    # off: the reference's 400
    assert o.request_batch(RequestBatch.from_lists([METERED], [b"tk"], NOW)).reason.tolist() == [abi.R_STREAM_OPTIONS]
    o.set_stream_metering(True)
    a = o.request_batch(RequestBatch.from_lists([METERED, WITH_USAGE, PLAIN], [b"tk"] * 3, NOW), counts=[30, 9, 4])
    assert a.reason.tolist() == [0, 0, 0]
    assert a.flags.tolist() == [1 | abi.FLAG_METERED, 1, 0]
    # the metered prompt is charged when the batch commits: twice on tpm (two entries), once on tpd; prompt and total items
    assert o.snapshot_rate(NOW)[0].tolist() == [3, 0, 60, 30]
    assert o.snapshot_quota()[0].tolist() == [30, 0, 30]
    m = o.snapshot_metrics()[0]
    assert m[abi.METRIC_USAGE:abi.METRIC_USAGE + 2].tolist() == [30, 0] and m[abi.METRIC_MESSAGES] == 0
    # chunks: a metered one is billed its count; a metered usage-bearing one is billed its count, its usage reported only;
    # an uncounted metered one is billed its length; the include_usage stream is billed its usage as before
    resp = ResponseBatch.from_lists([CHUNK, USAGE_CHUNK, CHUNK, USAGE_CHUNK], [0] * 4,
                                    [METERED_CHUNK, METERED_CHUNK, METERED_CHUNK, abi.RESP_STREAM], NOW + 1)
    c = o.response_batch(resp, counts=[3, 0, UNC, 0])
    assert c.reason.tolist() == [0] * 4
    assert c.counted.tolist() == [0, 0, 0, 1]
    assert c.usage[1].tolist() == [7, 5, 12] and c.usage[3].tolist() == [7, 5, 12]
    billed = 3 + 0 + len(CHUNK)
    assert o.snapshot_rate(NOW + 1)[0].tolist() == [3, 0, 60 + 2 * (billed + 12), 30 + billed + 12]
    assert o.snapshot_quota()[0].tolist() == [30 + 7, billed + 5, 30 + billed + 12]
    m = o.snapshot_metrics()[0]
    assert m[abi.METRIC_USAGE:abi.METRIC_USAGE + 2].tolist() == [30, billed] and m[abi.METRIC_MESSAGES] == 4
    # no count for the prompt: its length is billed
    o.request_batch(RequestBatch.from_lists([METERED], [b"tk"], NOW + 2))
    assert o.snapshot_quota()[0, 0] == 37 + len(METERED)
    # switch off again: the reference's 400
    o.set_stream_metering(False)
    assert o.request_batch(RequestBatch.from_lists([METERED], [b"tk"], NOW + 3)).reason.tolist() == [abi.R_STREAM_OPTIONS]


def test_oracle_metering_with_precharge_bills_once():
    o = MeteredOracle(small_tables())
    o.set_precharge(True)
    o.set_stream_metering(True)
    a = o.request_batch(RequestBatch.from_lists([METERED, WITH_USAGE], [b"tk"] * 2, NOW), counts=[30, 9])
    assert a.flags.tolist() == [1 | abi.FLAG_METERED, 1]
    assert o.snapshot_rate(NOW)[0].tolist() == [2, 0, 2 * (30 + 9), 30 + 9]  # metered: meter only; the other: pre-charge
    resp = ResponseBatch.from_lists([USAGE_CHUNK, USAGE_CHUNK], [0, 0], [METERED_CHUNK, abi.RESP_STREAM], NOW + 1)
    resp.precharged = np.array([30, 9], np.uint32)  # ignored on the metered row
    c = o.response_batch(resp, counts=[4, 0])
    assert c.counted.tolist() == [0, 1]
    assert o.snapshot_rate(NOW + 1)[0].tolist() == [2, 0, 2 * (30 + 9 + 4 + 12 - 9), 30 + 9 + 4 + 12 - 9]
    assert o.snapshot_quota()[0].tolist() == [30 + 7, 4 + 5, 30 + 4 + 12]


WIDE_BODIES = [
    b'{"model":"m","stream":true,"messages":[{"role":"user","content":[{"type":"text","text":"What is in this image?"},'
    b'{"type":"image_url","image_url":{"url":"https://x"}}]},{"role":"assistant","content":"A cat.","reasoning_content":'
    b'"The picture shows\\n a cat"},{"role":"assistant","tool_calls":[{"id":"c1","type":"function","function":{"name":"get",'
    b'"arguments":"{\\"city\\": \\"Paris\\", \\"n\\": 3}"}}]}]}',
    b'{"model":"m","messages":[{"role":"user","\\u0074ext":"escaped key","cont\\u0065nt":"also escaped"}],"text":7,'
    b'"arguments":{"text":"nested"},"contents":"not a key","reasoning_content":"why not"}',
]
WIDE_CHUNKS = [
    b'data: {"choices":[{"delta":{"reasoning_content":"Let me think"}}]}\n\ndata: {"choices":[{"delta":{"content":" ok"}}]}\n\n',
    b'data: {"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"arguments":"{\\"q\\": 1}"}}]}}]}\n\n',
]


def _bpe_keys_lib(tables):
    """tests/bpe_keys_host.cpp: the host build of bpe.cuh's scanner with a chosen key set"""
    os.makedirs(BUILD, exist_ok=True)
    src, out = os.path.join(HERE, "bpe_keys_host.cpp"), os.path.join(BUILD, "libbpe_keys.so")
    deps = [src] + [os.path.join(ROOT, "arks_b200", "csrc", f) for f in ("bpe.cuh", "json_common.cuh")]
    if not os.path.exists(out) or max(map(os.path.getmtime, deps)) > os.path.getmtime(out):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, src])
    L = C.CDLL(out)
    u32p = C.POINTER(C.c_uint32)
    L.bk_load.argtypes = [u32p, C.c_uint32, u32p, u32p, u32p, C.POINTER(C.c_uint8), C.c_uint32]
    L.bk_count.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    L.bk_count.restype = C.c_uint32
    t = tables.c_struct()
    L.bk_load(t.byte_id, t.n_merges, t.left, t.right, t.merged, t.cp_class, t.flags)
    L._keep = tables
    return L


def test_host_build_wide_count_matches_tokenizers():
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    L = _bpe_keys_lib(bpe.load_tokenizer(text))
    wide = lambda b: int(L.bk_count(b, len(b), 1))
    narrow = lambda b: int(L.bk_count(b, len(b), 0))
    n = lambda strs: sum(len(tok.encode(s, add_special_tokens=False).ids) for s in strs)
    for body in WIDE_BODIES:
        assert wide(body) == n(bpe.content_strings(body, bpe.METERED_KEYS)) > 0
        assert narrow(body) == n(bpe.content_strings(body))
        assert wide(body) > narrow(body)
    for ch in WIDE_CHUNKS:
        assert wide(ch) == n(bpe.sse_content_strings(ch, bpe.METERED_KEYS)) > 0
        assert narrow(ch) == n(bpe.sse_content_strings(ch))


def test_stream_processor_carries_the_metered_bit_cpu():
    """host/cpp over tests/meter_shim.c: RESP_METERED on every chunk of the metered stream, on no chunk of any other. In a
    process of its own: a shim loaded earlier (tests/test_cpp_host.py) would otherwise answer the host's calls"""
    code = f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_stream_metering as T; T.check_carry_over_meter_shim()"
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT)


def check_carry_over_meter_shim():
    import test_cpp_host as T
    T._shim()  # the oracle library the shim links against
    ork = orklib.build_oracle()
    shim = os.path.join(BUILD, "libarksgw_metershim.so")
    src = os.path.join(HERE, "meter_shim.c")
    if not os.path.exists(shim) or max(os.path.getmtime(src), os.path.getmtime(os.path.join(HERE, "abi_shim.c")),
                                       os.path.getmtime(ork)) > os.path.getmtime(shim):
        d = os.path.dirname(ork)
        subprocess.check_call(["gcc", "-O2", "-shared", "-fPIC", "-o", shim, src, "-L" + d, "-larks_oracle", "-Wl,-rpath," + d])
    S = C.CDLL(shim, mode=C.RTLD_GLOBAL)
    L = cpphost.load(cpphost.build(os.path.join(BUILD, "libarkshost_metershim.so"), against=shim))
    t = small_tables()
    ts = t.c_struct()
    ctx = C.c_void_p()
    S.arks_shim_create.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
    assert S.arks_shim_create(C.byref(ts), C.byref(ctx)) == 0
    S.arks_set_stream_metering.argtypes = [C.c_void_p, C.c_int]
    S.meter_shim_log.argtypes = [C.POINTER(C.c_uint8), C.POINTER(C.c_int32), C.c_uint32]
    S.meter_shim_log.restype = C.c_uint32

    def log():
        f, q = (C.c_uint8 * 256)(), (C.c_int32 * 256)()
        n = S.meter_shim_log(f, q, 256)
        return [int(f[k]) for k in range(n)]
    b = cpphost.Batcher(L, ctx, max_batch=64, max_bytes=1 << 20)
    try:
        b.set_fixed_clock(NOW)
        b.set_names(t)
        req_h = [(":method", "POST"), ("authorization", "Bearer tk")]
        ok = [(":status", "200")]
        assert "\n4 400 " in "\n" + b.stream_transcript(req_h, METERED, ok, [CHUNK])  # off: the reference's 400
        log()
        S.arks_set_stream_metering(ctx, 1)
        got = b.stream_transcript(req_h, METERED, ok, [CHUNK, CHUNK, USAGE_CHUNK])
        assert "\n4 " not in "\n" + got
        assert log() == [METERED_CHUNK] * 3
        b.stream_transcript(req_h, WITH_USAGE, ok, [CHUNK, USAGE_CHUNK])  # the same mode, an include_usage stream
        assert log() == [abi.RESP_STREAM] * 2
        b.stream_transcript(req_h, PLAIN, ok, [b'{"model":"m","usage":{"prompt_tokens":1,"completion_tokens":1,"total_tokens":2}}'])
        assert log() == [abi.RESP_END_OF_STREAM]
    finally:
        b.close()


# ---- GPU -----------------------------------------------------------------------------------------------------------------
def _metered_traffic(w, n, now, seed):
    """a varied batch: ~60 % streams, half of them without include_usage (metered), the rest include_usage streams and
    non-stream requests; the metered ones also carry content parts, reasoning and tool-call arguments"""
    req = w.request_batch(n, now, seed=seed, stream_frac=0.6, varied=True)
    rng = np.random.default_rng(seed)
    bodies = []
    for i in range(req.n):
        b = bytes(req.bodies[req.body_off[i]:req.body_off[i] + req.body_len[i]])
        if b'"include_usage":true' in b and rng.random() < 0.5:
            b = re.sub(rb',\s*"stream_options":\{"include_usage":true\}', b"", b)
            b = b[:-1] + (b',"extra":[{"type":"text","text":"part %d"}],"reasoning_content":"step %d then","tool":'
                          b'{"arguments":"{\\"k\\": %d}"}}' % (i, i * 7, i))
        bodies.append(b)
    toks = [bytes(req.tokens[req.token_off[i]:req.token_off[i + 1]]) for i in range(req.n)]
    return RequestBatch.from_lists(bodies, toks, now, pick_rand=req.pick_rand), bodies


def _expected_counts(tok, device, docs, wide, sse):
    """tokenizers' counts of `docs` (wide: the metered key set), checked against the device's and fed to the oracle; rows
    the device leaves uncounted keep ARKS_BPE_UNCOUNTED (both then bill the body length)"""
    out = np.array(device, np.uint32)
    for i, d in enumerate(docs):
        if device[i] == UNC:
            continue
        keys = bpe.METERED_KEYS if wide[i] else bpe.CONTENT_KEYS
        strs = bpe.sse_content_strings(d, keys) if sse[i] else bpe.content_strings(d, keys)
        out[i] = sum(len(tok.encode(s, add_special_tokens=False).ids) for s in strs)
    assert np.array_equal(out, device)
    return out


def _same(a, b, what):
    for k, v in a.fields().items():
        assert np.array_equal(v, b.fields()[k]), (what, k)


@pytest.mark.gpu
def test_gpu_stream_metering_matches_the_oracle(gwmod):
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    w = traffic.Workload(n_tenants=300, seed=23)
    g = gwmod.Gateway(0, 32768, 64 << 20)
    g.load_tables(w.tables)
    g.enable_metrics(True)
    with pytest.raises(Exception):
        g.set_stream_metering(True)  # no vocabulary yet
    g.load_bpe(bpe.load_tokenizer(text))
    g.set_stream_metering(True)
    with pytest.raises(Exception):
        g.load_bpe(None)  # refused while metering is on
    o = MeteredOracle(w.tables)
    o.set_stream_metering(True)
    n_metered = 0
    for step, n in enumerate((700, 3000, 9000)):  # warp path, exact engine, fast path
        now = NOW + step
        req, bodies = _metered_traffic(w, n, now, 40 + step)
        a = g.handle_request_body(req)
        wide = [is_metered_request(b) for b in bodies]
        est = _expected_counts(tok, a.bpe_count, bodies, wide, [False] * n)
        want = o.request_batch(req, counts=est)
        _same(a, want, ("request", step))
        metered = (a.flags & abi.FLAG_METERED) != 0
        n_metered += int(metered.sum())
        assert metered.sum() > 0.2 * n and np.all(a.reason[metered] == abi.R_OK)
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), step
        assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), step
        assert np.array_equal(g.snapshot_metrics(), o.snapshot_metrics()), step
        # the chunks: RESP_METERED on every chunk of a metered stream; half of them stream reasoning instead of content
        resp = w.response_batch(a, now, seed=70 + step, varied=True)
        owner = np.repeat(np.flatnonzero(a.reason == abi.R_OK), np.where(a.flags[a.reason == abi.R_OK] & 1, 4, 1))
        assert len(owner) == resp.n
        docs, flags = [], []
        for k in range(resp.n):
            d = bytes(resp.bodies[resp.body_off[k]:resp.body_off[k] + resp.body_len[k]])
            f = int(resp.flags[k])
            if metered[owner[k]]:
                f |= abi.RESP_METERED
                if owner[k] % 2:
                    d = d.replace(b'"delta":{"content":', b'"delta":{"reasoning_content":')
            docs.append(d)
            flags.append(f)
        resp = ResponseBatch.from_lists(docs, resp.qos.tolist(), flags, now)
        c = g.handle_response_body(resp)
        m = [(f & METERED_CHUNK) == METERED_CHUNK for f in flags]
        d = o.response_batch(resp, counts=_expected_counts(tok, c.bpe_count, docs, m, [bool(f & abi.RESP_STREAM) for f in flags]))
        _same(c, d, ("response", step))
        assert not np.any(c.counted[np.array(m)])
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), step
        assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), step
        assert np.array_equal(g.snapshot_metrics(), o.snapshot_metrics()), step
    assert n_metered > 1000
    # switch off: the same traffic is decided as the reference decides it
    g.set_stream_metering(False)
    o.set_stream_metering(False)
    req, _ = _metered_traffic(w, 3000, NOW + 10, 99)
    a, want = g.handle_request_body(req), o.request_batch(req)
    _same(a, want, "off")
    assert np.sum(a.reason == abi.R_STREAM_OPTIONS) > 300


@pytest.mark.gpu
def test_gpu_metering_adds_no_launch_without_metered_rows(gwmod):
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    w = traffic.Workload(n_tenants=100, seed=5)
    g = gwmod.Gateway(0, 4096, 16 << 20)
    g.load_tables(w.tables)
    g.load_bpe(bpe.load_tokenizer(text))

    def launches(fn):
        before = g.launch_count
        out = fn()
        return g.launch_count - before, out
    req = w.request_batch(1000, NOW, seed=1, stream_frac=0.5)  # include_usage streams and non-stream requests only
    d_off, a = launches(lambda: g.handle_request_body(req))
    resp = w.response_batch(a, NOW, seed=2)
    r_off, _ = launches(lambda: g.handle_response_body(resp))
    g.set_stream_metering(True)
    d_on, a2 = launches(lambda: g.handle_request_body(w.request_batch(1000, NOW + 1, seed=1, stream_frac=0.5)))
    assert d_on == d_off + 1  # the request meter runs whenever the mode is on
    r_on, _ = launches(lambda: g.handle_response_body(w.response_batch(a2, NOW + 1, seed=2)))
    assert r_on == r_off      # no metered chunk: no launch
    g.set_stream_metering(False)
    d_off2, _ = launches(lambda: g.handle_request_body(w.request_batch(1000, NOW + 2, seed=1, stream_frac=0.5)))
    assert d_off2 == d_off
