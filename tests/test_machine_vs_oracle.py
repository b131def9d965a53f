"""Differential fuzz on CPU: the device byte state machines (arks_b200/csrc/json_engine.cuh, compiled for the host
by tests/host_machine.cpp) against the oracle's function-by-function restatement of jsoniter / ssestream / gjson
(oracle/ork_json.c). Any disagreement on (error?, model bytes, stream flags, usage ints) fails."""
import random

import pytest

import hostmachine as hm
import orklib
from jsonfuzz import Gen

@pytest.mark.parametrize("seed", [11, 12])
def test_request_body_machine(seed):
    g = Gen(seed)
    for _ in range(30000):
        b = g.request()
        a, c = orklib.parse_request_body(b), hm.parse_request_body(b)
        assert a[0] == c[0] and (a[0] == 1 or a == c), (b, a, c)


@pytest.mark.parametrize("seed", [21, 22])
def test_response_body_machine(seed):
    g = Gen(seed)
    for _ in range(30000):
        b = g.response()
        a, c = orklib.parse_response_body(b), hm.parse_response_body(b)
        assert a[0] == c[0], (b, a, c)
        if a[0] == 0:
            assert (a[1] > 0, a[2]) == (c[1] > 0, c[2]), (b, a, c)


@pytest.mark.parametrize("seed", [31, 32])
def test_sse_chunk_machine(seed):
    g = Gen(seed)
    for _ in range(30000):
        b = g.sse_chunk()
        a, c = orklib.parse_sse_chunk(b), hm.parse_sse_chunk(b)
        assert a[0] == c[0] and (a[0] == 1 or a == c), (b, a, c)


@pytest.mark.parametrize("seed", [33, 34])
def test_sse_chunk_split_path(seed):
    """SseSplit + per-event parse + in-order combine gives the oracle's verdict on every chunk, whether the chunk is
    regular (event-parallel path) or not (falls back to the sequential machine); both paths must be exercised."""
    g = Gen(seed)
    n_reg = n_irr = 0
    for it in range(30000):
        b = g.sse_chunk()
        if it % 3 == 0:  # the fuzzer likes CR LF and odd fields; make a share of the corpus look like real servers
            b = b.replace(b"\r\n", b"\n").replace(b"data:  ", b"data: ")
        if it % 7 == 0:
            b = b": ping\n\n".join([b] * 1) + b""
        a = orklib.parse_sse_chunk(b)
        rc, usage, fell_back = hm.parse_sse_chunk_split(b)
        n_irr += fell_back
        n_reg += not fell_back
        assert a[0] == rc and (rc == 1 or a[1] == usage), (b, a, rc, usage, fell_back)
    assert n_reg > 3000 and n_irr > 3000, (n_reg, n_irr)


def test_sse_split_cases():
    ev = b'{"id":"x","choices":[],"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'
    ch = b'{"id":"x","choices":[{"index":0,"delta":{"content":"hi"}}],"usage":null}'
    cases = [
        b"data: " + ch + b"\n\ndata: " + ev + b"\n\ndata: [DONE]\n\n",
        b"data: " + ev + b"\n\ndata: [DONE]\n\ndata: {broken\n\n",       # nothing after [DONE] is parsed
        b"data: " + ev + b"\n\ndata: {broken\n\ndata: [DONE]\n\n",       # a bad event before it fails the stream
        b"data:" + ev + b"\n\n",                                           # no space after the colon
        b"data: " + ev + b"\n",                                             # never dispatched
        b"data: " + ev + b"\n\n\n",                                        # empty event -> not JSON
        b": comment\ndata: " + ev + b"\n: another\n\n",
        b"data: " + ev + b"\ndata: x\n\n",                                 # multi-line data (irregular)
        b"data: " + ev + b"\r\n\r\n",                                      # CR LF (irregular)
        b"event: thread.run\ndata: " + ev + b"\n\n",                       # wrapped event (irregular)
        b"data: [DONE] trailing\n\ndata: " + ev + b"\n\n",                # HasPrefix("[DONE]")
        b"data: [DONE\n\ndata: " + ev + b"\n\n",
        b"data: \n\n", b"data:\n\n", b"data\n\n", b"\n", b"", b"data: 5\n\n", b"data: null\n\n",
        b"x" * 15 + b"\n",
    ]
    for pad in range(0, 20):  # every alignment of the line starts against the 16-byte units
        for c in cases:
            b = b": " + b"p" * pad + b"\n" + c
            a = orklib.parse_sse_chunk(b)
            rc, usage, _ = hm.parse_sse_chunk_split(b)
            assert a[0] == rc and (rc == 1 or a[1] == usage), (b, a, rc, usage)
    ok = b"data: " + b'{"a":"' + b"x" * 65000 + b'"}\n\n'
    bad = b"data: " + b'{"a":"' + b"x" * 65600 + b'"}\n\n'
    tail = b"data: [DONE]\n\n" + b"y" * 70000
    assert hm.parse_sse_chunk_split(ok)[0] == 0 and hm.parse_sse_chunk_split(bad)[0] == 1
    assert hm.parse_sse_chunk_split(tail)[0] == orklib.parse_sse_chunk(tail)[0] == 1


@pytest.mark.parametrize("mode", [1, 4, 8])
def test_other_schedules_same_results(mode):
    """consume_evsync / consume_rounds<R> are only different schedules of the same machine."""
    hm.set_evsync(mode)
    try:
        g = Gen(41 + mode)
        for _ in range(8000):
            b = g.request()
            a, c = orklib.parse_request_body(b), hm.parse_request_body(b)
            assert a[0] == c[0] and (a[0] == 1 or a == c), (b, a, c)
            b = g.response()
            a, c = orklib.parse_response_body(b), hm.parse_response_body(b)
            assert a[0] == c[0] and (a[0] == 1 or (a[1] > 0, a[2]) == (c[1] > 0, c[2])), (b, a, c)
            b = g.sse_chunk().replace(b"\r\n", b"\n")
            a = orklib.parse_sse_chunk(b)
            rc, usage, _ = hm.parse_sse_chunk_split(b)
            assert a[0] == rc and (rc == 1 or a[1] == usage), (b, a, rc, usage)
        r = random.Random(5)
        for _ in range(300):
            b = _long_doc(r, "req")
            a, c = orklib.parse_request_body(b), hm.parse_request_body(b)
            assert a[0] == c[0] and (a[0] == 1 or a == c), (b, a, c)
    finally:
        hm.set_evsync(False)


CASES_REQ = [
    (b'{"model":"a","model":null}', (0, b"", 0, 0, 0)),                      # last duplicate wins, null -> ""
    (b'{"MODEL":"a"}', (0, b"a", 0, 0, 0)),                                  # case-insensitive field hash
    (b'{"stream_options":{"include_usage":true},"stream_options":{}}', (0, b"", 0, 1, 2)),   # pointer reuse
    (b'{"stream_options":{"include_usage":true},"stream_options":null}', (0, b"", 0, 0, 0)),
    (b'null', (0, b"", 0, 0, 0)),                                            # readObjectStart accepts null
    (b'{"model":"a"}\x00garbage', (0, b"a", 0, 0, 0)),                       # Unmarshal's `c == 0` quirk
    (b'{"model":"a"} x', (1,)),
    (b'{"a":{"b":1,null:2},"model":"m"}', (0, b"m", 0, 0, 0)),               # ReadObjectCB reads keys with ReadString
    (b'{"a":-01,"model":"m"}', (0, b"m", 0, 0, 0)),                          # trySkipNumber leniency
    (b'{"a":01,"model":"m"}', (1,)),
    (b'{"a":"x\x01","model":"m"}', (1,)),                                    # control char before any backslash
    (b'{"a":"\\n\x01","model":"m"}', (0, b"m", 0, 0, 0)),                    # ... not checked on the slow path
    (b'{"model":"\\ud83d\\ude00"}', (0, "\U0001F600".encode(), 0, 0, 0)),
    (b'{"model":"\\ud800x"}', (0, "\ufffdx".encode(), 0, 0, 0)),
    (b'{"model":"a",}', (1,)),
    (b'', (1,)),
    (b'[]', (1,)),
    (b'{"stream":"true"}', (1,)),
]


@pytest.mark.parametrize("body,want", CASES_REQ)
def test_request_known_answers(body, want):
    for impl in (orklib, hm):
        got = impl.parse_request_body(body)
        if want[0] == 1:
            assert got[0] == 1, (impl.__name__, body, got)
        else:
            assert got == want, (impl.__name__, body, got)


def test_depth_limit_10000():
    deep_ok = b'{"a":' + b"[" * 9999 + b"]" * 9999 + b',"model":"m"}'
    deep_bad = b'{"a":' + b"[" * 10000 + b"]" * 10000 + b',"model":"m"}'
    for impl in (orklib, hm):
        assert impl.parse_request_body(deep_ok)[0] == 0
        assert impl.parse_request_body(deep_bad)[0] == 1


def test_sse_line_limit_64k():
    ok = b"data: " + b'{"a":"' + b"x" * 65000 + b'"}\n\n'
    bad = b"data: " + b'{"a":"' + b"x" * 65600 + b'"}\n\n'
    for impl in (orklib, hm):
        assert impl.parse_sse_chunk(ok)[0] == 0
        assert impl.parse_sse_chunk(bad)[0] == 1


def _long_doc(r, kind):
    """chat-shaped documents whose strings are long and salted with escapes / control bytes / UTF-8 at every alignment:
    exercises the 16-byte skip path of consume()"""
    salt = [b'\\n', b'\\"', b'\\\\', b'\\u00e9', b'\\ud83d\\ude00', b'\xc3\xa9', b'\xe4\xb8\xad', b'"', b'\\', b'\n', b'\x1f', b'\\x',
            b'\\u12', b'\t', b'\r\n', b'\x00', b'/', b'{', b'}', b':', b',', b'[', b']']
    def text(n):
        out = bytearray()
        while len(out) < n:
            out += bytes(r.choice(b"abcdefghijklmnopqrstuvwxyz      .,'-0123456789") for _ in range(r.randint(1, 70)))
            if r.random() < 0.5:
                out += r.choice(salt[:7] if r.random() < 0.8 else salt)
        return bytes(out)
    pad = b" " * r.randint(0, 17)
    if kind == "req":
        return (pad + b'{"model":"qwen-7b","messages":[{"role":"user","content":"' + text(r.randint(0, 900)) + b'"},{"role":"' +
                text(r.randint(0, 40)) + b'","content":"' + text(r.randint(0, 300)) + b'"}],"stream":true}')
    if kind == "resp":
        return (pad + b'{"id":"x","model":"m","choices":[{"message":{"content":"' + text(r.randint(0, 700)) +
                b'"}}],"usage":{"prompt_tokens":12,"completion_tokens":30,"total_tokens":42}}')
    frames = b"".join(b'data: {"choices":[{"delta":{"content":"' + text(r.randint(0, 200)) + b'"}}]}' + r.choice([b"\n\n", b"\r\n\r\n"])
                      for _ in range(r.randint(1, 4)))
    return frames + b'data: {"choices":[],"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}}\n\ndata: [DONE]\n\n'


@pytest.mark.parametrize("seed", [61, 62, 63])
def test_long_strings_bulk_path(seed):
    import random
    r = random.Random(seed)
    n_ok = 0
    for _ in range(6000):
        b = _long_doc(r, "req")
        a, c = orklib.parse_request_body(b), hm.parse_request_body(b)
        assert a[0] == c[0] and (a[0] == 1 or a == c), (b, a, c)
        n_ok += a[0] == 0
        b = _long_doc(r, "resp")
        a, c = orklib.parse_response_body(b), hm.parse_response_body(b)
        assert a[0] == c[0] and (a[0] == 1 or (a[1] > 0, a[2]) == (c[1] > 0, c[2])), (b, a, c)
        b = _long_doc(r, "sse")
        a, c = orklib.parse_sse_chunk(b), hm.parse_sse_chunk(b)
        assert a[0] == c[0] and (a[0] == 1 or a == c), (b, a, c)
    assert n_ok > 500  # the corpus is not all errors


@pytest.mark.parametrize("mode", [0, 1, 8])
def test_client_app_traffic_through_the_engine(mode):
    """the bench's heterogeneous bodies (arks_b200.traffic: client applications, server dialects, escapes, UTF-8) are
    valid for the oracle and give the same extraction in every schedule of the engine"""
    import numpy as np
    from arks_b200 import traffic
    rng = np.random.default_rng(77 + mode)
    hm.set_evsync(mode)
    try:
        for it in range(1500):
            stream = bool(it % 3 == 0)
            b = traffic.chat_request_body_varied(rng, 1024, stream=stream)
            a, c = orklib.parse_request_body(b), hm.parse_request_body(b)
            assert a == c and a[0] == 0 and a[1] == traffic.MODEL.encode() and a[2] == (2 if stream else a[2]), (b, a, c)
            p, q = int(rng.integers(1, 5000)), int(rng.integers(1, 5000))
            b = traffic.chat_response_body_varied(rng, p, q, 600)
            a, c = orklib.parse_response_body(b), hm.parse_response_body(b)
            assert a[0] == c[0] == 0 and a[2] == c[2] == (p, q, p + q), (b, a, c)
    finally:
        hm.set_evsync(0)
