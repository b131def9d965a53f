"""Every scan path against hostile bytes past each body's end.

The scan kernels read past the end of a body and mask those bytes off by the body's length: the fast path (mask_scan.cuh)
reads whole 32-byte sectors and keeps the next chunk in its ring for a `\\uXXXX` that straddles a chunk boundary, the warp
path (warp_scan.cuh) bulk-copies the body padded to 16 into shared memory and reads 32 bytes per lane, the exact engine
copies whole 16-byte units up to the padded length, and SseSplit cuts lines 16 bytes at a time. The ABI asks only for
16-byte aligned starts and a `bodies_bytes` that covers the last body; the padding may hold anything, and behind
`bodies_bytes` lies stale device memory. A kernel that reads one byte too far gives the same verdict when that byte is 0
(a NUL after the document is the one trailing byte the decoders accept), so every test here puts bytes there that would
CHANGE the answer: the rest of the document the body was cut from, or a closing quote, brace, bracket, digit, backslash,
newline. The oracle always gets the exact bytes [off, off + len).

CPU part: the host builds read the bytes behind the document from the test's buffer (hostmachine `past=`; the hook
ARKS_HOST_PAST_END of json_common.cuh), for both filters, the exact engine under its three schedules, SseT, the split SSE
path and the BPE scanner.

GPU part (`-m gpu`): every scan path on every staging route the batch size allows, with hostile padding inside
`bodies_bytes` (bodies 32-aligned with poisoned gaps, and packed densely on 16 so that the next body follows), and hostile
bytes behind `bodies_bytes` (a primer batch staged first in the same slot on the same route leaves them there); the staging
route edges; four slots in flight. Combinations (scan path x staging route), `arks_last_staging_route` 0 tiny (<= 16 KiB),
1 small (<= 256 KiB), 2 large:
  requests:  warp (<= 2 048 rows) x {tiny, small, large}, exact engine alone (2 049 - 4 095 rows) x {small, large},
             fast (>= 4 096 rows) x {small, large}                                                       = 7 combinations
  responses: JSON on the same three paths (7), all-SSE (event-parallel and irregular chunks in one batch) x 3, mixed x 3
                                                                                                         = 13 combinations
  each with two layouts (32-aligned starts with poisoned gaps; dense 16-byte packing) and a primer: 80 batches.
Unreachable: the exact engine alone and the fast path on the tiny route (2 049 rows of 16-byte aligned bodies need 32 KiB,
4 096 rows leave 4 bytes each), 6 combinations."""
import json

import numpy as np
import pytest

import hostmachine as hm
import orklib

PAST = 64  # bytes behind a body the drivers may see (a 32-byte sector past the 16-byte padding, and the next chunk)
FILLS = {**{"%r" % c: c for c in (b'"', b"\\", b"}", b"]", b"\n", b"\0")}, **{"digit %d" % d: b"%d" % d for d in range(10)}}


def fixed_pasts(body: bytes):
    """(name, bytes behind the body) for every fixed fill, and 0xA5 ^ p as the host drivers' own default"""
    out = [(k, v * PAST) for k, v in FILLS.items()]
    out.append(("0xA5^p", bytes((0xA5 ^ p) & 0xFF for p in range(len(body), len(body) + PAST))))
    return out


def completing(doc: bytes, cut: int) -> bytes:
    """what follows doc[:cut] when the padding holds the rest of the document, and more of the same text after it"""
    rest = doc[cut:] + doc
    while len(rest) < PAST:
        rest += doc
    return rest[:PAST]


def cuts(doc: bytes):
    """every offset of a short document, the last 48 of a long one (the body is doc[:cut], the full document included)"""
    return range(1, len(doc) + 1) if len(doc) < 256 else range(len(doc) - 48, len(doc) + 1)


def cut_corpus(docs):
    """(body, past) pairs: every cut of every document with the completing padding and every fixed fill"""
    out = []
    for d in docs:
        for c in cuts(d):
            body = d[:c]
            out.append((body, completing(d, c)))
            out += [(body, p) for _, p in fixed_pasts(body)]
    return out


# ---- the documents ----------------------------------------------------------------------------------------------------
def request_docs():
    from arks_b200 import traffic
    from jsonfuzz import Gen
    rng, gen = np.random.default_rng(41), Gen(41)
    docs = [b'{"model":"gpt-4","stream":true,"stream_options":{"include_usage":true}}',
            b'{"model":"m\\u00e9","stream":false,"messages":[{"role":"user","content":"hi \\"there\\"\\\\"}]}',
            b'{"stream":123,"model":"m"}', b'{"model":"\\u1234","stream":null}',
            b'{"messages":[{"content":"hello world"}],"model":"q","stream_options":{"include_usage":false}}']
    docs += [traffic.chat_request_body_varied(rng, 400, stream=bool(k & 1)) for k in range(4)]
    docs += [gen.request() for _ in range(6)]
    return docs


def response_docs():
    from arks_b200 import traffic
    from jsonfuzz import Gen
    rng, gen = np.random.default_rng(42), Gen(42)
    docs = [b'{"model":"m","usage":{"prompt_tokens":12,"completion_tokens":345,"total_tokens":357}}',
            b'{"usage":{"total_tokens":12},"model":"m\\u1234"}', b'{"choices":[{"message":{"content":"ab\\\\c"}}],"usage":{"prompt_tokens":1.5e1}}']
    docs += [traffic.chat_response_body_varied(rng, int(rng.integers(1, 400)), int(rng.integers(1, 500)), 300) for _ in range(4)]
    docs += [gen.response() for _ in range(6)]
    return docs


USAGE_EV = b'data: {"choices":[],"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}\n\n'


def sse_docs():
    from arks_b200 import traffic
    from jsonfuzz import Gen
    rng, gen = np.random.default_rng(43), Gen(43)
    docs = [USAGE_EV, USAGE_EV.replace(b"\n", b"\r\n"), b'data: {"choices":[{"delta":{"content":"x"}}]}\n\n' + USAGE_EV + b"data: [DONE]\n\n",
            b": comment\n" + USAGE_EV, b"event: x\ndata: 1\n\n" + USAGE_EV.replace(b"\n\n", b"\r\r")]
    docs += traffic.sse_response_chunks(rng, 5, 9, 700, 2)
    docs += [gen.sse_chunk() for _ in range(6)]
    return docs


def known_answers():
    """(kind, body, bytes behind it, what the exact bytes mean): the padding would complete the document, and must not"""
    U = b'{"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":12'
    rows = [
        ("resp", U, b"3}}" + b"}" * 20, "error"),                       # 12 continued to 123: a body error, not 123 billed
        ("resp", U + b"}", b"}" * 40, "error"),
        ("resp", U + b"}}", b"3}}" * 10, (1, 2, 12)),
        ("resp", U[:-1] + b"}}", b"2}}" * 10, (1, 2, 1)),
        ("req", b'{"model":"m","stream":tru', b'e}' * 20, "error"),
        ("req", b'{"model":"m","stream":true', b'}' * 40, "error"),
        ("req", b'{"model":"m","stream":1', b'2}' * 20, "error"),
        ("req", b'{"model":"gpt', b'-4"}' * 10, "error"),                # a string closed in the padding
        ("req", b'{"model":"gpt-4"', b'}' * 40, "error"),                # the closing brace in the padding: not admitted
        ("req", b'{"model":"gpt-4"}', b'-x"}' * 10, (b"gpt-4", 0, 0, 0)),
        ("req", b'{"model":"\\u12', b'34"}' * 10, "error"),              # a cut \u escape completed by hex digits
        ("req", b'{"model":"\\u1234"}', b"5" * 40, ("ሴ".encode(), 0, 0, 0)),
        ("req", b'{"model":"ab\\', b'"}' * 20, "error"),                 # a lone backslash
        ("req", b'{"stream_options":{"include_usage":tru', b'e}}' * 10, "error"),
        ("req", b'{"messages":[{"content":"hello wor', b'ld"}]}' * 6, "error"),
        ("sse", USAGE_EV[:-1], b"\n" * PAST, None),                       # the event's blank line in the padding
        ("sse", USAGE_EV[:-2], b"\n\n" * 32, None),                       # its LF and blank line in the padding
        ("sse", USAGE_EV + b"data: [DONE", b"]\n\n" * 20, None),
        ("sse", USAGE_EV[:-2] + b"\r", b"\n\r\n" * 20, None),
        ("sse", b'data: {"choices":[],"usage":{"total_tokens":12', b'3}}\n\n' * 10, None),
    ]
    # kFastMaxLen: bodies of exactly 2 047 and 2 048 bytes whose valid tail is in the padding
    for n in (2047, 2048):
        head = b'{"model":"m","p":"'
        rows.append(("req", head + b"x" * (n - len(head)), b'"}' * 32, "error"))
        rows.append(("req", head + b"x" * (n - len(head) - 2) + b'"}', b"x" * PAST, (b"m", 0, 0, 0)))
        rh = b'{"usage":{"total_tokens":7},"p":"'
        rows.append(("resp", rh + b"x" * (n - len(rh)), b'"}' * 32, "error"))
        rows.append(("resp", rh + b"x" * (n - len(rh) - 2) + b'"}', b'9}' * 32, (0, 0, 7)))
    return rows


# ---- CPU: the host builds with chosen bytes behind the body ----------------------------------------------------------
def check_request(body, past):
    ref = orklib.parse_request_body(body)
    for sched in (0, 1, 8):
        hm.set_evsync(sched)
        got = hm.parse_request_body(body, past)
        assert got[0] == ref[0] and (got[0] or got == ref), ("engine, schedule", sched, body[-40:], past[:16], got, ref)
    hm.set_evsync(0)
    e = hm.engine_request(body, past)
    assert (e is not None) == (ref[0] == 0) and e == hm.engine_request(body), (body[-40:], past[:16], e)
    for f in (hm.fast_request, hm.warp_request):
        r = f(body, past)
        assert r is None or r == e, (f.__name__, body[-40:], past[:16], r, e)
        assert (r is None) == (f(body) is None), (f.__name__, "declines depending on the padding", body[-40:], past[:16])
    return ref


def check_response(body, past):
    ref = orklib.parse_response_body(body)
    for sched in (0, 1, 8):
        hm.set_evsync(sched)
        rc, nonempty, u = hm.parse_response_body(body, past)
        assert rc == ref[0] and (rc or (u == ref[2] and nonempty == (ref[1] > 0))), ("engine", sched, body[-40:], past[:16], rc, u, ref)
    hm.set_evsync(0)
    e = hm.engine_response(body, past)
    assert (e is not None) == (ref[0] == 0) and e == hm.engine_response(body), (body[-40:], past[:16], e)
    assert e is None or e[1] == ref[2]
    for f in (hm.fast_response, hm.warp_response):
        r = f(body, past)
        assert r is None or r == e, (f.__name__, body[-40:], past[:16], r, e)
        assert (r is None) == (f(body) is None), (f.__name__, "declines depending on the padding", body[-40:], past[:16])
    return ref


def check_sse(body, past):
    ref = orklib.parse_sse_chunk(body)
    assert hm.parse_sse_chunk(body, past) == ref, ("SseT", body[-40:], past[:16], ref)
    rc, u, _ = hm.parse_sse_chunk_split(body, past)
    assert (rc, u) == ref, ("SseSplit", body[-40:], past[:16], rc, u, ref)
    return ref


CHECK = {"req": check_request, "resp": check_response, "sse": check_sse}


@pytest.mark.parametrize("kind,docs", [("req", request_docs), ("resp", response_docs), ("sse", sse_docs)])
def test_cut_documents_with_completing_and_fixed_padding(kind, docs):
    """every cut of generated documents, the rest of the document behind the cut and every fixed fill: the engine under
    all three schedules, SseT and the split SSE path equal the oracle on the exact bytes; the filters equal the engine or
    decline"""
    n = 0
    for body, past in cut_corpus(docs()):
        CHECK[kind](body, past)
        n += 1
    assert n > 2000


def test_known_answers():
    """the written-out cases: a number, a string, a `\\u` escape or an SSE line completed by the padding"""
    for kind, body, past, want in known_answers():
        for p in [past] + [q for _, q in fixed_pasts(body)]:
            ref = CHECK[kind](body, p)
            if want == "error":
                assert ref[0] == 1, (body[-40:], ref)
            elif kind == "resp":
                assert ref[0] == 0 and ref[2] == want, (body[-40:], ref)
            elif kind == "req":
                assert ref[0] == 0 and (ref[1],) + tuple(ref[2:]) == want, (body[-40:], ref)
    # the SSE rows in the terms of the reference's line scanner: an event is dispatched by its blank line only, so none of
    # the cut usage events bills anything, and `data: [DONE` is not [DONE]
    assert orklib.parse_sse_chunk(USAGE_EV[:-1]) == (0, (0, 0, 0)) and orklib.parse_sse_chunk(USAGE_EV) == (0, (3, 4, 7))


@pytest.fixture(scope="module")
def qwen():
    from arks_b200 import bpe
    from test_bpe import BUILD
    pytest.importorskip("tokenizers")
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    tables = bpe.load_tokenizer(text)
    hm.bpe_load(tables)
    return tok, tables


def referee_count(tok, body: bytes, sse: bool):
    """tokenizers' count of the `content` strings, None when the body is not a whole JSON document"""
    from arks_b200 import bpe
    try:
        strings = bpe.sse_content_strings(body) if sse else bpe.content_strings(body)
    except ValueError:
        return None
    return sum(len(tok.encode(s, add_special_tokens=False).ids) for s in strings)


def test_bpe_count_ignores_the_padding(qwen):
    """the BPE scanner (bpe_scan_body) counts the same for every byte behind the body, and what `tokenizers` counts on the
    exact bytes whenever they are a whole document"""
    tok, _ = qwen
    docs = [(d, False) for d in request_docs() + response_docs()] + [(d, True) for d in sse_docs()]
    docs += [(b, k == "sse") for k, b, _, _ in known_answers()]
    n_ref = 0
    for d, sse in docs:
        for c in cuts(d):
            body = d[:c]
            counts = {hm.bpe_count(body, p) for p in [completing(d, c)] + [q for _, q in fixed_pasts(body)]}
            assert len(counts) == 1, (body[-40:], counts)
            want = referee_count(tok, body, sse) if (not sse or c == len(d)) else None
            if want is not None and counts != {0xFFFFFFFF}:
                assert counts == {want}, (body[-40:], counts, want)
                n_ref += 1
    assert n_ref > 20


# ------------------------------------------------------------------------------------------------------------------
# GPU part
# ------------------------------------------------------------------------------------------------------------------
NOW = 1_700_000_000
N_TENANTS = 8
TINY, SMALL = 16 << 10, 256 << 10  # arks_gateway.cu kTinyBatchBytes, kSmallBatchBytes
MAX_BATCH, MAX_BATCH_BYTES = 8192, 4 << 20
UNC = 0xFFFFFFFF


def align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


def meta_cap(max_batch: int) -> int:
    """the metadata block of a slot (arks_create): four 4-byte columns, pick_rand, flags, 256 token bytes per row, 256 KiB"""
    n = max_batch
    return align(4 * n, 256) * 4 + align(8 * n, 256) + align(n, 256) + align(256 * n, 256) + SMALL + 256


def request_meta(n: int, tok_bytes: int) -> int:
    return align(4 * n, 256) * 2 + align(4 * (n + 1), 256) + align(8 * n, 256) + align(tok_bytes + 1, 256)


def expected_route(kind: str, n: int, bodies_bytes: int, tok_bytes: int = 0, max_batch: int = MAX_BATCH) -> int:
    """this test's own copy of the staging rule, checked against arks_last_staging_route"""
    small = bodies_bytes <= SMALL and (kind != "req" or request_meta(n, tok_bytes) + bodies_bytes <= meta_cap(max_batch))
    return (0 if bodies_bytes <= TINY else 1) if small else 2


def pack_hostile(rows, layout: str):
    """rows: [(body, bytes behind it)]. 'a32': every body starts on a 32-byte boundary and the gap behind it holds the
    start of its hostile bytes; 'dense16': every body starts at the next 16-byte boundary, behind its padding comes the
    next body. bodies_bytes ends at the last body padded to 16. -> (buf, off, len, the last body's bytes behind
    bodies_bytes)"""
    buf, off, lens = bytearray(), [], []
    for i, (b, p) in enumerate(rows):
        p = (p * (PAST // len(p) + 1))[:PAST]  # a short pattern repeated
        off.append(len(buf))
        lens.append(len(b))
        buf += b
        k = align(len(buf), 16 if layout == "dense16" or i == len(rows) - 1 else 32) - len(buf)
        buf += p[:k]
    tail = rows[-1][1][k:]
    return np.frombuffer(bytes(buf), np.uint8).copy(), np.array(off, np.uint32), np.array(lens, np.uint32), tail


def with_bodies(batch, buf):
    import copy
    b = copy.copy(batch)
    b.bodies = buf
    return b


def req_filler(size: int) -> bytes:
    head = b'{"model":"m","p":"'
    return head + b"x" * (size - len(head) - 2) + b'"}'


def resp_filler(size: int) -> bytes:
    head = b'{"usage":{"prompt_tokens":2,"completion_tokens":3,"total_tokens":5},"p":"'
    return head + b"x" * (size - len(head) - 2) + b'"}'


SSE_FILLER = USAGE_EV


def gpu_rows(kind: str):
    """the hostile rows of one side: the known answers with every fill, every cut with the completing bytes and one of the
    fixed fills in turn"""
    docs = {"req": request_docs, "resp": response_docs, "sse": sse_docs}[kind]()
    rows = []
    for k, b, p, _ in known_answers():
        if k == kind:
            rows += [(b, p)] + [(b, q) for _, q in fixed_pasts(b)]
    for d in docs:
        for j, c in enumerate(cuts(d)):
            rows.append((d[:c], completing(d, c)))
            rows.append((d[:c], fixed_pasts(d[:c])[j % len(FILLS)][1]))
    return rows


def fit_rows(corpus, n: int, route: int, small_filler: bytes, big_filler: bytes, seed: int):
    """n rows on the given route: as many hostile rows as the route's byte budget leaves room for, small valid fillers up
    to n rows (three large ones on the large route), shuffled, and a hostile row last (its bytes go past bodies_bytes)"""
    cap = {0: TINY - 2 * PAST, 1: SMALL - 2 * PAST, 2: 1 << 40}[route]
    n_big = 3 if route == 2 else 0
    rows, used, fc = [], 0, align(len(small_filler), 32)
    for r in corpus:
        c = align(len(r[0]), 32) + 32
        if len(rows) + n_big + 1 >= n or used + c + fc * (n - len(rows)) > cap:
            break
        rows.append(r)
        used += c
    last = rows.pop()
    rows += [(big_filler, b"}" * PAST)] * n_big
    rows += [(small_filler, b"}" * PAST)] * (n - len(rows) - 1)
    order = np.random.default_rng(seed).permutation(len(rows))
    return [rows[i] for i in order] + [last]


def gpu_tables():
    from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token
    toks = [simple_token("u%d" % i, "ns", "tk-%d" % i, "m", [("rpm", 10**9), ("tpm", 10**15), ("tpd", 10**16)], "q" if i % 2 else "")
            for i in range(N_TENANTS)]
    return Tables(toks, [simple_quota("q", "ns", [("prompt", 10**15), ("response", 10**15), ("total", 10**15)])], [simple_endpoint("m", "ns")])


class Bench:
    """one device context and the oracle behind it, with the stand-in vocabulary loaded and the metrics on"""

    def __init__(self, gwmod, tables, max_batch=MAX_BATCH, max_batch_bytes=MAX_BATCH_BYTES, vocab=None):
        self.g = gwmod.Gateway(0, max_batch, max_batch_bytes)
        self.g.load_tables(tables)
        self.g.enable_metrics(True)
        if vocab is not None:
            self.g.load_bpe(vocab)
        self.o = orklib.Oracle(tables)
        self.now = NOW
        self.bpe = vocab is not None

    def state(self, ctx):
        g, o = self.g, self.o
        assert np.array_equal(g.snapshot_rate(self.now), o.snapshot_rate(self.now)), ctx + ": rate counters differ"
        assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), ctx + ": quota usage differs"
        assert np.array_equal(g.snapshot_metrics(), o.snapshot_metrics()), ctx + ": metrics differ"

    def run(self, kind, batch, ctx, route=None):
        """one batch on the device and the oracle: every result field, the counters, the route; -> (result, declined)"""
        from arks_b200 import abi
        self.now += 61
        batch.now_unix = self.now
        if kind == "req":
            a, b = self.g.handle_request_body(batch), self.o.request_batch(batch)
        else:
            a, b = self.g.handle_response_body(batch), self.o.response_batch(batch)
        got_route, declined = self.g.last_staging_route, self.g.last_declined
        for k, v in a.fields().items():
            w = b.fields()[k]
            if v is not None and not np.array_equal(v, w):
                bad = np.flatnonzero((v != w).reshape(len(v), -1).any(axis=1))
                i = int(bad[0])
                body = bytes(batch.bodies[batch.body_off[i]:batch.body_off[i] + batch.body_len[i]])
                raise AssertionError(f"{ctx} field {k}: {len(bad)} rows differ, first {bad[:5]}: gpu={v[bad[:5]]} oracle={w[bad[:5]]} body {body[-60:]!r}")
        self.state(ctx)
        if route is not None:
            assert got_route == route, (ctx, "staging route", got_route, route)
        if self.bpe and a.bpe_count is not None:
            for i in range(batch.n):
                body = bytes(batch.bodies[batch.body_off[i]:batch.body_off[i] + batch.body_len[i]])
                if kind == "req":
                    ok = a.reason[i] != abi.R_REQUEST_BODY
                else:
                    sse = bool(batch.flags[i] & abi.RESP_STREAM)
                    ok = (orklib.parse_sse_chunk(body) if sse else orklib.parse_response_body(body))[0] == 0 and batch.qos[i] >= 0
                if ok:
                    assert a.bpe_count[i] == hm.bpe_count(body), (ctx, i, body[-60:], int(a.bpe_count[i]), hm.bpe_count(body))
        return a, declined

    def run_hostile(self, kind, make, rows, route, ctx):
        """both layouts, each behind a primer that leaves the last body's hostile bytes behind bodies_bytes in the slot"""
        out = []
        for layout in ("a32", "dense16"):
            buf, off, lens, tail = pack_hostile(rows, layout)
            batch = make(buf, off, lens)
            primer = with_bodies(batch, np.concatenate([buf, np.frombuffer((tail + b"}" * PAST)[:PAST], np.uint8)]))
            assert expected_route(kind, batch.n, len(buf) + PAST, tok_bytes(batch)) == route == expected_route(kind, batch.n, len(buf), tok_bytes(batch)), ctx
            self.run(kind, primer, f"{ctx} {layout} primer", route)
            out.append(self.run(kind, batch, f"{ctx} {layout}", route))
        return out


def tok_bytes(batch) -> int:
    return int(batch.token_off[-1]) if hasattr(batch, "token_off") else 0


def make_request(n):
    from arks_b200 import abi
    from arks_b200.abi import RequestBatch
    tb, to = abi.pack_concat([b"tk-%d" % (i % N_TENANTS) for i in range(n)])
    return lambda buf, off, lens: RequestBatch(buf, off, lens, tb, to, NOW)


def make_response(flags):
    from arks_b200.abi import ResponseBatch
    n = len(flags)
    qos = np.array([i % N_TENANTS for i in range(n)], np.int32)
    return lambda buf, off, lens: ResponseBatch(buf, off, lens, qos, np.array(flags, np.uint8), NOW)


# (rows, scan path it takes, route): warp <= 2 048 rows, exact engine alone 2 049 - 4 095, fast path >= 4 096
REQ_CASES = [(100, "warp", 0), (1000, "warp", 1), (1000, "warp", 2), (2049, "exact", 1), (3000, "exact", 2),
             (4096, "fast", 1), (4500, "fast", 2)]


def host_declines(rows, path, kind):
    if path == "exact":
        return -1
    f = {("warp", "req"): hm.warp_request, ("fast", "req"): hm.fast_request, ("warp", "resp"): hm.warp_response,
         ("fast", "resp"): hm.fast_response}[path, kind]
    return sum(1 for b, _ in rows if f(b) is None)


@pytest.fixture(scope="module")
def vocab():
    from arks_b200 import bpe
    from test_bpe import BUILD
    pytest.importorskip("tokenizers")
    _, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    tables = bpe.load_tokenizer(text)
    hm.bpe_load(tables)
    return tables


@pytest.mark.gpu
def test_requests_hostile_bytes_every_path_and_route_gpu(gwmod, vocab):
    """requests: warp path, exact engine alone and fast path on every staging route their row counts allow, hostile bytes
    in the padding, the next body behind the padding, stale hostile bytes behind bodies_bytes; every field, bpe_count, the
    counters and the metrics equal the oracle; the path proven by last_declined (exactly the rows its filter declines on
    the host, -1 for the exact engine alone)"""
    t = Bench(gwmod, gpu_tables(), vocab=vocab)
    corpus = gpu_rows("req")
    for n, path, route in REQ_CASES:
        rows = fit_rows(corpus, n, route, req_filler(13) if n > 2048 else req_filler(40), req_filler(100_000), n)
        for a, declined in t.run_hostile("req", make_request(n), rows, route, f"requests n={n} {path} route {route}"):
            assert declined == host_declines(rows, path, "req"), (n, path, declined)
        corpus = corpus[len(rows) // 3:] + corpus[:len(rows) // 3]  # the next case starts elsewhere in the corpus


RESP_CASES = [(100, "warp", 0), (1000, "warp", 1), (1000, "warp", 2), (2049, "exact", 1), (3000, "exact", 2),
              (4096, "fast", 1), (4500, "fast", 2)]


@pytest.mark.gpu
def test_responses_hostile_bytes_every_path_and_route_gpu(gwmod, vocab):
    """responses: complete JSON bodies on the three scan paths, all-SSE batches (regular chunks on the event-parallel
    lane, CR and comment chunks on the sequential one) and mixed batches, on every staging route; usage, counted,
    reason, bpe_count, counters and metrics equal the oracle"""
    from arks_b200 import abi
    t = Bench(gwmod, gpu_tables(), vocab=vocab)
    json_rows, sse_rows = gpu_rows("resp"), gpu_rows("sse")
    for n, path, route in RESP_CASES:
        small = b'{"usage":{"total_tokens":5}}' if n > 2048 else resp_filler(80)
        rows = fit_rows(json_rows, n, route, small, resp_filler(100_000), n)
        for _, declined in t.run_hostile("resp", make_response([abi.RESP_END_OF_STREAM] * n), rows, route, f"JSON n={n} {path} route {route}"):
            assert declined == host_declines(rows, path, "resp"), (n, path, declined)
        json_rows = json_rows[len(rows) // 3:] + json_rows[:len(rows) // 3]
    big_sse = USAGE_EV * 1200
    for n, route in ((100, 0), (600, 1), (600, 2)):
        rows = fit_rows(sse_rows, n, route, SSE_FILLER, big_sse, n)
        t.run_hostile("sse", make_response([abi.RESP_STREAM] * n), rows, route, f"all-SSE n={n} route {route}")
        mixed = fit_rows([r for pair in zip(sse_rows, json_rows) for r in pair], n, route, SSE_FILLER, big_sse, n + 1)
        flags = [abi.RESP_END_OF_STREAM if b.startswith(b"{") else abi.RESP_STREAM for b, _ in mixed]
        assert 0 < flags.count(abi.RESP_STREAM) < n
        t.run_hostile("resp", make_response(flags), mixed, route, f"mixed n={n} route {route}")
        sse_rows = sse_rows[n // 2:] + sse_rows[:n // 2]


def sse_filler(size: int) -> bytes:
    return USAGE_EV[:-2] + b" " * (size - len(USAGE_EV)) + b"\n\n"


def sized_rows(total: int, filler, rows: int = 40):
    """`rows` valid bodies packed on 32 and a buffer of exactly `total` bytes (the last body ends inside it) -> buf, off, len"""
    base = [filler(100)] * (rows - 1)
    used = align(100, 32) * (rows - 1)
    last = filler(min(total - used, 90_000))
    bodies = base + [last]
    from arks_b200 import abi
    buf, off, lens = abi.pack_blobs(bodies)
    out = np.full(total, ord("}"), np.uint8)  # hostile bytes in every gap and behind the last body
    for o, l in zip(off, lens):
        out[o:o + l] = buf[o:o + l]
    assert int(off[-1]) + int(lens[-1]) <= total
    return out, off, lens


@pytest.mark.gpu
def test_staging_route_edges_gpu(gwmod):
    """both sides of every staging edge, results and counters equal to the oracle, the route asserted: bodies_bytes 16 384 /
    16 385 and 262 144 / 262 145 for requests and each response mode, with and without `precharged`; a request whose
    metadata and bodies fill the metadata block exactly, and 16 bytes more; token bytes at capacity and one over; max_batch
    and one more row; bodies_bytes == max_bytes and one more; kZeroCopyRows 2 048 / 2 049 rows with the optional outputs
    NULL and set; a refused batch stages nothing, moves no counter, and the next batch is exact"""
    from arks_b200 import abi
    from arks_b200.abi import RequestBatch, RequestResult, ResponseBatch, ResponseResult
    from arks_b200.gateway import ArksError
    max_batch, max_batch_bytes = 4096, 1 << 20
    max_bytes = align(max_batch_bytes + 16, 256)
    t = Bench(gwmod, gpu_tables(), max_batch, max_batch_bytes)
    g = t.g
    for total, route in ((TINY, 0), (TINY + 1, 1), (SMALL, 1), (SMALL + 1, 2), (max_bytes, 2)):
        buf, off, lens = sized_rows(total, req_filler)
        req = make_request(len(off))(buf, off, lens)
        assert expected_route("req", req.n, total, tok_bytes(req), max_batch) == route
        t.run("req", req, f"requests, bodies_bytes {total}", route)
        for mode in ("json", "sse", "mixed"):
            fl = {"json": [abi.RESP_END_OF_STREAM] * 40, "sse": [abi.RESP_STREAM] * 40, "mixed": [abi.RESP_STREAM, abi.RESP_END_OF_STREAM] * 20}[mode]
            buf, off, lens = sized_rows(total, sse_filler if mode == "sse" else resp_filler)
            if mode == "mixed":
                for i in range(0, 40, 2):  # the SSE rows of a mixed batch: one usage event in the same room
                    buf[off[i]:off[i] + lens[i]] = np.frombuffer(sse_filler(int(lens[i])), np.uint8)
            for pre in (None, np.full(40, 3, np.uint32)):
                resp = make_response(fl)(buf, off, lens)
                resp.precharged = pre
                t.run("resp", resp, f"{mode} responses, bodies_bytes {total}, precharged {pre is not None}", route)
    # bodies_bytes beyond max_bytes (= align_up(max_batch_bytes + 16, 256)): refused as a whole
    buf, off, lens = sized_rows(max_bytes + 1, req_filler)
    before = (g.snapshot_rate(t.now), g.snapshot_quota(), g.snapshot_metrics())
    with pytest.raises(ArksError) as e:
        g.handle_request_body(make_request(len(off))(buf, off, lens))
    assert e.value.code == abi.E_CAPACITY and g.last_staging_route == -1
    with pytest.raises(ArksError):
        g.run_request(t.now + 1)  # the slot was left unstaged: its previous batch is not run again
    resp = make_response([abi.RESP_END_OF_STREAM] * len(off))(buf, off, lens)
    with pytest.raises(ArksError) as e:
        g.handle_response_body(resp)
    assert e.value.code == abi.E_CAPACITY and g.last_staging_route == -1
    with pytest.raises(ArksError):
        g.run_response(t.now + 1)
    after = (g.snapshot_rate(t.now), g.snapshot_quota(), g.snapshot_metrics())
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    # metadata + bodies exactly fill the metadata block (long bearer tokens), and 16 bytes more take the large route
    n = 64
    fixed = request_meta(n, 0) - align(1, 256)
    for extra, route in ((0, 1), (16, 2)):
        bb = 204_800 + extra
        tok_len = meta_cap(max_batch) - bb - fixed - 1
        toks = [b"tk-%d" % (i % N_TENANTS) for i in range(n - 1)]
        toks.append(b"x" * (tok_len - sum(len(x) for x in toks)))
        tb, to = abi.pack_concat(toks)
        buf, off, lens = sized_rows(bb, req_filler, n)
        req = RequestBatch(buf, off, lens, tb, to, NOW)
        assert request_meta(n, tok_len) + 204_800 == meta_cap(max_batch)
        assert expected_route("req", n, bb, tok_len, max_batch) == route
        t.run("req", req, f"metadata block full + {extra}", route)
    # token bytes at the capacity of the metadata block, and one over
    for over in (0, 1):
        tok_len = meta_cap(max_batch) - fixed - 1 + over
        toks = [b"tk-%d" % (i % N_TENANTS) for i in range(n - 1)]
        toks.append(b"y" * (tok_len - sum(len(x) for x in toks)))
        tb, to = abi.pack_concat(toks)
        buf, off, lens = sized_rows(16384, req_filler, n)
        req = RequestBatch(buf, off, lens, tb, to, NOW)
        if over:
            with pytest.raises(ArksError) as e:
                g.handle_request_body(req)
            assert e.value.code == abi.E_CAPACITY and g.last_staging_route == -1
        else:
            t.run("req", req, "token bytes at capacity", 2)
    # rows: max_batch and one more
    for rows, ok in ((max_batch, True), (max_batch + 1, False)):
        bodies = [req_filler(20)] * rows
        req = RequestBatch.from_lists(bodies, [b"tk-%d" % (i % N_TENANTS) for i in range(rows)], NOW)
        if ok:
            t.run("req", req, "max_batch rows", 1)
        else:
            with pytest.raises(ArksError) as e:
                g.handle_request_body(req)
            assert e.value.code == abi.E_CAPACITY
            with pytest.raises(ArksError):
                g.run_request(t.now + 1)
    t.state("after the refused batches")
    # kZeroCopyRows: the result rows in the pinned block (<= 2 048) or copied back, optional outputs NULL and set
    for rows in (2048, 2049):
        for optional in (False, True):
            req = RequestBatch.from_lists([req_filler(30 + i % 50) for i in range(rows)], [b"tk-%d" % (i % N_TENANTS) for i in range(rows)], NOW)
            t.now += 61
            req.now_unix = t.now
            out = RequestResult.empty(rows)
            if not optional:
                out.model_off = out.model_len = out.bpe_count = None
            a, b = g.handle_request_body(req, out), t.o.request_batch(req)
            for k, v in a.fields().items():
                assert v is None or np.array_equal(v, b.fields()[k]), (rows, optional, k)
            t.state(f"zero-copy edge {rows}")
            resp = ResponseBatch.from_lists([resp_filler(90 + i % 40) for i in range(rows)], [i % N_TENANTS for i in range(rows)], [abi.RESP_END_OF_STREAM] * rows, t.now)
            out = ResponseResult.empty(rows)
            if not optional:
                out.bpe_count = None
            c, d = g.handle_response_body(resp, out), t.o.response_batch(resp)
            for k, v in c.fields().items():
                assert np.array_equal(v, d.fields()[k]), (rows, optional, k)
            t.state(f"zero-copy edge {rows} responses")


@pytest.mark.gpu
def test_four_slots_in_flight_gpu(gwmod):
    """request batches on all four slots at once, on the tiny, small and large routes, zero-copy (<= 2 048 rows) and copied
    results mixed, a response batch in the same slot right behind each request; waited for in another order than they were
    submitted, then every slot reused, so each batch finds its slot's previous tenant's hostile bytes. Results and counters
    equal the serial oracle in submission order"""
    from arks_b200 import abi
    from arks_b200.abi import RequestResult, ResponseResult
    t = Bench(gwmod, gpu_tables())
    g, o = t.g, t.o
    req_rows, resp_rows = gpu_rows("req"), gpu_rows("resp")
    plan = [(100, 0), (1000, 1), (3000, 2), (2500, 1)]
    for cycle in range(2):
        subs = []
        for slot, (n, route) in enumerate(plan):
            t.now += 7
            rows = fit_rows(req_rows, n, route, req_filler(13) if n > 2048 else req_filler(40), req_filler(100_000), 10 * cycle + slot)
            buf, off, lens, tail = pack_hostile(rows, "dense16" if (slot + cycle) % 2 else "a32")
            req = make_request(n)(buf, off, lens)
            req.now_unix = t.now
            g.select_slot(slot)
            g.submit_request_async(req)
            assert g.last_staging_route == route
            rrows = fit_rows(resp_rows, n, route, b'{"usage":{"total_tokens":5}}' if n > 2048 else resp_filler(80), resp_filler(100_000), 20 * cycle + slot)
            rbuf, roff, rlens, _ = pack_hostile(rrows, "a32")
            resp = make_response([abi.RESP_END_OF_STREAM] * n)(rbuf, roff, rlens)
            resp.now_unix = t.now
            g.submit_response_async(resp)
            subs.append((slot, req, resp, RequestResult.empty(n), ResponseResult.empty(n)))
            req_rows = req_rows[n // 4:] + req_rows[:n // 4]
            resp_rows = resp_rows[n // 4:] + resp_rows[:n // 4]
        for slot, req, resp, ra, rb in [subs[k] for k in (2, 0, 3, 1)]:
            g.wait_request(slot, ra)
            g.wait_response(slot, rb)
        for slot, req, resp, ra, rb in subs:
            want = o.request_batch(req)
            for k, v in ra.fields().items():
                assert np.array_equal(v, want.fields()[k]), (cycle, slot, k)
            want = o.response_batch(resp)
            for k, v in rb.fields().items():
                assert np.array_equal(v, want.fields()[k]), (cycle, slot, "response", k)
        t.state(f"four slots, cycle {cycle}")
