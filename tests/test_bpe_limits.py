"""The on-device BPE count at its limits, where a body must be reported ARKS_BPE_UNCOUNTED instead of a wrong number: the
piece-length limit (kBpeMaxPiece = 128 bytes) and the capacity of the pre-token work list. The referee is always HF
`tokenizers` (token counts of the counted strings, piece lengths from its Split pre-tokenizer); a count the device produced
is never the expectation.

CPU: the host build of bpe.cuh (tests/bpe_vocab_host.cpp) with pieces of 127, 128 and 129 bytes for every alternative of
the Qwen2 and Llama 3 patterns, and `ignore_merges` vocabulary entries at the edge.
GPU: a body with exactly as many pre-tokens as the work list holds is counted, one more is not; after a batch overflows the
list, no row is counted with entries a previous batch (or a previous vocabulary slot of the same batch) left in it, on
request and SSE response batches, through the zero-copy and the device result block, with one and with two vocabularies;
the N4 pre-charge and N5 metering bill exactly what `tokenizers` counts."""
import copy
import json

import numpy as np
import pytest

from arks_b200 import abi, bpe
from arks_b200.abi import RequestBatch, ResponseBatch
from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token
from test_model_vocab import BUILD, LLAMA, HostSlot, llama3_standin, n_tokens

tokenizers = pytest.importorskip("tokenizers")

UNC = bpe.UNCOUNTED
NOW = 1_700_000_000
MAX_BATCH_BYTES = 1 << 20
FLUSH = 32  # work-list entries one lane hands over per atomic (kBpeFlush)
QWEN = "qwen-7b"


def work_list_cap(max_batch_bytes: int) -> int:
    """entries of the pre-token work list of a context created with `max_batch_bytes` (arks_gateway.cu: arks_create sizes
    max_bytes = align_up(max_batch_bytes + 16, 256); arks_load_bpe_vocab allocates max_bytes / 3 + 1024 entries)"""
    max_bytes = (max_batch_bytes + 16 + 255) // 256 * 256
    return min(max_bytes // 3 + 1024, 0xFFFFFFF0)


CAP = work_list_cap(MAX_BATCH_BYTES)


def splitter(pattern):
    from tokenizers import Regex, pre_tokenizers
    return pre_tokenizers.Split(Regex(pattern), behavior="isolated", invert=False)


def pieces(split, s: str):
    """the pre-tokens of `s`, as `tokenizers` cuts it"""
    return [p for p, _ in split.pre_tokenize_str(s)]


@pytest.fixture(scope="module")
def qwen():
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    return tok, bpe.load_tokenizer(text), splitter(bpe.QWEN2_PATTERN)


@pytest.fixture(scope="module")
def llama():
    """(tokenizer with ignore_merges, tokenizer.json dict, tables, splitter)"""
    tok, _, tj = llama3_standin()
    return tok, tj, bpe.load_tokenizer(tj), splitter(bpe.LLAMA3_PATTERN)


# ---- CPU: piece-length edges -------------------------------------------------------------------------------------------
def edge_texts(L: int):
    """(what, text): texts whose longest pre-token is L bytes under both patterns, one per kind of pattern alternative"""
    return [
        ("letters", "a" * L),
        ("letters ending in a 2-byte letter", "a" * (L - 2) + "é"),
        ("letters ending in a 3-byte letter", "a" * (L - 3) + "你"),
        ("letters ending in a 4-byte letter", "a" * (L - 4) + "\U00020000"),
        ("2-byte letters", "a" * (L % 2) + "é" * (L // 2)),
        ("letters led by a space", " " + "b" * (L - 1)),
        ("letters led by punctuation", "(" + "c" * (L - 1)),
        ("letters led by a 3-byte non-letter", "—" + "d" * (L - 3)),
        ("punctuation and newlines", "!" * (L - 2) + "\n\n"),
        ("space, punctuation, CR LF", " " + "." * (L - 4) + "\r\n\n"),
        ("white space ending in a newline", " " * (L - 1) + "\n"),
        ("white space and tabs ending in newlines", " \t" * ((L - 2) // 2) + " " * (L % 2) + "\n\n"),
        ("white space at the end of the text", "xyz" + " " * L),
        ("white space ending in a 3-byte space", "xyz" + " " * (L - 3) + "　"),
    ]


def edge_bodies(text: str):
    """the text as a counted string next to ordinary ones, with and without \\u escapes"""
    doc = {"model": "m", "messages": [{"role": "user", "content": "hello there"}, {"role": "user", "content": text}],
           "x": {"content": "tail 12345"}}
    return [json.dumps(doc, ensure_ascii=a).encode() for a in (False, True)]


def _edges(host, tok, split):
    for L in (127, 128, 129):
        for what, text in edge_texts(L):
            longest = max(len(p.encode()) for p in pieces(split, text))
            assert longest == L, (what, L, longest)
            for body in edge_bodies(text):
                want = n_tokens(tok, bpe.content_strings(body)) if L <= bpe.MAX_PIECE else UNC
                assert host.count(body) == want, (what, L, body[:80])


def test_piece_length_edges_qwen2(qwen):
    tok, tables, split = qwen
    _edges(HostSlot(tables), tok, split)


def test_piece_length_edges_llama3(llama):
    tok, _, tables, split = llama
    assert tables.flags == bpe.BPE_DIGITS3 | bpe.BPE_IGNORE_MERGES
    _edges(HostSlot(tables), tok, split)


def test_ignore_merges_vocabulary_entries_at_the_edge(llama):
    """vocabulary-only entries (in no merge) of 2, 128 and 129 bytes: a piece equal to one of up to 128 bytes is one token,
    as `tokenizers` counts it; a 129-byte piece is uncounted even though it is a vocabulary entry"""
    from tokenizers import Tokenizer
    _, tj, _, split = llama
    tj = copy.deepcopy(tj)
    vocab = tj["model"]["vocab"]
    two = next(a + b for a in "qjzxkv" for b in "qjzxkv" if a + b not in vocab)
    t128, t129 = "q" * 127 + "z", "q" * 128 + "z"
    near = "q" * 127 + "j"  # 128 bytes, not an entry: counted by merges
    assert not {t128, t129, near} & set(vocab)
    nid = max(vocab.values()) + 1
    for k, s in enumerate((two, t128, t129)):
        vocab[s] = nid + k
    tok = Tokenizer.from_str(json.dumps(tj))
    tables = bpe.load_tokenizer(tj)
    strs = {bytes(tables.tok_bytes[tables.tok_off[k]:tables.tok_off[k + 1]]) for k in range(len(tables.tok_off) - 1)}
    assert two.encode() in strs and t128.encode() in strs and t129.encode() not in strs
    host = HostSlot(tables)
    for s in (two, t128, t129):
        assert pieces(split, s) == [s]
        assert n_tokens(tok, [s]) == 1
    assert n_tokens(tok, [near]) > 1
    mixed = f"{two},\n{t128}!"
    assert pieces(split, mixed) == [two, ",\n", t128, "!"]
    assert n_tokens(tok, [mixed]) == 2 + n_tokens(tok, [",\n", "!"])  # the two entries one token each
    for text, want in ((two, 1), (t128, 1), (near, n_tokens(tok, [near])), (mixed, n_tokens(tok, [mixed])), (t129, UNC),
                       (" " + t128, UNC), (t128 + "\n" + t129, UNC)):
        body = json.dumps({"model": "m", "messages": [{"role": "user", "content": text}]}).encode()
        assert host.count(body) == want, text[:20]
        if want != UNC:
            assert want == n_tokens(tok, bpe.content_strings(body))


# ---- GPU: the work list ------------------------------------------------------------------------------------------------
def digits(n: int) -> str:
    """n one-byte pre-tokens ("1 1 1 ..."), each one token, under both patterns"""
    return ("1 " * ((n + 1) // 2))[:n]


# texts that do not end in a number character (digits() appended after them adds one pre-token per byte)
TEMPLATES = ["Order", " the quick brown fox", "你好, world", "café au lait", "x = [1,2,3];", "Hello\n\nthere —", "éèê 'll"]


def heavy_text(split, n_pieces: int, k: int) -> str:
    """a text of exactly n_pieces pre-tokens: template k, padded with digits()"""
    t = TEMPLATES[k % len(TEMPLATES)]
    s = t + digits(n_pieces - len(pieces(split, t)))
    assert len(pieces(split, s)) == n_pieces, (t, n_pieces)
    return s


def request_body(model: str, text=None, stream=False) -> bytes:
    doc = {"model": model}
    if stream:
        doc["stream"] = True
    doc["messages"] = [] if text is None else [{"role": "user", "content": text}]
    return json.dumps(doc, ensure_ascii=False, separators=(",", ":")).encode()


def sse_chunk(text=None) -> bytes:
    delta = {"role": "assistant"} if text is None else {"content": text}
    return b"data: " + json.dumps({"id": "c", "choices": [{"index": 0, "delta": delta}]}, ensure_ascii=False).encode() + b"\n\n"


def token_tables(models, rules=(("rpm", 10**6), ("tpm", 10**12), ("tpd", 10**12))):
    """one token `tk` with a qos entry per model, all on quota `q`"""
    tok = simple_token("u", "ns", "tk", models[0], list(rules), "q")
    for m in models[1:]:
        q = copy.deepcopy(tok["spec"]["qos"][0])
        q["arksEndpoint"]["name"] = m
        tok["spec"]["qos"].append(q)
    return Tables([tok], [simple_quota("q", "ns", [("prompt", 10**12), ("response", 10**12), ("total", 10**12)])],
                  [simple_endpoint(m, "ns") for m in models])


def requests(bodies, now=NOW):
    return RequestBatch.from_lists(bodies, [b"tk"] * len(bodies), now)


def want_counts(tok, bodies, sse=False, keys=bpe.CONTENT_KEYS):
    """tokenizers' count of every body (tok: one tokenizer, or one per row)"""
    toks = tok if isinstance(tok, list) else [tok] * len(bodies)
    strs = bpe.sse_content_strings if sse else bpe.content_strings
    return np.array([n_tokens(t, strs(b, keys)) for t, b in zip(toks, bodies)], np.int64)


def prime(g, tok, model="m"):
    """the first batch a context sends to the work list: one row of exactly CAP pre-tokens, counted exactly. Every entry of
    the list, [0, CAP), then names row 0; the stale-entry checks below rely on it (a row index from uninitialised memory
    could name any row)"""
    body = request_body(model, digits(CAP))
    a = g.handle_request_body(requests([body]))
    want = want_counts(tok, [body])
    assert want[0] == CAP
    assert int(a.bpe_count[0]) == want[0]
    return body, want


def overflow_bodies(split, n: int, n_pieces: int, make, first):
    """row 0: `first` (no counted string); rows 1..n-1: make(text) of n_pieces pre-tokens each, a multiple of FLUSH, so that
    every flush is FLUSH entries wide and one of them straddles the end of the list; more than CAP pre-tokens in all"""
    assert n_pieces % FLUSH == 0 and (n - 1) * n_pieces > CAP
    return [first] + [make(heavy_text(split, n_pieces, k)) for k in range(n - 1)]


def check_overflowed(dev, want):
    """row 0 reads 0; every other row is uncounted or exactly `want`; some of each"""
    dev = np.asarray(dev)
    assert want[0] == 0
    assert int(dev[0]) == 0, f"row 0 has no counted string but reads {int(dev[0])} (CAP % {FLUSH} = {CAP % FLUSH})"
    rest, w = dev[1:], want[1:]
    unc = rest == UNC
    assert unc.any() and (~unc).any(), int(unc.sum())
    bad = np.flatnonzero(~unc & (rest.astype(np.int64) != w))
    assert len(bad) == 0, [(int(i) + 1, int(rest[i]), int(w[i])) for i in bad[:5]]


def check_exact_after(g, tok, split, model="m", now=NOW):
    """an ordinary batch after the overflow is counted exactly"""
    bodies = [request_body(model)] + [request_body(model, heavy_text(split, 64 + k, k)) for k in range(40)]
    a = g.handle_request_body(requests(bodies, now))
    assert np.array_equal(a.bpe_count.astype(np.int64), want_counts(tok, bodies))


@pytest.mark.gpu
def test_gpu_work_list_capacity_boundary(gwmod, qwen):
    """one row (one lane: deterministic): exactly CAP pre-tokens are counted, CAP + 1 are uncounted"""
    tok, tables, split = qwen
    assert CAP % FLUSH != 0  # the last flush of the exact-capacity row is a partial one
    g = gwmod.Gateway(0, 64, MAX_BATCH_BYTES)
    g.load_tables(token_tables(["m"]))
    g.load_bpe(tables)
    prime(g, tok)
    body = request_body("m", digits(CAP + 1))
    assert len(pieces(split, digits(CAP + 1))) == CAP + 1
    assert int(g.handle_request_body(requests([body])).bpe_count[0]) == UNC
    prime(g, tok)  # and exactly CAP again
    check_exact_after(g, tok, split)


@pytest.mark.gpu
@pytest.mark.parametrize("n,n_pieces", [(2000, 192), (3000, 128)], ids=["zero-copy", "device-block"])
def test_gpu_overflow_counts_no_stale_entries(gwmod, qwen, n, n_pieces):
    """request batches of <= 2048 rows (results written to the pinned block) and of more (the device block)"""
    tok, tables, split = qwen
    g = gwmod.Gateway(0, 4096, MAX_BATCH_BYTES)
    g.load_tables(token_tables(["m"]))
    g.load_bpe(tables)
    prime(g, tok)
    bodies = overflow_bodies(split, n, n_pieces, lambda t: request_body("m", t), request_body("m"))
    a = g.handle_request_body(requests(bodies))
    check_overflowed(a.bpe_count, want_counts(tok, bodies))
    check_exact_after(g, tok, split)


@pytest.mark.gpu
def test_gpu_sse_overflow_after_a_request_batch(gwmod, qwen):
    """the stale entries would cross phases: a request batch fills the list, an SSE response batch overflows it"""
    tok, tables, split = qwen
    g = gwmod.Gateway(0, 4096, MAX_BATCH_BYTES)
    g.load_tables(token_tables(["m"]))
    g.load_bpe(tables)
    prime(g, tok)
    chunks = overflow_bodies(split, 2000, 192, sse_chunk, sse_chunk())
    c = g.handle_response_body(ResponseBatch.from_lists(chunks, [0] * len(chunks), [abi.RESP_STREAM] * len(chunks), NOW))
    check_overflowed(c.bpe_count, want_counts(tok, chunks, sse=True))
    check_exact_after(g, tok, split)


@pytest.mark.gpu
def test_gpu_overflow_with_a_llama3_default_vocabulary(gwmod, llama):
    """slot 0 holds a Llama 3 vocabulary (digits3 + ignore_merges): its own scan and merge instantiations"""
    tok, _, tables, split = llama
    g = gwmod.Gateway(0, 4096, MAX_BATCH_BYTES)
    g.load_tables(token_tables(["m"]))
    g.load_bpe_vocab(0, tables)
    prime(g, tok)
    bodies = overflow_bodies(split, 2000, 192, lambda t: request_body("m", t), request_body("m"))
    a = g.handle_request_body(requests(bodies))
    check_overflowed(a.bpe_count, want_counts(tok, bodies))
    check_exact_after(g, tok, split)


@pytest.mark.gpu
def test_gpu_overflow_with_two_vocabularies(gwmod, qwen, llama):
    """the split path: row 0 is bound to slot 0 and has no content; the heavy rows name llama-3 (slot 1), whose launch
    overflows the list slot 0's launch of the same batch reused"""
    qtok, qtables, qsplit = qwen
    ltok, _, ltables, lsplit = llama
    g = gwmod.Gateway(0, 4096, MAX_BATCH_BYTES)
    g.load_bpe(qtables)
    g.load_bpe_vocab(1, ltables)
    g.bind_model_vocab(LLAMA, 1)
    g.load_tables(token_tables([QWEN, LLAMA]))
    prime(g, qtok, QWEN)
    bodies = overflow_bodies(lsplit, 2000, 192, lambda t: request_body(LLAMA, t), request_body(QWEN))
    a = g.handle_request_body(requests(bodies))
    assert np.all(a.reason == abi.R_OK)
    check_overflowed(a.bpe_count, want_counts([qtok] + [ltok] * (len(bodies) - 1), bodies))
    check_exact_after(g, ltok, lsplit, LLAMA)
    check_exact_after(g, qtok, qsplit, QWEN)


def _same(a, b, what):
    for k, v in a.fields().items():
        assert np.array_equal(v, b.fields()[k]), (what, k)


def referee_counts(dev, want):
    """what the oracle bills with: tokenizers' counts, ARKS_BPE_UNCOUNTED only where the device reported it"""
    return np.where(np.asarray(dev) == UNC, UNC, want).astype(np.uint32)


@pytest.mark.gpu
def test_gpu_overflow_metering_bills_tokenizers_counts(gwmod, qwen):
    """N5: row 0 is an admitted metered stream without content; the heavy rows are metered streams too, counted rows billed
    their count, overflowed ones their body length"""
    from meter_model import MeteredOracle
    tok, tables, split = qwen
    t = token_tables(["m"])
    g = gwmod.Gateway(0, 4096, MAX_BATCH_BYTES)
    g.load_tables(t)
    g.load_bpe(tables)
    g.set_stream_metering(True)
    o = MeteredOracle(t)
    o.set_stream_metering(True)
    body, want = prime(g, tok)  # an ordinary request: not metered
    o.request_batch(requests([body]), counts=want.astype(np.uint32))
    bodies = overflow_bodies(split, 2000, 192, lambda s: request_body("m", s, stream=True), request_body("m", stream=True))
    req = requests(bodies)
    a = g.handle_request_body(req)
    want = want_counts(tok, bodies, keys=bpe.METERED_KEYS)
    _same(a, o.request_batch(req, counts=referee_counts(a.bpe_count, want)), "request")
    assert np.all(a.reason == abi.R_OK) and np.all(a.flags & abi.FLAG_METERED)
    assert np.array_equal(g.snapshot_rate(NOW), o.snapshot_rate(NOW))
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota())
    check_overflowed(a.bpe_count, want)


@pytest.mark.gpu
def test_gpu_overflow_precharge_charges_tokenizers_counts(gwmod, qwen):
    """N4: row 0 is an admitted ordinary request without content; counted rows are pre-charged their count, overflowed
    ones nothing"""
    import orklib
    tok, tables, split = qwen
    t = token_tables(["m"])
    g = gwmod.Gateway(0, 4096, MAX_BATCH_BYTES)
    g.load_tables(t)
    g.load_bpe(tables)
    g.set_precharge(True)
    o = orklib.Oracle(t)
    o.set_precharge(True)
    body, want = prime(g, tok)
    o.set_estimates(want.astype(np.uint32))
    o.request_batch(requests([body]))
    bodies = overflow_bodies(split, 2000, 192, lambda s: request_body("m", s), request_body("m"))
    req = requests(bodies)
    a = g.handle_request_body(req)
    want = want_counts(tok, bodies)
    o.set_estimates(referee_counts(a.bpe_count, want))
    _same(a, o.request_batch(req), "request")
    assert np.all(a.reason == abi.R_OK)
    assert np.array_equal(g.snapshot_rate(NOW), o.snapshot_rate(NOW))
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota())
    check_overflowed(a.bpe_count, want)
