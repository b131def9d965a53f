"""Per-model BPE vocabularies (include/arks_gateway.h: arks_load_bpe_vocab, arks_bind_model_vocab) and the Llama 3 tokenizer
family: numbers split in runs of up to three (`\\p{N}{1,3}`) and `"ignore_merges": true` (a pre-token that is a vocabulary
entry is one token).

CPU: the host build of bpe.cuh with slot flags (tests/bpe_vocab_host.cpp) against HF `tokenizers`, what load_tokenizer
refuses, and the process flags (--bpe.*) as library calls. GPU: two vocabularies in one context, every row counted with its
model's tokenizer on the warp, exact and fast scan paths, bindings landing with the next generation, N4 / N5 billing with
per-model counts, and the single-vocabulary case launching exactly what it did before."""
import copy
import ctypes as C
import json
import os
import random
import subprocess

import numpy as np
import pytest

from arks_b200 import __main__ as main_mod
from arks_b200 import bpe, traffic

tokenizers = pytest.importorskip("tokenizers")

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
UNC = bpe.UNCOUNTED
NOW = 1_700_000_000
LLAMA = "llama-3"


def llama3_standin(n: int = 20_000):
    """a Llama 3 style stand-in (LLAMA3_PATTERN, ignore_merges) with vocabulary-only tokens: for 300 frequent pre-tokens of
    the generated traffic the merge that builds them is removed, so that they stay in the vocabulary but in no merge. Only
    the whole-piece lookup then counts them as one token. -> (tokenizer with ignore_merges, the same without, its
    tokenizer.json dict)"""
    from tokenizers import Regex, Tokenizer, pre_tokenizers
    tok, text = bpe.standin_tokenizer(n, cache_dir=BUILD, pattern=bpe.LLAMA3_PATTERN, ignore_merges=True)
    split = pre_tokenizers.Split(Regex(bpe.LLAMA3_PATTERN), behavior="isolated", invert=False)
    b2u = bpe.bytes_to_unicode()
    rng = np.random.default_rng(11)
    seen = {}
    for _ in range(300):
        for s in bpe.content_strings(traffic.chat_request_body_varied(rng, 900)):
            for piece, _ in split.pre_tokenize_str(s):
                seen[piece] = seen.get(piece, 0) + 1
    tj = json.loads(text)
    pick = {"".join(b2u[b] for b in p.encode()) for p in sorted(seen, key=lambda p: (-seen[p], p)) if 3 <= len(p.encode()) <= 24}
    pick = set(sorted(pick)[:300])
    merges = tj["model"]["merges"]
    pair = lambda m: tuple(m) if isinstance(m, list) else tuple(m.split(" "))  # noqa: E731
    kept = [m for m in merges if "".join(pair(m)) not in pick]
    assert len(merges) - len(kept) >= 100
    tj["model"]["merges"] = kept
    with_im = Tokenizer.from_str(json.dumps(tj))
    tj_off = copy.deepcopy(tj)
    tj_off["model"]["ignore_merges"] = False
    return with_im, Tokenizer.from_str(json.dumps(tj_off)), tj


@pytest.fixture(scope="module")
def llama():
    return llama3_standin()


def _lib():
    """tests/bpe_vocab_host.cpp, compiled like tests/bpe_keys_host.cpp"""
    os.makedirs(BUILD, exist_ok=True)
    src, out = os.path.join(HERE, "bpe_vocab_host.cpp"), os.path.join(BUILD, "libbpe_vocab.so")
    deps = [src] + [os.path.join(ROOT, "arks_b200", "csrc", f) for f in ("bpe.cuh", "json_common.cuh")]
    if not os.path.exists(out) or max(map(os.path.getmtime, deps)) > os.path.getmtime(out):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", out, src])
    L = C.CDLL(out)
    u32p, u8p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)
    L.bv_load.argtypes = [C.c_uint32, u32p, C.c_uint32, u32p, u32p, u32p, u8p, C.c_uint32, u8p, u32p, C.c_uint32]
    L.bv_count.argtypes = [C.c_uint32, C.c_char_p, C.c_size_t]
    L.bv_count.restype = C.c_uint32
    L.bv_pretokenize.argtypes = [C.c_uint32, C.c_char_p, C.c_uint32, u32p, C.c_uint32]
    L.bv_pretokenize.restype = C.c_uint32
    return L


class HostSlot:
    """one vocabulary slot of the host build"""
    _next = 0

    def __init__(self, tables, flags=None):
        self.L = _lib()
        self.slot = HostSlot._next % bpe.MAX_VOCABS
        HostSlot._next += 1
        self.tables = tables
        t = tables.c_struct()
        tb, to = tables.tok_bytes, tables.tok_off
        u8p, u32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)
        self.L.bv_load(self.slot, t.byte_id, t.n_merges, t.left, t.right, t.merged, t.cp_class, tables.flags if flags is None else flags,
                       tb.ctypes.data_as(u8p) if tb is not None else None, to.ctypes.data_as(u32p) if to is not None else None,
                       0 if to is None else len(to) - 1)

    def count(self, body: bytes) -> int:
        return int(self.L.bv_count(self.slot, body, len(body)))

    def pretokenize(self, text: bytes):
        ends = (C.c_uint32 * (len(text) + 1))()
        k = self.L.bv_pretokenize(self.slot, text, len(text), ends, len(text) + 1)
        return list(ends[:k])


def n_tokens(tok, strings) -> int:
    return sum(len(tok.encode(s, add_special_tokens=False).ids) for s in strings)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
def test_llama3_pretokenizer_matches_the_split_pattern(llama):
    """the generator of test_bpe.py::test_pretokenizer_matches_the_split_pattern, against Split(LLAMA3_PATTERN)"""
    from tokenizers import Regex, pre_tokenizers
    host = HostSlot(bpe.load_tokenizer(llama[2]))
    split = pre_tokenizers.Split(Regex(bpe.LLAMA3_PATTERN), behavior="isolated", invert=False)
    r = random.Random(1)
    pool = list("abcXYZ019 \t\n\r'.,!?-_()\"\\/sStTmMdDrReEvVlL") + ["é", "你", "好", "—", "🙂", " ", "　", " ", "́", "ſ", "K", "٣", "²",
                                                                   "½", "ǅ", "ʰ", "ª", "\x0b", "\x0c", "\x85", "​", "﻿", "\x1f", "\x7f"]
    for t in range(60000):
        if t % 3 == 0:
            s = "".join(chr(r.choice([r.randint(1, 0x2FFF), r.randint(0x3000, 0xD7FF), r.randint(0xE000, 0xFFFF),
                                      r.randint(0x10000, 0x2FFFF), r.randint(32, 126)])) for _ in range(r.randint(0, 10)))
        else:
            s = "".join(r.choice(pool) for _ in range(r.randint(0, 14)))
        want = [len(s[:e].encode()) for _, (b, e) in split.pre_tokenize_str(s)]
        assert host.pretokenize(s.encode()) == want, repr(s)
    assert host.pretokenize(b"12345678") == [3, 6, 8]


def test_llama3_counts_match_tokenizers(llama):
    tok, tok_off, tj = llama
    tables = bpe.load_tokenizer(tj)
    assert tables.flags == bpe.BPE_DIGITS3 | bpe.BPE_IGNORE_MERGES
    host = HostSlot(tables)
    merges_only = HostSlot(tables, flags=bpe.BPE_DIGITS3)  # the same vocabulary without the whole-piece lookup
    rng = np.random.default_rng(3)
    differ = 0
    for _ in range(1200):
        b = traffic.chat_request_body_varied(rng, 900, stream=bool(rng.random() < 0.3))
        strs = bpe.content_strings(b)
        assert host.count(b) == n_tokens(tok, strs), b
        assert merges_only.count(b) == n_tokens(tok_off, strs), b
        differ += host.count(b) != merges_only.count(b)
    assert differ > 100  # the injected vocabulary-only tokens are hit
    for _ in range(400):
        b = traffic.chat_response_body_varied(rng, 10, 20, 600)
        assert host.count(b) == n_tokens(tok, bpe.content_strings(b)), b
    r = random.Random(5)
    pool = list("abc XYZ 0123  \t'.,!?-()") + ["é", "你好", "—", "🙂", " the", " and", "ing", "\n", "\n\n", "  ", "'s", "'RE", "\\",
                                                 "\"", "1234567", "٣٤٥٦"]
    for _ in range(3000):
        text = "".join(r.choice(pool) for _ in range(r.randint(0, 60)))
        body = json.dumps({"model": "m", "messages": [{"role": "user", "content": text}, {"content": text[::-1]}]},
                          ensure_ascii=bool(r.random() < 0.5)).encode()
        assert host.count(body) == n_tokens(tok, bpe.content_strings(body)), body
    for ch in traffic.sse_response_chunks(np.random.default_rng(4), 10, 20, 4096):
        assert host.count(ch) == n_tokens(tok, bpe.sse_content_strings(ch))
    assert host.count(b'{"content":"' + b"a" * 200 + b'"}') == UNC


def test_qwen2_slot_is_unchanged():
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    tables = bpe.load_tokenizer(text)
    assert tables.flags == 0 and tables.tok_bytes is None
    host = HostSlot(tables)
    rng = np.random.default_rng(8)
    for _ in range(300):
        b = traffic.chat_request_body_varied(rng, 900)
        assert host.count(b) == n_tokens(tok, bpe.content_strings(b))
    assert host.pretokenize(b"12345678") == list(range(1, 9))


def test_standin_defaults_are_unchanged():
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    assert os.path.exists(os.path.join(BUILD, "standin_bpe_20000_b9e.json"))
    tj = json.loads(text)
    assert tj["pre_tokenizer"]["pretokenizers"][0]["pattern"]["Regex"] == bpe.QWEN2_PATTERN
    assert not tj["model"].get("ignore_merges")


def _tj(text):
    return json.loads(text)


def test_load_tokenizer_refuses_other_families(llama):
    _, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    base = _tj(text)
    bpe.load_tokenizer(base)  # the Qwen2 form itself loads

    def refused(edit, what):
        tj = copy.deepcopy(base)
        edit(tj)
        with pytest.raises(ValueError, match=what):
            bpe.load_tokenizer(tj)
    gpt2 = {"type": "ByteLevel", "add_prefix_space": False, "trim_offsets": True, "use_regex": True}
    refused(lambda tj: tj.__setitem__("pre_tokenizer", gpt2), "pre-tokenizer")
    refused(lambda tj: tj["pre_tokenizer"]["pretokenizers"][1].__setitem__("use_regex", True), "use_regex")
    refused(lambda tj: tj["pre_tokenizer"]["pretokenizers"][0]["pattern"].__setitem__("Regex", r"\p{N}+|[^\p{N}]+"), "split pattern")
    refused(lambda tj: tj["model"].__setitem__("byte_fallback", True), "byte_fallback")
    refused(lambda tj: tj.__setitem__("normalizer", {"type": "Lowercase"}), "normalizer")
    refused(lambda tj: tj["model"].__setitem__("type", "WordPiece"), "model type")
    refused(lambda tj: tj["model"].__setitem__("end_of_word_suffix", "</w>"), "end_of_word_suffix")
    nfc = copy.deepcopy(base)
    nfc["normalizer"] = {"type": "NFC"}
    assert bpe.load_tokenizer(nfc).flags == bpe.BPE_NFC
    # the Llama 3 form: flags and the token strings of 2..128 bytes, the injected ones among them
    t = bpe.load_tokenizer(llama[2])
    strs = {bytes(t.tok_bytes[t.tok_off[k]:t.tok_off[k + 1]]) for k in range(len(t.tok_off) - 1)}
    assert all(2 <= len(s) <= bpe.MAX_PIECE for s in strs)
    assert len(strs) > 15_000


class FakeEngine:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *a: self.calls.append((name,) + a)


def test_process_flags_become_library_calls():
    loaded = {"q.json": bpe.BpeTables(*([None] * 5), 0), "l.json": bpe.BpeTables(*([None] * 5), bpe.BPE_IGNORE_MERGES | bpe.BPE_DIGITS3)}
    load = loaded.__getitem__
    e = FakeEngine()
    main_mod.configure_bpe(e, main_mod.parse_args([]), load=load)
    assert e.calls == []
    args = main_mod.parse_args(["--bpe.tokenizer", "q.json", "--bpe.model-tokenizer", "llama-3=l.json", "--bpe.model-tokenizer",
                                "llama-3-70b=./l.json", "--bpe.model-tokenizer", f"qwen-7b={os.path.abspath('q.json')}", "--bpe.precharge",
                                "--bpe.stream-metering"])
    main_mod.configure_bpe(e, args, load=load)
    assert e.calls == [("load_bpe", loaded["q.json"]), ("load_bpe_vocab", 1, loaded["l.json"]), ("bind_model_vocab", "llama-3", 1),
                       ("bind_model_vocab", "llama-3-70b", 1), ("set_precharge", True), ("set_stream_metering", True)]
    # an ignore_merges default vocabulary needs its token strings: the slot form
    e = FakeEngine()
    main_mod.configure_bpe(e, main_mod.parse_args(["--bpe.tokenizer", "l.json"]), load=load)
    assert e.calls == [("load_bpe_vocab", 0, loaded["l.json"])]
    for bad in (["--bpe.precharge"], ["--bpe.model-tokenizer", "m=l.json"], ["--bpe.tokenizer", "q.json", "--bpe.model-tokenizer", "m"]):
        with pytest.raises(ValueError):
            main_mod.configure_bpe(FakeEngine(), main_mod.parse_args(bad), load=load)


def test_process_flags_share_a_slot_per_file(tmp_path):
    """the same file under another spelling (a symlink) takes no slot of its own"""
    real = tmp_path / "llama.json"
    real.write_text("{}")
    (tmp_path / "alias.json").symlink_to(real)
    flagged = bpe.BpeTables(*([None] * 5), bpe.BPE_DIGITS3)
    e = FakeEngine()
    args = main_mod.parse_args(["--bpe.tokenizer", "q.json", "--bpe.model-tokenizer", f"a={real}", "--bpe.model-tokenizer",
                                f"b={tmp_path / 'alias.json'}"])
    main_mod.configure_bpe(e, args, load=lambda p: flagged)
    assert e.calls == [("load_bpe", flagged), ("load_bpe_vocab", 1, flagged), ("bind_model_vocab", "a", 1), ("bind_model_vocab", "b", 1)]


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def two_model_objects(n_tenants=300, seed=23):
    """traffic.Workload's config with a second model: every token has a qos entry for qwen-7b and one for llama-3, each
    namespace an endpoint for both"""
    w = traffic.Workload(n_tenants=n_tenants, seed=seed)
    tokens, quotas, endpoints = copy.deepcopy(w.objects)
    for t in tokens:
        q = copy.deepcopy(t["spec"]["qos"][0])
        q["arksEndpoint"]["name"] = LLAMA
        t["spec"]["qos"].append(q)
    endpoints += [dict(copy.deepcopy(e), metadata=dict(e["metadata"], name=LLAMA)) for e in endpoints]
    return w, (tokens, quotas, endpoints)


def two_model_batch(w, n, now, seed, meter_half=False):
    """w's traffic with about half of the bodies naming llama-3; noise rows (unknown token, other model, no model, ...)
    resolve no qos entry. meter_half: half of the include_usage streams drop the option (metered under N5)"""
    from arks_b200.abi import RequestBatch
    req = w.request_batch(n, now, seed=seed, stream_frac=0.6 if meter_half else 0.2, varied=True, noise_frac=0.04)
    rng = np.random.default_rng(seed)
    bodies, toks = [], []
    for i in range(req.n):
        b = bytes(req.bodies[req.body_off[i]:req.body_off[i] + req.body_len[i]])
        if rng.random() < 0.5:
            b = b.replace(b'"model":"qwen-7b"', b'"model":"llama-3"')
        if rng.random() < 0.5:  # numbers: the two pre-tokenizers split them differently
            b = b.replace(b'"content":"', b'"content":"order %d of %d: ' % (rng.integers(10**9), rng.integers(10**5)), 1)
        if meter_half and rng.random() < 0.5:
            b = b.replace(b',"stream_options":{"include_usage":true}', b"")
        bodies.append(b)
        toks.append(bytes(req.tokens[req.token_off[i]:req.token_off[i + 1]]))
    return RequestBatch.from_lists(bodies, toks, now, pick_rand=req.pick_rand), bodies


def expected(toks, slots, docs, sse, wide=None):
    """tokenizers' count of every doc with the tokenizer of its slot (wide: the metered key set); -1 for a body that is not
    JSON (the noise rows: there is nothing to compare)"""
    out = []
    for i, d in enumerate(docs):
        keys = bpe.METERED_KEYS if wide is not None and wide[i] else bpe.CONTENT_KEYS
        try:
            strs = bpe.sse_content_strings(d, keys) if sse[i] else bpe.content_strings(d, keys)
        except ValueError:
            out.append(-1)
            continue
        out.append(n_tokens(toks[slots[i]], strs))
    return np.array(out, np.int64)


def check(dev, want, min_counted=0.95, why=None):
    """the device's counts equal `want` wherever both exist; nearly every row has both. why(i): what to report of row i"""
    both = (dev != UNC) & (want >= 0)
    assert both.mean() > min_counted
    bad = np.flatnonzero(both & (dev.astype(np.int64) != want))
    assert len(bad) == 0, (len(bad), [(int(i), int(dev[i]), int(want[i]), why(i) if why else None) for i in bad[:4]])
    return both


def fill(dev, want):
    """`want` with the device's value where there is nothing to compare (the counts the oracle is handed)"""
    return np.where((dev == UNC) | (want < 0), dev.astype(np.int64), want).astype(np.uint32)


def row_slots(qos, models):
    """the slot a row is counted with: 1 when its qos entry is llama-3's (bound to slot 1), else 0. The entry, not the body:
    a body may name a model twice (the noise rows add a "MODEL" key, which Go's case-insensitive decoding takes)"""
    return [1 if q >= 0 and models[q] == LLAMA else 0 for q in qos]


def resp_docs(resp):
    return [bytes(resp.bodies[resp.body_off[k]:resp.body_off[k] + resp.body_len[k]]) for k in range(resp.n)]


@pytest.fixture(scope="module")
def vocabs(llama):
    qtok, qtext = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    return (qtok, llama[0], llama[1]), (bpe.load_tokenizer(qtext), bpe.load_tokenizer(llama[2]))


def _same(a, b, what):
    for k, v in a.fields().items():
        assert np.array_equal(v, b.fields()[k]), (what, k)


@pytest.mark.gpu
def test_gpu_counts_each_row_with_its_models_vocabulary(gwmod, vocabs):
    import orklib
    from arks_b200 import abi
    from arks_b200.tables import Tables
    toks, tabs = vocabs
    w, objs = two_model_objects()
    tables = Tables(*objs)
    g = gwmod.Gateway(0, 32768, 64 << 20)
    with pytest.raises(Exception):
        g.load_bpe_vocab(1, tabs[1])  # slot 0 first
    g.load_bpe(tabs[0])
    with pytest.raises(Exception):
        g.load_bpe(tabs[1])  # ignore_merges needs the token strings: the slot form
    with pytest.raises(Exception):
        g.bind_model_vocab(LLAMA, 1)  # slot 1 is empty
    g.load_bpe_vocab(1, tabs[1])
    g.bind_model_vocab(LLAMA, 1)
    g.load_tables(tables)
    with pytest.raises(Exception):
        g.load_bpe_vocab(1, None)  # bound
    with pytest.raises(Exception):
        g.load_bpe(None)  # another slot is loaded
    o = orklib.Oracle(tables)
    models = qos_models(tables)
    gen0 = g.generation
    for step, n in enumerate((700, 3000, 9000)):  # warp path, exact engine, fast path
        now = NOW + step * 3600
        req, bodies = two_model_batch(w, n, now, 40 + step)
        a = g.handle_request_body(req)
        _same(a, o.request_batch(req), ("request", step))
        slots = row_slots(a.qos, models)
        assert 0.3 * n < sum(slots) < 0.6 * n and np.sum(a.qos < 0) > 0.01 * n
        want = expected(toks, slots, bodies, [False] * n)
        ok = check(a.bpe_count, want, why=lambda i: (slots[i], int(a.qos[i]), int(a.reason[i]), bodies[i][:160]))
        # the other vocabulary's count, and for llama-3 rows the count without the whole-piece lookup, would differ on
        # many rows: each row really uses its own vocabulary and flags
        other = expected(toks, [1 - s for s in slots], bodies, [False] * n)
        assert np.sum((other != want) & ok) > 0.1 * n
        merges_only = expected(toks, [2 * s for s in slots], bodies, [False] * n)
        assert np.sum((merges_only != want) & ok) > 0.1 * n
        resp = w.response_batch(a, now, seed=70 + step, varied=True)
        c = g.handle_response_body(resp)
        _same(c, o.response_batch(resp), ("response", step))
        docs = resp_docs(resp)
        rslots = row_slots(resp.qos, models)
        assert sum(rslots) > 0.3 * resp.n
        check(c.bpe_count, expected(toks, rslots, docs, [bool(f & abi.RESP_STREAM) for f in resp.flags]))
    # response rows of an older generation: counted with the binding of the current one
    req, bodies = two_model_batch(w, 2000, NOW + 86_400, 99)
    a = g.handle_request_body(req)
    resp = w.response_batch(a, NOW + 86_400, seed=98)
    resp.gen = np.full(resp.n, g.generation, np.uint32)
    g.bind_model_vocab(LLAMA, 0)
    g.load_tables(tables)  # the binding is gone from this generation on
    assert g.generation == gen0 + 1
    c = g.handle_response_body(resp)
    docs = resp_docs(resp)
    sse = [bool(f & abi.RESP_STREAM) for f in resp.flags]
    check(c.bpe_count, expected(toks, [0] * resp.n, docs, sse))
    g.load_bpe_vocab(1, None)  # no longer bound anywhere: may be emptied
    g.load_bpe(None)


def qos_models(tables):
    """model name of every qos entry, in table order"""
    return [bytes(tables.str_bytes[tables.str_off[m]:tables.str_off[m + 1]]).decode() for m in tables.qos_model_str]


@pytest.mark.gpu
def test_gpu_binding_lands_with_the_next_generation_of_the_store(gwmod, vocabs):
    """the object store: arks_bind_model_vocab, then arks_config_prepare + commit publishes it"""
    from arks_b200 import abi
    from arks_b200.abi import RequestBatch
    toks, tabs = vocabs
    g = gwmod.Gateway(0, 1024, 4 << 20)
    g.load_bpe(tabs[0])
    g.load_bpe_vocab(1, tabs[1])
    g.upsert_quota("ns", "q", [(abi.QUOTA_TYPES[k], 10**9) for k in ("prompt", "response", "total")])
    g.upsert_token("ns", "u", "sk-1", [(m, "q", [(abi.RULES["rpm"], 10**6)]) for m in ("qwen-7b", LLAMA)])
    for m in ("qwen-7b", LLAMA):
        g.upsert_endpoint("ns", m, [1])
    g.commit_tables(g.config_prepare())
    text = "Call 12345678 and 2024 apples; " + " ".join(["interoperability", "transformation", "hello world"] * 3)
    bodies = [json.dumps({"model": m, "messages": [{"role": "user", "content": text}]}).encode() for m in ("qwen-7b", LLAMA)]

    def counts(now):
        a = g.handle_request_body(RequestBatch.from_lists(bodies, [b"sk-1"] * 2, now))
        assert a.reason.tolist() == [0, 0]
        return a.bpe_count.tolist()
    q = [n_tokens(toks[0], [text])] * 2
    l = [q[0], n_tokens(toks[1], [text])]
    assert q != l
    assert counts(NOW) == q
    g.bind_model_vocab(LLAMA, 1)
    assert counts(NOW + 1) == q  # not before the next generation
    p = g.config_prepare()
    assert counts(NOW + 2) == q  # prepared, not committed
    g.commit_tables(p)
    assert counts(NOW + 3) == l
    g.bind_model_vocab(LLAMA, 0)
    assert counts(NOW + 4) == l
    g.commit_tables(g.config_prepare())
    assert counts(NOW + 5) == q


@pytest.mark.gpu
def test_gpu_precharge_and_metering_bill_per_model_counts(gwmod, vocabs):
    """N4 + N5 with two vocabularies: every counter equals the metering oracle fed with each row's model's count"""
    from arks_b200 import abi
    from arks_b200.abi import ResponseBatch
    from arks_b200.tables import Tables
    from meter_model import METERED_CHUNK, MeteredOracle, is_metered_request
    toks, tabs = vocabs
    w, objs = two_model_objects(200, seed=31)
    tables = Tables(*objs)
    models = qos_models(tables)
    g = gwmod.Gateway(0, 32768, 64 << 20)
    g.enable_metrics(True)
    g.load_bpe(tabs[0])
    g.load_bpe_vocab(1, tabs[1])
    g.bind_model_vocab(LLAMA, 1)
    g.load_tables(tables)
    g.set_precharge(True)
    g.set_stream_metering(True)
    o = MeteredOracle(tables)
    o.set_precharge(True)
    o.set_stream_metering(True)
    for step, n in enumerate((700, 3000, 9000)):  # warp path, exact engine, fast path
        now = NOW + step
        req, bodies = two_model_batch(w, n, now, 50 + step, meter_half=True)
        a = g.handle_request_body(req)
        wide = [is_metered_request(b) for b in bodies]
        want = expected(toks, row_slots(a.qos, models), bodies, [False] * n, wide)
        check(a.bpe_count, want)
        est = fill(a.bpe_count, want)
        _same(a, o.request_batch(req, counts=est), ("request", step))
        metered = (a.flags & abi.FLAG_METERED) != 0
        assert metered.sum() > 0.1 * n
        for snap in ("snapshot_quota", "snapshot_metrics"):
            assert np.array_equal(getattr(g, snap)(), getattr(o, snap)()), (step, snap)
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), step
        resp = w.response_batch(a, now, seed=80 + step, varied=True)
        owner = np.repeat(np.flatnonzero(a.reason == abi.R_OK), np.where(a.flags[a.reason == abi.R_OK] & 1, 4, 1))
        assert len(owner) == resp.n
        flags = [int(f) | (abi.RESP_METERED if metered[owner[k]] else 0) for k, f in enumerate(resp.flags)]
        pre = np.array([0 if metered[owner[k]] else a.bpe_count[owner[k]] for k in range(resp.n)], np.uint32)
        pre = np.where(pre == UNC, 0, pre).astype(np.uint32)
        docs = resp_docs(resp)
        resp = ResponseBatch.from_lists(docs, resp.qos.tolist(), flags, now)
        resp.precharged = pre
        c = g.handle_response_body(resp)
        m = [(f & METERED_CHUNK) == METERED_CHUNK for f in flags]
        rslots = row_slots(resp.qos, models)
        want = expected(toks, rslots, docs, [bool(f & abi.RESP_STREAM) for f in flags], m)
        check(c.bpe_count, want)
        cnt = fill(c.bpe_count, want)
        _same(c, o.response_batch(resp, counts=cnt), ("response", step))
        for snap in ("snapshot_quota", "snapshot_metrics"):
            assert np.array_equal(getattr(g, snap)(), getattr(o, snap)()), (step, snap)
        assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), step


@pytest.mark.gpu
def test_gpu_single_vocabulary_launches_and_counts_as_before(gwmod, vocabs):
    """slot 0 only and no binding: the same counts and the same kernel launches per batch as a context that never called
    the new functions; a loaded but unbound slot 1 changes neither"""
    _, tabs = vocabs
    w, objs = two_model_objects(100, seed=5)
    from arks_b200.tables import Tables
    tables = Tables(*objs)

    def run(g):
        out = []
        for step, n in enumerate((700, 3000, 9000)):
            req, _ = two_model_batch(w, n, NOW + step, 60 + step)
            before = g.launch_count
            a = g.handle_request_body(req)
            mid = g.launch_count
            c = g.handle_response_body(w.response_batch(a, NOW + step, seed=61 + step, varied=True))
            out.append((mid - before, g.launch_count - mid, a.bpe_count.copy(), c.bpe_count.copy()))
        return out
    plain = gwmod.Gateway(0, 16384, 64 << 20)
    plain.load_tables(tables)
    plain.load_bpe(tabs[0])
    new = gwmod.Gateway(0, 16384, 64 << 20)
    new.load_bpe_vocab(0, tabs[0])
    new.bind_model_vocab(LLAMA, 0)
    new.load_tables(tables)
    extra = gwmod.Gateway(0, 16384, 64 << 20)
    extra.load_bpe(tabs[0])
    extra.load_bpe_vocab(1, tabs[1])
    extra.load_tables(tables)
    want = run(plain)
    for g in (new, extra):
        for x, y in zip(run(g), want):
            assert x[0] == y[0] and x[1] == y[1]
            assert np.array_equal(x[2], y[2]) and np.array_equal(x[3], y[3])


@pytest.mark.gpu
def test_gpu_flagged_default_vocabulary_without_bindings(gwmod, vocabs):
    """a Llama 3 vocabulary as the default (slot 0) with nothing bound: the two kernels run with its own pre-tokenizer and
    whole-piece lookup, on the warp, exact and fast paths. The same vocabulary without ignore_merges through arks_load_bpe
    (ARKS_BPE_DIGITS3 only) is counted like `tokenizers` without it. Each launches what a Qwen2 context launches"""
    from arks_b200.tables import Tables
    toks, tabs = vocabs
    w, objs = two_model_objects(100, seed=7)
    tables = Tables(*objs)
    digits_only = copy.copy(tabs[1])
    digits_only.flags = bpe.BPE_DIGITS3
    ctxs = []
    for load, tok in ((lambda g: g.load_bpe_vocab(0, tabs[1]), toks[1]), (lambda g: g.load_bpe(digits_only), toks[2]),
                      (lambda g: g.load_bpe(tabs[0]), toks[0])):
        g = gwmod.Gateway(0, 16384, 64 << 20)
        g.load_tables(tables)
        load(g)
        ctxs.append((g, tok))
    for step, n in enumerate((700, 3000, 9000)):
        req, bodies = two_model_batch(w, n, NOW + step, 90 + step)
        qwen = expected({0: toks[0]}, [0] * n, bodies, [False] * n)
        launched = []
        for k, (g, tok) in enumerate(ctxs):
            before = g.launch_count
            a = g.handle_request_body(req)
            launched.append(g.launch_count - before)
            want = expected({0: tok}, [0] * n, bodies, [False] * n)
            ok = check(a.bpe_count, want)
            if k < 2:  # Qwen2's count differs on many rows: the flags are honoured
                assert np.sum((qwen != want) & ok) > 0.1 * n
        assert launched[0] == launched[1] == launched[2], launched
