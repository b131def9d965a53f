"""The JSON filters, the exact engine and the SSE line layer at the exact edge of every fixed capacity they have.

Seeded random traffic almost never lands ON a capacity, so each limit gets a pair of documents here: the largest one that
must be ACCEPTED (and then give what the exact engine and the oracle give) and the smallest one that must be DECLINED (filters)
or is an error (engine, SSE). Moving a constant by one, or an off-by-one in its comparison, fails a test. The member that
is read (`model`, `include_usage`, `total_tokens`, the usage event) always comes AFTER the stretch that exhausts the
capacity, so a walk that stops early gives a visibly wrong answer rather than the default one.

No expected value comes from a device: verdicts and fields are the oracle's (orklib), `json.loads` is a second referee
for valid documents, and where the reference's rule is known it is written down as a known answer:
  * bufio.MaxScanTokenSize = 64 * 1024 (bufio/scan.go): a line of 65 535 bytes before its '\\n' is a token, a line of
    65 536 bytes is ErrTooLong, terminated or not, CR counted;
  * json-iterator's maxDepth = 10000 (iter.go, incrementDepth: `depth <= maxDepth`) and encoding/json's maxNestingDepth
    = 10000 (scanner.go: `depth > maxNestingDepth`): 10 000 open containers parse, the 10 001st is an error.

CPU part: the host builds of the same headers (tests/hostmachine.py). GPU part (`-m gpu`): the same documents through
every scan path of the device, the path proven with Gateway.last_declined."""
import json

import numpy as np
import pytest

import hostmachine as hm
import orklib
import pymodel

# ---- the constants under test, as this file believes them (a change in the headers must be repeated here on purpose) ----
FAST_MAX_LEN = 2048        # mask_scan.cuh / warp_scan.cuh kFastMaxLen
FAST_MAX_MEMBERS = 8       # mask_scan.cuh kFastMaxMembers
MINI_CAP = {"mask": 192, "warp": 160}  # kFastMiniCap of mask_scan.cuh / warp_scan.cuh
FAST_MAX_TOK = 512         # warp_scan.cuh kFastMaxTok
FAST_MAX_DEPTH = 32        # warp_scan.cuh kFastMaxDepth; mask_scan.cuh: `depth >= 32`
MAX_DEPTH = 10000          # json_common.cuh kMaxDepth
SSE_LINE_MAX = 65536       # json_engine.cuh SseT::step, SseSplit::end_line, SseSplit::finish; oracle/ork_json.c

FILTERS = {"mask": (hm.fast_request, hm.fast_response), "warp": (hm.warp_request, hm.warp_response)}


def structure_tokens(doc: bytes, both_quotes: bool):
    """positions of the bytes outside strings plus the opening quote of every string (what mask_scan.cuh walks and what
    one iteration of warp_scan.cuh's mini walk consumes); with both_quotes also the closing quotes (warp_scan.cuh's token
    list). Written from the definition, not from either header."""
    out, in_str, i = [], False, 0
    while i < len(doc):
        c = doc[i]
        if in_str:
            if c == 0x5c:
                i += 2
                continue
            if c == 0x22:
                in_str = False
                if both_quotes:
                    out.append(i)
        else:
            out.append(i)
            if c == 0x22:
                in_str = True
        i += 1
    return out


def inner_tokens(doc: bytes, key: bytes) -> int:
    """tokens of the object that is the value of `key`, from behind its '{' up to and including its '}'"""
    open_ = doc.index(b'"' + key + b'":{') + len(key) + 3
    depth, n = 1, 0
    for p in structure_tokens(doc, False):
        if p <= open_:
            continue
        n += 1
        if doc[p] in b"{[":
            depth += 1
        elif doc[p] in b"}]":
            depth -= 1
            if depth == 0:
                return n
    raise AssertionError("unterminated")


def accepted_request(which, b, model=b"m", st=0, so=0, iu=0):
    """the filter takes the document and says what the engine, the oracle, json.loads and the known answer say"""
    f = FILTERS[which][0](b)
    assert f is not None, (which, "declined a document it must accept", b[:80], len(b))
    e = hm.engine_request(b)
    assert f == e, (which, b[:80], f, e)
    rc, m, *flags = orklib.parse_request_body(b)
    assert rc == 0 and tuple(flags) == f[1:] == (st, so, iu), (which, b[:80], f, flags)
    assert m == b[f[0][0]:f[0][0] + f[0][1]] == model, (which, b[:80], f, m)
    p = pymodel.request_fields(b)
    assert p is not None and (p["err"], p["model"], p["stream"], p["so_present"], p["include_usage"]) == (0, model, st, so, iu), (b[:80], p)


def accepted_response(which, b, usage):
    f = FILTERS[which][1](b)
    assert f is not None, (which, "declined a document it must accept", b[:80], len(b))
    e = hm.engine_response(b)
    assert f == e, (which, b[:80], f, e)
    rc, ml, u = orklib.parse_response_body(b)
    assert rc == 0 and tuple(u) == f[1] == tuple(usage), (which, b[:80], f, u)
    d = json.loads(b)
    assert tuple(d["usage"].get(k, 0) for k in ("prompt_tokens", "completion_tokens", "total_tokens")) == tuple(usage)


def declined_request(which, b, valid=True):
    """the filter leaves the document to the exact engine; `valid`: engine and oracle then parse it (the filter declined
    for capacity, not because the document is wrong)"""
    assert FILTERS[which][0](b) is None, (which, "accepted a document beyond its capacity", b[:80], len(b))
    rc = orklib.parse_request_body(b)[0]
    assert rc == (0 if valid else 1) and (hm.engine_request(b) is not None) == valid, (b[:80], rc)
    assert hm.parse_request_body(b) == orklib.parse_request_body(b) or not valid


def declined_response(which, b, valid=True):
    assert FILTERS[which][1](b) is None, (which, "accepted a document beyond its capacity", b[:80], len(b))
    rc = orklib.parse_response_body(b)[0]
    assert rc == (0 if valid else 1) and (hm.engine_response(b) is not None) == valid, (b[:80], rc)


# ------------------------------------------------------------------------------------------------------------------
# document builders (shared by the CPU and the GPU part)
# ------------------------------------------------------------------------------------------------------------------
def padded_request(total_len: int) -> bytes:
    head, tail = b'{"p":"', b'","model":"m","stream":true}'
    return head + b"x" * (total_len - len(head) - len(tail)) + tail


def padded_response(total_len: int) -> bytes:
    head, tail = b'{"p":"', b'","model":"m","usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'
    return head + b"x" * (total_len - len(head) - len(tail)) + tail


def members_request(n_other: int, klen: int, real_at: str) -> bytes:
    """`n_other` members whose keys are `klen` bytes long (logged when klen is 5, 6 or 14) around the real model / stream"""
    other = ['"%s":%d' % (("k%0" + str(klen - 1) + "d") % i, i) for i in range(n_other)]
    real = ['"model":"m"', '"stream":true']
    at = {"first": 0, "middle": n_other // 2, "last": n_other}[real_at]
    return ("{" + ",".join(other[:at] + real + other[at:]) + "}").encode()


def members_request_mixed(n_logged: int) -> bytes:
    """keys of lengths 5, 6 and 14 in turn, `n_logged` logged members in all, the three real names last"""
    lens = [5, 6, 14]
    other = ['"%s":null' % ("q" * lens[i % 3]) for i in range(n_logged - 3)]
    # (equal keys among the fillers are fine: only the names that are read must not repeat)
    return ("{" + ",".join(other + ['"stream_options":{"include_usage":true}', '"stream":false', '"model":"m"']) + "}").encode()


def members_response(n_other: int, real_at: str) -> bytes:
    other = ['"k%04d":%d' % (i, i) for i in range(n_other)]
    real = ['"model":"m"', '"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}']
    at = {"first": 0, "middle": n_other // 2, "last": n_other}[real_at]
    return ("{" + ",".join(other[:at] + real + other[at:]) + "}").encode()


def mini_request(n_tok: int) -> bytes:
    """stream_options whose object has exactly n_tok tokens behind its '{', its '}' the last, include_usage the last member"""
    for zeros in range(1, 200):
        for blanks in range(2):
            b = ('{"stream_options":{"x":[' + ",".join("0" * zeros) + "]" + " " * blanks + ',"include_usage":true},"model":"m"}').encode()
            if inner_tokens(b, b"stream_options") == n_tok:
                return b
    raise AssertionError(n_tok)


def mini_response(n_tok: int) -> bytes:
    for zeros in range(1, 200):
        for blanks in range(2):
            b = ('{"usage":{"x":[' + ",".join("0" * zeros) + "]" + " " * blanks + ',"total_tokens":357},"model":"m"}').encode()
            if inner_tokens(b, b"usage") == n_tok:
                return b
    raise AssertionError(n_tok)


def tok_request(n_tok: int, pad: int) -> bytes:
    """exactly n_tok bytes outside strings and quotes in the whole document; `pad` bytes of string in front move the
    structure across warp_scan.cuh's 1 KiB segments"""
    for zeros in range(1, 600):
        for blanks in range(2):
            b = ('{"p":"' + "x" * pad + '","a":[' + ",".join("0" * zeros) + "]" + " " * blanks + ',"model":"m"}').encode()
            n = len(structure_tokens(b, True))
            if n == n_tok:
                return b
            if n > n_tok:
                break
    raise AssertionError(n_tok)


def tok_response(n_tok: int, pad: int) -> bytes:
    for zeros in range(1, 600):
        for blanks in range(2):
            b = ('{"p":"' + "x" * pad + '","a":[' + ",".join("0" * zeros) + "]" + " " * blanks +
                 ',"model":"m","usage":{"total_tokens":357}}').encode()
            n = len(structure_tokens(b, True))
            if n == n_tok:
                return b
            if n > n_tok:
                break
    raise AssertionError(n_tok)


def nest(levels: int, kind: str, spoil: bool = False) -> bytes:
    """`levels` containers inside each other: kind "arr", "obj" (keys are the empty string: 4 bytes a level) or "alt";
    spoil: the innermost one is closed with the other kind's bracket"""
    opens, closes = [], []
    for i in range(levels):
        obj = kind == "obj" or (kind == "alt" and i % 2 == 1)
        opens.append(b'{"":' if obj and i < levels - 1 else b"{" if obj else b"[")
        closes.append(b"}" if obj else b"]")
    if spoil:
        closes[-1] = b"]" if closes[-1] == b"}" else b"}"
    return b"".join(opens) + b"".join(reversed(closes))


def deep_request(depth: int, kind: str, spoil: bool = False) -> bytes:
    """total nesting `depth`, the top-level object included"""
    return b'{"d":' + nest(depth - 1, kind, spoil) + b',"model":"m","stream":true}'


def deep_response(depth: int, kind: str, spoil: bool = False) -> bytes:
    return b'{"choices":' + nest(depth - 1, kind, spoil) + b',"model":"m","usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'


def deep_event(depth: int, kind: str) -> bytes:
    return b'{"choices":[],"d":' + nest(depth - 1, kind) + b',"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'


USAGE_EV = b'data: {"id":"c","choices":[],"usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}\n\n'
DELTA_EV = b'data: {"id":"c","choices":[{"index":0,"delta":{"content":"hi"}}],"usage":null}\n\n'


def long_line(total: int, kind: str) -> bytes:
    """one line of exactly `total` bytes (no line end): a data line whose payload is one long string ("string": the
    in-string skip of SseT), many short tokens ("tokens": the byte-by-byte step) or a comment line"""
    if kind == "comment":
        return b":" + b"c" * (total - 1)
    if kind == "string":
        head, tail = b'data: {"choices":[{"delta":{"content":"', b'"}}]}'
        return head + b"x" * (total - len(head) - len(tail)) + tail
    head, tail = b'data: {"choices":[{"d":[', b"0]}]}"
    fill = total - len(head) - len(tail)
    return head + b"0," * (fill // 2) + b" " * (fill % 2) + tail


# ------------------------------------------------------------------------------------------------------------------
# CPU part: the filters
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["mask", "warp"])
def test_kFastMaxLen_2048_bytes(which):
    """kFastMaxLen: a document of 2 048 bytes is the longest either filter takes, one of 2 049 bytes goes to the exact engine."""
    for n in (FAST_MAX_LEN - 1, FAST_MAX_LEN):
        assert len(padded_request(n)) == n
        accepted_request(which, padded_request(n), st=2)
        accepted_response(which, padded_response(n), (3, 4, 7))
    declined_request(which, padded_request(FAST_MAX_LEN + 1))
    declined_response(which, padded_response(FAST_MAX_LEN + 1))


@pytest.mark.parametrize("real_at", ["first", "middle", "last"])
@pytest.mark.parametrize("klen", [5, 6, 14])
def test_kFastMaxMembers_8_logged_request_members(klen, real_at):
    """kFastMaxMembers: mask_scan.cuh logs the top-level members whose key is 5, 6 or 14 bytes long; 8 of them (the real
    `model` and `stream` included) are accepted, the 9th sends the document to the exact engine. Keys of another length
    are not logged and do not count; warp_scan.cuh has no member log and takes all of them."""
    n_real = 2
    accepted_request("mask", members_request(FAST_MAX_MEMBERS - n_real - 1, klen, real_at), st=2)
    accepted_request("mask", members_request(FAST_MAX_MEMBERS - n_real, klen, real_at), st=2)
    declined_request("mask", members_request(FAST_MAX_MEMBERS - n_real + 1, klen, real_at))
    accepted_request("warp", members_request(FAST_MAX_MEMBERS - n_real + 1, klen, real_at), st=2)
    accepted_request("mask", members_request(40, klen + 1 if klen != 5 else 7, real_at), st=2)


def test_kFastMaxMembers_mixed_key_lengths():
    """kFastMaxMembers counts the logged lengths together: 5-, 6- and 14-byte keys summing to 8 / 9, the names that are
    read last."""
    accepted_request("mask", members_request_mixed(FAST_MAX_MEMBERS), st=1, so=1, iu=2)
    declined_request("mask", members_request_mixed(FAST_MAX_MEMBERS + 1))
    accepted_request("warp", members_request_mixed(FAST_MAX_MEMBERS + 1), st=1, so=1, iu=2)


@pytest.mark.parametrize("real_at", ["first", "middle", "last"])
def test_kFastMaxMembers_8_logged_response_members(real_at):
    """kFastMaxMembers with kFastKeyLensResp: on the response side only 5-byte keys are logged (`model`, `usage`)."""
    accepted_response("mask", members_response(FAST_MAX_MEMBERS - 2, real_at), (3, 4, 7))
    declined_response("mask", members_response(FAST_MAX_MEMBERS - 1, real_at))
    accepted_response("warp", members_response(FAST_MAX_MEMBERS - 1, real_at), (3, 4, 7))


@pytest.mark.parametrize("which", ["mask", "warp"])
def test_kFastMiniCap_tokens_inside_stream_options_and_usage(which):
    """kFastMiniCap (192 in mask_scan.cuh, 160 in warp_scan.cuh): the object of `stream_options` / `usage` may hold that
    many tokens (bytes outside strings, a string counting once) up to and including its '}'; one more and the document is
    left to the exact engine. include_usage / total_tokens are the LAST member, behind the tokens that use the capacity up."""
    cap = MINI_CAP[which]
    for n in (159, 160, 161, 191, 192, 193):
        rq, rs = mini_request(n), mini_response(n)
        if n <= cap:
            accepted_request(which, rq, so=1, iu=2)
            accepted_response(which, rs, (0, 0, 357))
        else:
            declined_request(which, rq)
            declined_response(which, rs)
    # the limit is the object's own: the same tokens behind its '}' are nobody's business
    far = ('{"stream_options":{"include_usage":true},"x":[' + ",".join("0" * 120) + '],"model":"m"}').encode()
    accepted_request(which, far, so=1, iu=2)


@pytest.mark.parametrize("pad", [0, 700, 1000])
def test_kFastMaxTok_512_bytes_outside_strings(pad):
    """kFastMaxTok: warp_scan.cuh keeps at most 512 tokens (bytes outside strings and the quotes) of a document; 513 in a
    document well below 2 KiB go to the exact engine. pad 0: all tokens in the first 1 KiB segment; 700: they straddle
    both; 1000: nearly all in the second. mask_scan.cuh has no such limit."""
    for n in (FAST_MAX_TOK - 1, FAST_MAX_TOK):
        accepted_request("warp", tok_request(n, pad))
        accepted_response("warp", tok_response(n, pad), (0, 0, 357))
    for n in (FAST_MAX_TOK + 1, FAST_MAX_TOK + 2):
        b = tok_request(n, pad)
        assert len(b) < FAST_MAX_LEN
        declined_request("warp", b)
        declined_response("warp", tok_response(n, pad))
        accepted_request("mask", b)
        accepted_response("mask", tok_response(n, pad), (0, 0, 357))


@pytest.mark.parametrize("kind", ["arr", "obj", "alt"])
@pytest.mark.parametrize("which", ["mask", "warp"])
def test_kFastMaxDepth_32_levels(which, kind):
    """kFastMaxDepth (one container bit per level in a 32-bit word): 32 levels, the top-level object included, are
    accepted; 33 go to the exact engine; the wrong closing bracket at the deepest level is declined and is a body error."""
    for d in (FAST_MAX_DEPTH - 1, FAST_MAX_DEPTH):
        accepted_request(which, deep_request(d, kind), st=2)
        accepted_response(which, deep_response(d, kind), (3, 4, 7))
    for d in (FAST_MAX_DEPTH + 1, FAST_MAX_DEPTH + 2):
        declined_request(which, deep_request(d, kind))
        declined_response(which, deep_response(d, kind))
    for d in (FAST_MAX_DEPTH - 1, FAST_MAX_DEPTH, FAST_MAX_DEPTH + 1):
        declined_request(which, deep_request(d, kind, spoil=True), valid=False)
        assert FILTERS[which][1](deep_response(d, kind, spoil=True)) is None
        assert orklib.parse_response_body(deep_response(d, kind, spoil=True))[0] == hm.parse_response_body(deep_response(d, kind, spoil=True))[0]


def backslash_doc(n: int, k: int) -> bytes:
    return ('{"a":"' + "z" * n + "\\" * k + ("" if k % 2 == 0 else "n") + '","model":"m"}').encode()


def test_backslash_run_filling_a_lane():
    """warp_scan.cuh declines a document when the 32 bytes of one lane are all backslashes (`m[l].B == 0xffffffff`:
    odd_tail has no answer); a run of 31, or of 32 that straddles two lanes, is accepted. mask_scan.cuh carries the run
    and accepts all of them (its own list stays in test_mask_scan.py)."""
    seen = [0, 0]
    for n in (0, 1, 7, 25, 26, 27, 31, 32, 33):
        for k in (31, 32, 33, 64, 65, 66):
            b = backslash_doc(n, k)
            start = b.index(b"\\")
            fills = any(b[a:a + 32] == b"\\" * 32 for a in range(0, len(b), 32))
            assert fills == (((start + 31) // 32) * 32 + 32 <= start + k)  # the rule, said twice
            seen[fills] += 1
            if fills:
                declined_request("warp", b)
            else:
                accepted_request("warp", b)
            accepted_request("mask", b)
    assert min(seen) > 10
    accepted_request("warp", backslash_doc(27, 32))  # 32 backslashes, bytes 33 .. 64: no lane is full
    declined_request("warp", backslash_doc(26, 32))  # bytes 32 .. 63: lane 1 exactly


# ------------------------------------------------------------------------------------------------------------------
# CPU part: the exact engine's depth limit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["arr", "obj", "alt"])
def test_kMaxDepth_10000_request_response_and_sse_event(kind):
    """kMaxDepth (kStackWords words of two bits a level: arrays AND objects): 9 999 and 10 000 containers inside each
    other parse and the member behind them is read; 10 001 is a body error. Requests (json-iterator), complete
    responses and SSE events (encoding/json) alike."""
    for d in (MAX_DEPTH - 1, MAX_DEPTH):
        b = deep_request(d, kind)
        assert orklib.parse_request_body(b) == hm.parse_request_body(b) == (0, b"m", 2, 0, 0), d
        assert hm.engine_request(b) is not None
        b = deep_response(d, kind)
        assert orklib.parse_response_body(b)[0::2] == hm.parse_response_body(b)[0::2] == (0, (3, 4, 7)), d
        ch = b"data: " + deep_event(d, kind) + b"\n\n"
        assert len(ch) < SSE_LINE_MAX
        assert orklib.parse_sse_chunk(ch) == hm.parse_sse_chunk(ch) == (0, (3, 4, 7)), d
        assert hm.parse_sse_chunk_split(ch) == (0, (3, 4, 7), False), d
    for d in (MAX_DEPTH + 1, MAX_DEPTH + 2):
        b = deep_request(d, kind)
        assert orklib.parse_request_body(b)[0] == hm.parse_request_body(b)[0] == 1, d
        assert hm.engine_request(b) is None
        b = deep_response(d, kind)
        assert orklib.parse_response_body(b)[0] == hm.parse_response_body(b)[0] == 1, d
        ch = b"data: " + deep_event(d, kind) + b"\n\n" + USAGE_EV
        assert orklib.parse_sse_chunk(ch)[0] == hm.parse_sse_chunk(ch)[0] == hm.parse_sse_chunk_split(ch)[0] == 1, d


# ------------------------------------------------------------------------------------------------------------------
# CPU part: the SSE line limit
# ------------------------------------------------------------------------------------------------------------------
def sse_all(chunk: bytes):
    """(error, usage) of the oracle, after checking that SseT and SseSplit + events say the same; third: SseSplit fell back"""
    a = orklib.parse_sse_chunk(chunk)
    c = hm.parse_sse_chunk(chunk)
    rc, usage, fell_back = hm.parse_sse_chunk_split(chunk)
    assert a[0] == c[0] == rc, (len(chunk), chunk[:60], a, c, rc)
    if rc == 0:
        assert a[1] == c[1] == usage, (len(chunk), chunk[:60], a, c, usage)
    return a[0], a[1] if rc == 0 else None, fell_back


@pytest.mark.parametrize("kind", ["string", "tokens", "comment"])
def test_sse_line_limit_65536_terminated(kind):
    """bufio.MaxScanTokenSize: a line of 65 535 bytes before its LF is a token and the usage event behind it is billed;
    65 536 bytes is a stream error (SseT::step, SseSplit::end_line). A chunk with a 65 535-byte line is still regular
    (event-parallel); the 65 536-byte one is decided by the sequential decoder."""
    for total in (SSE_LINE_MAX - 2, SSE_LINE_MAX - 1):
        line = long_line(total, kind)
        assert len(line) == total
        ch = line + (b"\n" if kind == "comment" else b"\n\n") + USAGE_EV
        assert sse_all(ch) == (0, (3, 4, 7), False), total
    for total in (SSE_LINE_MAX, SSE_LINE_MAX + 1):
        ch = long_line(total, kind) + (b"\n" if kind == "comment" else b"\n\n") + USAGE_EV
        assert sse_all(ch) == (1, None, True), total


@pytest.mark.parametrize("kind", ["string", "tokens", "comment"])
def test_sse_line_limit_65536_counts_the_cr(kind):
    """the CR of a CR LF line end is part of the scanner's token until dropCR: 65 534 bytes + CR pass, 65 535 + CR do not
    (CR LF chunks are never event-parallel)."""
    for total, err in ((SSE_LINE_MAX - 3, 0), (SSE_LINE_MAX - 2, 0), (SSE_LINE_MAX - 1, 1), (SSE_LINE_MAX, 1)):
        ch = long_line(total, kind) + (b"\r\n" if kind == "comment" else b"\r\n\r\n") + USAGE_EV.replace(b"\n", b"\r\n")
        assert sse_all(ch) == (err, None if err else (3, 4, 7), True), total


@pytest.mark.parametrize("kind", ["string", "tokens", "comment"])
def test_sse_line_limit_65536_unterminated_last_line(kind):
    """an unterminated last line is a token too (SseT::finish, SseSplit::finish): 65 535 bytes are read (and the event
    they begin is dropped, the usage before it stays), 65 536 are ErrTooLong."""
    for total in (SSE_LINE_MAX - 2, SSE_LINE_MAX - 1):
        assert sse_all(USAGE_EV + long_line(total, kind)) == (0, (3, 4, 7), False), total
        assert sse_all(USAGE_EV + long_line(total - 1, kind) + b"\r")[:2] == (0, (3, 4, 7)), total
    for total in (SSE_LINE_MAX, SSE_LINE_MAX + 1):
        assert sse_all(USAGE_EV + long_line(total, kind)) == (1, None, True), total
        assert sse_all(USAGE_EV + long_line(total - 1, kind) + b"\r")[0] == 1, total


def test_sse_line_limit_65536_around_done():
    """the scanner keeps reading behind `[DONE]`: nothing there is parsed, but a line of 65 536 bytes still fails the
    stream; in front of `[DONE]` the same."""
    done = b"data: [DONE]\n\n"
    for kind in ("string", "comment"):
        sep = b"\n" if kind == "comment" else b"\n\n"
        for total, err in ((SSE_LINE_MAX - 1, 0), (SSE_LINE_MAX, 1)):
            want = (err, None if err else (3, 4, 7), bool(err))
            assert sse_all(USAGE_EV + done + long_line(total, kind) + sep) == want, (kind, total)
            assert sse_all(USAGE_EV + done + b"data: {broken\n\n" + long_line(total, kind)) == want, (kind, total)
            assert sse_all(USAGE_EV + long_line(total, kind) + sep + done) == want, (kind, total)


def test_sse_line_limit_65536_at_every_offset_in_a_16_byte_unit():
    """SseSplit measures a line as `p - s` over 16-byte units: the long line starts at every offset 0 .. 15 of a unit."""
    for pad in range(16):
        head = b":" + b"p" * (pad + 14) + b"\n"  # a comment line of pad + 16 bytes: the next line starts at offset pad
        assert len(head) % 16 == pad
        for kind in ("string", "tokens"):
            assert sse_all(head + long_line(SSE_LINE_MAX - 1, kind) + b"\n\n" + USAGE_EV) == (0, (3, 4, 7), False), pad
            assert sse_all(head + long_line(SSE_LINE_MAX, kind) + b"\n\n" + USAGE_EV) == (1, None, True), pad
            assert sse_all(head + USAGE_EV + long_line(SSE_LINE_MAX - 1, kind)) == (0, (3, 4, 7), False), pad
            assert sse_all(head + USAGE_EV + long_line(SSE_LINE_MAX, kind)) == (1, None, True), pad


def test_sse_maximal_payload_is_the_usage_event():
    """the longest payload a `data: ` line can carry (65 535 - 6 bytes) billed as the usage event itself"""
    head = b'data: {"choices":[],"pad":"'
    tail = b'","usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'
    for total, err in ((SSE_LINE_MAX - 1, 0), (SSE_LINE_MAX, 1)):
        line = head + b"x" * (total - len(head) - len(tail)) + tail
        assert sse_all(DELTA_EV + line + b"\n\n") == (err, None if err else (3, 4, 7), bool(err))


# ------------------------------------------------------------------------------------------------------------------
# The same documents as one corpus: (body, mask_scan.cuh takes it, warp_scan.cuh takes it). The labels are the rules
# above, written out by hand; the host builds confirm them here and the device confirms them by count in the GPU part.
# ------------------------------------------------------------------------------------------------------------------
def request_corpus():
    rows = [(padded_request(FAST_MAX_LEN - 1), 1, 1), (padded_request(FAST_MAX_LEN), 1, 1), (padded_request(FAST_MAX_LEN + 1), 0, 0),
            (members_request_mixed(8), 1, 1), (members_request_mixed(9), 0, 1),
            (backslash_doc(27, 32), 1, 1), (backslash_doc(26, 32), 1, 0)]
    for klen, at in ((5, "last"), (6, "middle"), (14, "first")):
        rows += [(members_request(6, klen, at), 1, 1), (members_request(7, klen, at), 0, 1)]
    rows += [(mini_request(n), n <= 192, n <= 160) for n in (160, 161, 192, 193)]
    for pad in (0, 700):
        rows += [(tok_request(512, pad), 1, 1), (tok_request(513, pad), 1, 0)]
    for kind in ("arr", "obj", "alt"):
        rows += [(deep_request(32, kind), 1, 1), (deep_request(33, kind), 0, 0), (deep_request(32, kind, spoil=True), 0, 0),
                 (deep_request(MAX_DEPTH, kind), 0, 0), (deep_request(MAX_DEPTH + 1, kind), 0, 0)]
    return rows


def response_corpus():
    rows = [(padded_response(FAST_MAX_LEN - 1), 1, 1), (padded_response(FAST_MAX_LEN), 1, 1), (padded_response(FAST_MAX_LEN + 1), 0, 0)]
    for at in ("first", "middle", "last"):
        rows += [(members_response(6, at), 1, 1), (members_response(7, at), 0, 1)]
    rows += [(mini_response(n), n <= 192, n <= 160) for n in (160, 161, 192, 193)]
    for pad in (0, 700):
        rows += [(tok_response(512, pad), 1, 1), (tok_response(513, pad), 1, 0)]
    for kind in ("arr", "obj", "alt"):
        rows += [(deep_response(32, kind), 1, 1), (deep_response(33, kind), 0, 0), (deep_response(32, kind, spoil=True), 0, 0),
                 (deep_response(MAX_DEPTH, kind), 0, 0), (deep_response(MAX_DEPTH + 1, kind), 0, 0)]
    return rows


def sse_corpus():
    """(chunk, stream error?) — every chunk without an error bills the usage event (3, 4, 7)"""
    rows = []
    for kind in ("string", "tokens", "comment"):
        sep = b"\n" if kind == "comment" else b"\n\n"
        for total, err in ((SSE_LINE_MAX - 1, 0), (SSE_LINE_MAX, 1)):
            rows += [(long_line(total, kind) + sep + USAGE_EV, err), (USAGE_EV + long_line(total, kind), err),
                     (long_line(total - 1, kind) + b"\r" + sep + USAGE_EV, err),
                     (USAGE_EV + b"data: [DONE]\n\n" + long_line(total, kind) + sep, err)]
    head, tail = b'data: {"choices":[],"pad":"', b'","usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'
    for total, err in ((SSE_LINE_MAX - 1, 0), (SSE_LINE_MAX, 1)):
        rows.append((DELTA_EV + head + b"x" * (total - len(head) - len(tail)) + tail + b"\n\n", err))
    for kind in ("arr", "obj", "alt"):
        rows += [(b"data: " + deep_event(MAX_DEPTH, kind) + b"\n\n", 0), (b"data: " + deep_event(MAX_DEPTH + 1, kind) + b"\n\n" + USAGE_EV, 1)]
    return rows


def test_corpus_labels_are_what_the_host_builds_do():
    for rows, fns in ((request_corpus(), (hm.fast_request, hm.warp_request)), (response_corpus(), (hm.fast_response, hm.warp_response))):
        for b, mask, warp in rows:
            assert (fns[0](b) is not None) == bool(mask) and (fns[1](b) is not None) == bool(warp), (b[:80], len(b), mask, warp)
        assert 8 < sum(m for _, m, _ in rows) < len(rows) - 8 and 8 < sum(w for _, _, w in rows) < len(rows) - 8
    for ch, err in sse_corpus():
        assert sse_all(ch)[:2] == (err, None if err else (3, 4, 7)), (len(ch), ch[:60])


# ------------------------------------------------------------------------------------------------------------------
# GPU part: the corpus through every scan path of the device, the path proven by count
# ------------------------------------------------------------------------------------------------------------------
NOW = 1_700_000_000
N_TENANTS = 8
# ARKS_WARP_MAX = 2048: up to there a warp per document (warp_scan.cuh) in front of the exact engine; ARKS_FAST_MIN = 4096
# (= kSortMinBatch): from there on mask_scan.cuh in front of it; in between the exact engine alone (last_declined == -1)
SCAN_PATHS = [(2048, "warp"), (2049, "exact"), (4095, "exact"), (4096, "mask")]


def gpu_pair(gwmod, max_batch=8192, max_bytes=64 << 20):
    from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token
    toks = [simple_token("u%d" % i, "ns", "tk-%d" % i, "m", [("rpm", 10**9), ("tpm", 10**15), ("tpd", 10**16)], "q" if i % 2 else "")
            for i in range(N_TENANTS)]
    t = Tables(toks, [simple_quota("q", "ns", [("prompt", 10**15), ("total", 10**15)])], [simple_endpoint("m", "ns")])
    g = gwmod.Gateway(0, max_batch, max_bytes)
    g.load_tables(t)
    return g, orklib.Oracle(t)


def same_fields(a, b, ctx):
    for k, v in a.fields().items():
        w = b.fields()[k]
        if not np.array_equal(v, w):
            bad = np.flatnonzero((v != w).reshape(len(v), -1).any(axis=1))
            raise AssertionError(f"{ctx} field {k}: {len(bad)} rows differ, first {bad[:5]}: gpu={v[bad[:5]]} oracle={w[bad[:5]]}")


def same_state(g, o, now, ctx):
    assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), ctx + ": rate counters differ"
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), ctx + ": quota usage differs"


def plain_requests(rng, n):
    from arks_b200 import traffic
    return [traffic.chat_request_body_varied(rng, 900, stream=False).replace(traffic.MODEL.encode(), b"m") for _ in range(n)]


def plain_responses(rng, n):
    from arks_b200 import traffic
    return [traffic.chat_response_body_varied(rng, int(rng.integers(50, 401)), int(rng.integers(1, 513)), 600) for _ in range(n)]


def expect_declined(g, path, rows):
    """which path decided the batch, and that exactly the rows beyond its capacities were left to the exact engine"""
    d = g.last_declined
    if path == "exact":
        assert d == -1, (path, d)
    else:
        assert d == sum(1 for r in rows if not r[1 if path == "mask" else 2]), (path, d)


@pytest.mark.gpu
def test_request_corpus_through_every_scan_path_gpu(gwmod):
    """kFastMaxLen, kFastMaxMembers, kFastMiniCap (both), kFastMaxTok, kFastMaxDepth, the full lane of backslashes and
    kMaxDepth on the device: the boundary requests padded with plain traffic to 2 048 rows (ARKS_WARP_MAX: warp_scan.cuh),
    2 049 and 4 095 (exact engine alone) and 4 096 (ARKS_FAST_MIN / kSortMinBatch: mask_scan.cuh), boundary rows first
    and last. Every row is the oracle's; valid rows are admitted with their model; the filter declined exactly the rows
    beyond its capacities (a batch of plain traffic alone: none)."""
    from arks_b200 import abi
    from arks_b200.abi import RequestBatch
    g, o = gpu_pair(gwmod)
    rows = request_corpus()
    rng = np.random.default_rng(7)
    now = NOW
    for n, path in SCAN_PATHS:
        pad = plain_requests(rng, n)
        req = RequestBatch.from_lists(pad, [b"tk-%d" % (i % N_TENANTS) for i in range(n)], now)
        same_fields(g.handle_request_body(req), o.request_batch(req), f"plain n={n}")
        expect_declined(g, path, [])
        for where in ("first", "last"):
            now += 61
            k = len(rows)
            bodies = [r[0] for r in rows] + pad[k:] if where == "first" else pad[k:] + [r[0] for r in rows]
            at = 0 if where == "first" else n - k
            req = RequestBatch.from_lists(bodies, [b"tk-%d" % (i % N_TENANTS) for i in range(n)], now)
            a = g.handle_request_body(req)
            expect_declined(g, path, rows)
            same_fields(a, o.request_batch(req), f"requests n={n} {path} corpus {where}")
            same_state(g, o, now, f"requests n={n} {where}")
            for j, (b, _, _) in enumerate(rows):
                bad = orklib.parse_request_body(b)[0] != 0
                assert (a.reason[at + j] == abi.R_REQUEST_BODY) == bad, (n, where, j, b[:60], a.reason[at + j])
            assert np.all(a.reason[:at] == 0) and np.all(a.reason[at + k:] == 0)
        now += 61


@pytest.mark.gpu
def test_response_corpus_through_every_scan_path_gpu(gwmod):
    """the same limits on the response side (kFastKeyLensResp, `usage` as the inner object): complete bodies on the warp
    path, the exact engine alone and the fast path; usage (3, 4, 7) / (0, 0, 357) billed exactly where the oracle bills it."""
    from arks_b200 import abi
    from arks_b200.abi import ResponseBatch
    g, o = gpu_pair(gwmod)
    rows = response_corpus()
    rng = np.random.default_rng(8)
    now = NOW
    for n, path in SCAN_PATHS:
        pad = plain_responses(rng, n)
        resp = ResponseBatch.from_lists(pad, [i % N_TENANTS for i in range(n)], [abi.RESP_END_OF_STREAM] * n, now)
        same_fields(g.handle_response_body(resp), o.response_batch(resp), f"plain n={n}")
        expect_declined(g, path, [])
        for where in ("first", "last"):
            now += 61
            k = len(rows)
            bodies = [r[0] for r in rows] + pad[k:] if where == "first" else pad[k:] + [r[0] for r in rows]
            at = 0 if where == "first" else n - k
            qos = [i % N_TENANTS for i in range(n)]
            resp = ResponseBatch.from_lists(bodies, qos, [abi.RESP_END_OF_STREAM] * n, now)
            c = g.handle_response_body(resp)
            expect_declined(g, path, rows)
            same_fields(c, o.response_batch(resp), f"responses n={n} {path} corpus {where}")
            same_state(g, o, now, f"responses n={n} {where}")
            for j, (b, _, _) in enumerate(rows):
                rc, _, u = orklib.parse_response_body(b)
                assert (c.reason[at + j] == 0) == (rc == 0) and tuple(c.usage[at + j]) == (u if rc == 0 else (0, 0, 0)), (n, where, j, b[:60])
        now += 61


TINY_EV = b'data: {"choices":[{}]}\n\n'


def tiny_events(n: int, usage_at: int = -1) -> bytes:
    """a chunk of n events, the usage event at index usage_at (the others have choices and bill nothing)"""
    return b"".join(USAGE_EV if i == usage_at else TINY_EV for i in range(n))


@pytest.mark.gpu
def test_sse_line_limit_depth_and_event_list_gpu(gwmod):
    """scan_sse_kernel at its limits. Lines of 65 535 / 65 536 bytes (SseSplit::end_line / finish on the device, then
    SseT::step in the lane that turned irregular) next to ordinary chunks; the 65 529-byte payload that is the usage event
    (the 16-bit length of the event descriptor); events nested kMaxDepth deep. kSseEvCap = 320 events per warp tile: below
    kSortMinBatch a batch stays in arrival order and a tile holds bodies_per_warp(n) = ceil(n / 2048) consecutive chunks, so
    with n <= 2 048 a chunk is alone in its tile (319 / 320 / 321 / 2 049 events) and with 2 048 < n < 4 096 chunks 2k and
    2k + 1 share one: together exactly 320, 321, 270 + 51 with the overflow in either lane, the usage event as the 320th
    listed and as the first that does not fit. Rows with qos = -1 in those tiles: ARKS_R_QOS_GONE, nothing billed.
    All-SSE batches and mixed ones (the kind index)."""
    from arks_b200 import abi
    from arks_b200.abi import ResponseBatch
    g, o = gpu_pair(gwmod, 4096, 96 << 20)
    corpus = sse_corpus()
    plain = DELTA_EV * 3 + USAGE_EV + b"data: [DONE]\n\n"
    now = NOW

    def run(bodies, qos, flags, ctx, want):
        nonlocal now
        now += 61
        resp = ResponseBatch.from_lists(bodies, qos, flags, now)
        c = g.handle_response_body(resp)
        same_fields(c, o.response_batch(resp), ctx)
        same_state(g, o, now, ctx)
        for j, w in want.items():
            if qos[j] < 0:
                assert c.reason[j] == abi.R_QOS_GONE and tuple(c.usage[j]) == (0, 0, 0) and not c.counted[j], (ctx, j)
            elif w is None:
                assert c.reason[j] == abi.R_STREAMING and not c.counted[j], (ctx, j, c.reason[j])
            else:
                assert c.reason[j] != abi.R_STREAMING and tuple(c.usage[j]) == w and c.counted[j] == (w[2] != 0), (ctx, j, c.usage[j])

    # one chunk per tile (n <= 2048), and pairs (2048 < n < 4096): long lines and deep events between ordinary chunks
    for n in (len(corpus) * 2, 2048, 2050):
        bodies, want = [], {}
        for j in range(n):
            if j % 2 == 0 and j // 2 < len(corpus):
                ch, err = corpus[j // 2]
                bodies.append(ch)
                want[j] = None if err else (3, 4, 7)
            else:
                bodies.append(plain)
                want[j] = (3, 4, 7)
        qos = [j % N_TENANTS for j in range(n)]
        run(bodies, qos, [abi.RESP_STREAM] * n, f"all-sse corpus n={n}", want)
    # mixed batch: the SSE rows go through the kind index next to complete bodies
    jb = [r[0] for r in response_corpus()]
    bodies, flags, want = [], [], {}
    for j in range(2 * len(corpus)):
        if j % 2:
            bodies.append(jb[(j // 2) % len(jb)]); flags.append(abi.RESP_END_OF_STREAM)
        else:
            bodies.append(corpus[j // 2][0]); flags.append(abi.RESP_STREAM)
            want[j] = None if corpus[j // 2][1] else (3, 4, 7)
    run(bodies, [j % N_TENANTS for j in range(len(bodies))], flags, "mixed corpus", want)

    # kSseEvCap, a chunk alone in its tile
    cases = [(tiny_events(319, 318), (3, 4, 7)), (tiny_events(320, 319), (3, 4, 7)), (tiny_events(321, 320), (3, 4, 7)),
             (tiny_events(321, 319), (3, 4, 7)), (tiny_events(2049, 2048), (3, 4, 7)), (tiny_events(320), (0, 0, 0)),
             (tiny_events(321, 5) + b"data: {broken\n\n", None), (tiny_events(320, 5) + b"data: [DONE]\n\ndata: {broken\n\n", (3, 4, 7))]
    bodies = [c[0] for c in cases] + [plain] * 40
    want = {j: c[1] for j, c in enumerate(cases)}
    qos = [j % N_TENANTS if j != 2 else -1 for j in range(len(bodies))]
    run(bodies, qos, [abi.RESP_STREAM] * len(bodies), "event list, one chunk per tile", want)

    # kSseEvCap, two chunks per tile (n = 2050: bodies_per_warp == 2, arrival order)
    pairs = [(tiny_events(160, 159), tiny_events(160, 159)),   # 320: both listed, the usage event the 320th
             (tiny_events(160, 159), tiny_events(161, 160)),   # 321: one of the two is re-parsed sequentially
             (tiny_events(161, 160), tiny_events(160, 159)),
             (tiny_events(270, 0), tiny_events(51, 50)),       # 320 + 1
             (tiny_events(51, 50), tiny_events(270, 269)),
             (tiny_events(320, 319), plain),                   # 320 + 5: whichever lane comes second falls back
             (plain, tiny_events(320, 319)),
             (tiny_events(319, 318), tiny_events(1, 0)),       # exactly full
             (tiny_events(320, 319), tiny_events(321, 320))]   # both beyond
    n = 2050
    bodies = [plain] * n
    want = {}
    for p, (a, b) in enumerate(pairs):
        for base in (64 * p, n - 64 * (p + 1)):               # first and last warps of the grid
            bodies[base], bodies[base + 1] = a, b
            want[base] = want[base + 1] = (3, 4, 7)
    qos = [j % N_TENANTS for j in range(n)]
    for p in (1, 3, 5):
        qos[64 * p + 1] = -1                                    # the partner of an overflowing chunk has no qos entry
    run(bodies, qos, [abi.RESP_STREAM] * n, "event list, two chunks per tile", want)
