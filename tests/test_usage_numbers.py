"""Usage counters written as numbers with a fraction or an exponent, long digit strings and quoted counters, against
gjson's Result.Int as `pymodel.gjson_int` states it with Python's int and float alone.

The referee is never the oracle or the device. The corpus goes where a decimal-to-int64 conversion goes wrong: the
int64 wrap of long plain integers, values within a few units of 2^52, 2^53 and 2^63 (2^63 - 512 rounds up to 2^63), .5
ties above 2^53, long runs of 9s below an integer, trailing zeros against negative exponents, exponents up to +-400,
signed zeros and numbers of 512 to 4 096 bytes. Each number sits in every usage field behind prefixes of every length
mod 16, so that it starts at every byte of the engine's 16-byte units. CPU: the oracle, the host builds of the exact
engine (JSON, SSE sequential and SSE event-split paths) and the two filters, which may decline instead. GPU: every scan
path of handle_response_body, with the rate, quota and metric counters that the values wrap."""
import random

import numpy as np
import pytest

import hostmachine as hm
import orklib
from arks_b200 import abi
from arks_b200.abi import RequestBatch, ResponseBatch
from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token
from pymodel import INT64_MIN, gjson_int

NOW = 1_700_000_000
P52, P53, P63 = 1 << 52, 1 << 53, 1 << 63


def _digits(r, n, lead_nonzero=True):
    s = "".join(r.choice("0123456789") for _ in range(n))
    return (r.choice("123456789") + s[1:]) if lead_nonzero and n else s


def _sci(v: int, frac: str = ""):
    """forms of the decimal `v.frac` (v >= 0): plain with a fraction, and with the point moved by an exponent"""
    d = str(v) + frac
    p = len(str(v))
    out = [f"{v}.{frac or '0'}", f"{d[0]}.{d[1:] or '0'}e{p - 1}", f"{d[0]}.{d[1:] or '0'}E+{p - 1}",
           f"{d}e-{len(frac)}", f"0.{d}e{p}"]
    return out


def number_corpus(seed=2024):
    """raw JSON number tokens (bytes); every one is valid JSON"""
    r = random.Random(seed)
    nums = []
    # plain integers of 1..40 digits, both signs: the int64 wrap at 2^64
    for n in range(1, 41):
        for _ in range(3):
            d = _digits(r, n)
            nums += [d, "-" + d]
    for v in (P63 - 1, P63, P63 + 1, (1 << 64) - 1, 1 << 64, (1 << 64) + 1, P53 - 1, P53, P53 + 1, 10**19, 10**20):
        nums += [str(v), "-" + str(v)]
    nums += ["0", "-0"]
    # within a few units of 2^52, 2^53 and 2^63, and around the rounding boundary 2^63 - 512
    for base in (P52, P53, P63, P63 - 512, P63 - 1024):
        for dv in range(-5, 6):
            v = base + dv
            for frac in ("", "0", "25", "5", "50000000000000001", "75", "0000001", "9999999", "49999999999999999999"):
                for s in _sci(v, frac):
                    nums += [s, "-" + s]
    # .5 ties above 2^53 (doubles are multiples of 2^s there): halfway cases round to even
    for s in range(1, 11):
        for _ in range(6):
            q = r.randrange(1 << 52, 1 << 53)
            v = (q << s) + (1 << (s - 1))
            if v >= P63:
                continue
            for t in _sci(v) + _sci(v, "0000000000000000000001") + _sci(v - 1, "99999999999999999999"):
                nums += [t, "-" + t]
    for k in range(0, 40):
        for t in _sci(P53 + 2 * k + 1, "5") + _sci(P53 + 2 * k, "5"):
            nums.append(t)
    # long runs of 9s just below an integer
    for n in range(16, 61):
        for ip in ("0", "2", "1023", str(P52 - 1), str(P53 - 2), str(r.randrange(1, 10**12))):
            nums += [ip + "." + "9" * n, "-" + ip + "." + "9" * n]
        nums += ["9" * n + "e-" + str(n), "2" + "9" * n + "e-" + str(n), "0." + "9" * n + "e1"]
    # mantissas with trailing zeros against negative exponents
    for k in range(0, 41):
        for j in (k - 1, k, k + 1, k + 3):
            if j >= 0:
                m = r.choice(["1", "3", "9223372036854775807", "9007199254740993", "12"])
                nums += [f"{m}{'0' * k}e-{j}", f"-{m}{'0' * k}.{'0' * r.randint(1, 3)}e-{j}"]
    # exponents 0..+-400, e / E, with and without +
    for ex in list(range(0, 25)) + [30, 99, 100, 101, 300, 308, 309, 310, 324, 325, 399, 400]:
        for _ in range(2):
            m = _digits(r, r.randint(1, 25))
            mant = m[0] + ("." + m[1:] if len(m) > 1 else "")
            e = r.choice("eE")
            nums += [f"{mant}{e}{ex}", f"{mant}{e}+{ex}", f"-{mant}{e}-{ex}", f"{mant}{e}-{ex}", f"{mant}{e}{ex:03d}"]
    nums += ["-0.0", "0.0", "0e400", "0E-400", "-0e+400", "1e-400", "-1e-400", "0.000e0", "1e400", "-1e400"]
    # numbers of 512 to 4 096 bytes
    for L in (512, 513, 1000, 2047, 2048, 4000, 4096):
        z = L - 8
        nums += ["0." + "0" * z + "1e" + str(z + 1),                        # exactly 1
                 "0." + "0" * (z - 2) + "123e" + str(z + 19),                # 1.23e19: beyond int64
                 "1." + "0" * z + "1",                                       # 1 plus a tail
                 "2." + "9" * (L - 2),                                       # rounds to 3
                 "9007199254740993." + "0" * (L - 18) + "1",                 # just above the 2^53 + 1 tie
                 "9223372036854775295." + "9" * (L - 20),                    # above 2^63 - 513: still below the boundary
                 _digits(r, 19) + "." + _digits(r, L - 20, False),
                 "-" + _digits(r, 5) + "." + _digits(r, L - 7, False) + "e13"]
    nums.append("0." + "0" * 600 + "1e700")  # 1e99: a long number whose value is out of range
    # random fraction / exponent numbers: 1..25 significant digits, exponents up to +-30
    for _ in range(4000):
        m = _digits(r, r.randint(1, 25))
        dot = r.randint(1, len(m))
        t = m[:dot] + ("." + m[dot:] if dot < len(m) else "")
        if r.random() < 0.7 or dot == len(m):
            t += r.choice("eE") + r.choice(["", "+", "-"]) + str(r.randint(0, 30))
        nums.append(("-" if r.random() < 0.5 else "") + t)
    return [s.encode() for s in nums]


def tokens():
    """every number, and every number quoted (gjson parseInt of the string)"""
    nums = number_corpus()
    return nums + [b'"' + n + b'"' for n in nums if len(n) < 600]


OTHER = (b"7", b"11", b"18")


def usage_obj(tok, f):
    v = [OTHER[0], OTHER[1], OTHER[2]]
    v[f] = tok
    return b'{"prompt_tokens":%s,"completion_tokens":%s,"total_tokens":%s}' % tuple(v)


def want_usage(tok, f):
    v = [gjson_int(OTHER[0]), gjson_int(OTHER[1]), gjson_int(OTHER[2])]
    v[f] = gjson_int(tok)
    return tuple(v)


def json_body(tok, f, pad):
    return b'{"id":"' + b"x" * pad + b'","model":"m","usage":' + usage_obj(tok, f) + b"}"


def sse_body(tok, f, pad, crlf=False):
    b = (b": " + b"p" * pad + b"\ndata: {\"id\":\"c\",\"choices\":[],\"usage\":" + usage_obj(tok, f) + b"}\n\n"
         b"data: [DONE]\n\n")
    return b.replace(b"\n", b"\r\n") if crlf else b


def cases():
    """(token, field, pad): every token in every field; the pad walks the number's start through all 16 offsets"""
    out = []
    for k, t in enumerate(tokens()):
        for f in range(3):
            out.append((t, f, (5 * k + 3 * f) % 16 + 16 * (k % 2)))
    return out


KNOWN = [  # total_tokens: (raw, Go's answer)
    (b"999999999999999e3", 999999999999998976),
    (b"9.007199254740993e15", 9007199254740992),
    (b"9007199254740993.5", 9007199254740994),
    (b"2.99999999999999999999", 3),
    (b"1000000000000000000000e-3", 1000000000000000000),
    (b"-43532650.201462016849340E-10", 0),
    (b"9223372036854775295.0", 9223372036854774784),
    (b"-9223372036854775808.0", INT64_MIN),
    (b"9223372036854775296.0", INT64_MIN),           # 2^63 - 512: the tie rounds to even, 2^63
    (b"0." + b"0" * 600 + b"1e700", INT64_MIN),      # 1e99, 600 bytes of zeros
    (b"0.99999999999999999", 1),                     # within half an ulp below 1
    (b"0.9999999999999999", 0),
    (b"4503599627370495.5", 4503599627370495),       # 2^52 - 0.5 is a double
    (b"4503599627370495.75", 4503599627370496),      # halfway between 2^52 - 0.5 and 2^52: ties to the even 2^52
    (b"4503599627370496.5", 4503599627370496),       # 2^52 + 0.5: ties to even
    (b"4503599627370497.5", 4503599627370498),
    (b"-0.0", 0),
    (b"1e-400", 0),
    (b"0e400", 0),
    (b"18446744073709551617", 1),                    # plain: wraps
    (b'"-18446744073709551617"', -1),
    (b'"1.5"', 0),
]


def test_referee_known_answers():
    for raw, want in KNOWN:
        assert gjson_int(raw) == want, raw


def test_corpus_covers_the_edges():
    toks = tokens()
    assert max(len(t) for t in toks) >= 4096 and sum(len(t) >= 512 for t in toks) >= 50
    vals = [gjson_int(t) for t in toks]
    assert vals.count(INT64_MIN) > 100
    assert sum(abs(v) > P53 for v in vals if v != INT64_MIN) > 200
    starts = {(len(json_body(t, f, p).split(t)[0])) % 16 for t, f, p in cases()[:600]}
    assert starts == set(range(16))


@pytest.mark.parametrize("raw,want", KNOWN)
def test_known_answers_every_path(raw, want):
    u = (7, 11, want)
    assert orklib.parse_response_body(json_body(raw, 2, 3))[2] == u
    assert orklib.parse_sse_chunk(sse_body(raw, 2, 3))[1] == u
    assert hm.parse_response_body(json_body(raw, 2, 3))[2] == u
    assert hm.parse_sse_chunk(sse_body(raw, 2, 3)) == (0, u)
    assert hm.parse_sse_chunk(sse_body(raw, 2, 3, crlf=True)) == (0, u)
    assert hm.parse_sse_chunk_split(sse_body(raw, 2, 3)) == (0, u, False)


def _check_one(tok, f, pad):
    want = want_usage(tok, f)
    ctx = (tok[:80], len(tok), f, pad)
    jb, sb = json_body(tok, f, pad), sse_body(tok, f, pad)
    a = orklib.parse_response_body(jb)
    assert a[0] == 0 and a[2] == want, (ctx, a, want)
    a = orklib.parse_sse_chunk(sb)
    assert a == (0, want), (ctx, a, want)
    c = hm.parse_response_body(jb)
    assert c[0] == 0 and c[2] == want, (ctx, c, want)
    assert hm.parse_sse_chunk(sb) == (0, want), ctx
    assert hm.parse_sse_chunk(sse_body(tok, f, pad, crlf=True)) == (0, want), ctx
    assert hm.parse_sse_chunk_split(sb) == (0, want, False), ctx
    for filt in (hm.fast_response, hm.warp_response):
        got = filt(jb)
        assert got is None or got[1] == want, (ctx, filt.__name__, got, want)
    return hm.fast_response(jb) is None


def test_every_number_every_path_cpu():
    n_declined = n = 0
    for tok, f, pad in cases():
        n_declined += _check_one(tok, f, pad)
        n += 1
    assert n > 20000 and 0 < n_declined < n, (n, n_declined)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: every scan path, and the counters the values land in
# ---------------------------------------------------------------------------------------------------------------------

def gpu_tables():
    toks = [simple_token("a", "ns", "ta", "m", [("tpm", 10**12), ("tpd", 10**15), ("rpm", 10**6)], "qa"),
            simple_token("b", "ns", "tb", "m", [("tpm", 10**9), ("tpm", 5 * 10**8), ("tpd", 10**12), ("rpd", 10**6)], "qb"),
            simple_token("c", "ns", "tc", "m", [("tpd", 10**13)], "")]
    quotas = [simple_quota("qa", "ns", [("prompt", 10**12), ("response", 10**12), ("total", 10**12)]),
              simple_quota("qb", "ns", [("total", 10**13), ("total", 10**14), ("prompt", 10**13), ("response", 10**13)])]
    return Tables(toks, quotas, [simple_endpoint("m", "ns")])


def _run(g, o, bodies, flags, wants, now, ctx, filtered, precharged=None):
    qos = [i % 3 for i in range(len(bodies))]
    resp = ResponseBatch.from_lists(bodies, qos, flags, now)
    if precharged is not None:
        resp.precharged = np.ascontiguousarray(precharged, np.uint32)
    c = g.handle_response_body(resp)
    declined = g.last_declined
    d = o.response_batch(resp)
    assert np.array_equal(c.reason, np.zeros(len(bodies), np.uint8)), ctx
    want = np.array(wants, np.int64)
    bad = np.flatnonzero(np.any(c.usage != want, axis=1))
    assert len(bad) == 0, (ctx, len(bad), [(bodies[i][:120], c.usage[i].tolist(), want[i].tolist()) for i in bad[:3]])
    assert np.array_equal(c.counted, (want[:, 2] != 0).astype(c.counted.dtype)), ctx
    for k, v in c.fields().items():
        assert np.array_equal(v, d.fields()[k]), (ctx, k)
    if filtered:
        assert declined > 0, (ctx, declined)
    assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), ctx
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), ctx
    assert np.array_equal(g.snapshot_metrics(), o.snapshot_metrics()), ctx


def _batch(cs, n, kind, seed):
    r = random.Random(seed)
    pick = [cs[r.randrange(len(cs))] for _ in range(n)]
    bodies, flags, wants = [], [], []
    for k, (t, f, pad) in enumerate(pick):
        sse = kind == "sse" or kind == "sse_crlf" or (kind == "mixed" and k % 2)
        if sse:
            bodies.append(sse_body(t, f, pad, crlf=kind == "sse_crlf"))
            flags.append(abi.RESP_STREAM | (abi.RESP_END_OF_STREAM if k % 3 else 0))
        else:
            bodies.append(json_body(t, f, pad))
            flags.append(abi.RESP_END_OF_STREAM)
        wants.append(want_usage(t, f))
    return bodies, flags, wants


@pytest.mark.gpu
def test_every_scan_path_and_the_counters_gpu(gwmod):
    t = gpu_tables()
    g = gwmod.Gateway(0, 8192, 64 << 20)
    g.load_tables(t)
    g.enable_metrics()
    o = orklib.Oracle(t)
    cs = cases()
    now = NOW
    plan = [("json", 2048, True), ("json", 700, True), ("json", 3000, False), ("json", 4095, False), ("json", 8192, True),
            ("sse", 3000, False), ("sse", 8192, False), ("sse_crlf", 2500, False), ("mixed", 5000, False)]
    for step, (kind, n, filtered) in enumerate(plan):
        bodies, flags, wants = _batch(cs, n, kind, 100 + step)
        _run(g, o, bodies, flags, wants, now, f"{kind} x{n}", filtered)
        now += 1
    # the whole corpus once, on the fast path and its slow list
    for lo in range(0, len(cs), 8192):
        part = cs[lo:lo + 8192]
        if len(part) < 4096:
            part = part + cs[:4096 - len(part)]
        bodies = [json_body(*c) for c in part]
        _run(g, o, bodies, [abi.RESP_END_OF_STREAM] * len(part), [want_usage(c[0], c[1]) for c in part], now,
             f"corpus {lo}", True)
    # N4 on: `total - precharged` on extreme totals, modulo 2^64 like the counters
    g.set_precharge(True)
    o.set_precharge(True)
    bodies, flags, wants = _batch(cs, 3000, "mixed", 7)
    pre = np.random.default_rng(7).integers(0, 1 << 32, len(bodies), dtype=np.uint64).astype(np.uint32)
    _run(g, o, bodies, flags, wants, now, "precharged", False, precharged=pre)
    g.set_precharge(False)
    o.set_precharge(False)
    # the wrapped counters decide the next requests as the reference's do
    rates = g.snapshot_rate(now)
    assert (rates[:, 2:] < 0).any() or (rates[:, 2:] > 10**12).any(), rates
    for k in range(3):
        who = [b"ta", b"tb", b"tc"] * 300
        req = RequestBatch.from_lists([b'{"model":"m"}'] * len(who), who, now + k)
        a, b = g.handle_request_body(req), o.request_batch(req)
        for f, v in a.fields().items():
            assert np.array_equal(v, b.fields()[f]), (k, f)
        assert np.array_equal(g.snapshot_rate(now + k), o.snapshot_rate(now + k))
        assert np.array_equal(g.snapshot_quota(), o.snapshot_quota())
