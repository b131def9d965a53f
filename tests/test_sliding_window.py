"""Opt-in sliding-window rate limits (include/arks_gateway.h: arks_set_sliding_window): the limiter reads
est = cur + floor(prev * (W - e) / W) per rule instead of the fixed window's cur, and with the rate-limit report on each figure
gets the seconds until its estimate reaches 0 (x-ratelimit-reset-*) and a rate-limit 429 the seconds until it admits again
(retry-after, expiresAt).

CPU: the hand scenario of DESIGN.md §5 in both modes; the oracle's sliding mode (tests/sliding_oracle.c) against a serial
model of Redis keys written here, on seeded event logs; the oracle's reset / retry bisection against a linear scan; the
header shaping of both hosts; the process flag.
GPU: limit_admit's closed form over the estimate against the oracle on every scan path, across minute and day windows
(adjacent and skipped), around the hot-group threshold, with N4 / N5, across a generation swap; switching on at any batch;
switched off (or never set), nothing changes."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from arks_b200 import abi, replies
from arks_b200.abi import ArksRequestBatch, ArksRequestResult, ArksResponseBatch, ArksResponseResult, ArksTables
from arks_b200.abi import RequestBatch, RequestResult, ResponseBatch, ResponseResult
from arks_b200.tables import Tables, simple_endpoint, simple_token

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
sys.path.insert(0, HERE)
import test_ratelimit_headers as RH  # noqa: E402  (its GPU tables, traffic and helpers)

NOW = RH.NOW
MIN0 = NOW - NOW % 60  # a minute boundary (NOW is 20 s into its minute)
WIN = (60, 86400, 60, 86400)
RULES = ("rpm", "rpd", "tpm", "tpd")
I64 = 1 << 63


# ---- the oracle with the sliding-window mode ---------------------------------------------------------------------------------
def sw_oracle_path() -> str:
    os.makedirs(BUILD, exist_ok=True)
    out = os.path.join(BUILD, "libarks_oracle_sw.so")
    od = os.path.join(ROOT, "oracle")
    srcs = [os.path.join(HERE, "sliding_oracle.c"), os.path.join(ROOT, "include", "arks_gateway.h")] + \
        [os.path.join(od, f) for f in os.listdir(od) if f.endswith((".c", ".h"))]
    if RH._stale(out, srcs):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-Wl,-Bsymbolic", "-o", out,
                               os.path.join(HERE, "sliding_oracle.c"), os.path.join(od, "ork_json.c")])
    return out


_L = None


def sw_lib():
    global _L
    if _L is None:
        L = C.CDLL(sw_oracle_path())
        L.ork_create.restype = C.c_void_p
        L.ork_create.argtypes = [C.POINTER(ArksTables)]
        L.ork_destroy.argtypes = [C.c_void_p]
        L.ork_reload.argtypes = [C.c_void_p, C.POINTER(ArksTables)]
        for f in ("ork_set_sliding_window", "ork_set_ratelimit_report", "ork_set_precharge"):
            getattr(L, f).argtypes = [C.c_void_p, C.c_int]
            getattr(L, f).restype = None
        L.ork_set_estimates.argtypes = [C.c_void_p, abi.u32p, C.c_uint32]
        L.ork_set_estimates.restype = None
        L.ork_request_batch.argtypes = [C.c_void_p, C.POINTER(ArksRequestBatch), C.POINTER(ArksRequestResult)]
        L.ork_response_batch.argtypes = [C.c_void_p, C.POINTER(ArksResponseBatch), C.POINTER(ArksResponseResult)]
        L.ork_snapshot_rate.argtypes = [C.c_void_p, C.c_int64, abi.i64p]
        L.ork_snapshot_rate_prev.argtypes = [C.c_void_p, C.c_int64, abi.i64p]
        L.ork_snapshot_metrics.argtypes = [C.c_void_p, abi.i64p]
        L.ork_snapshot_quota.argtypes = [C.c_void_p, abi.i64p]
        L.ork_sliding_times.argtypes = [C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int,
                                        C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.ork_sliding_times.restype = None
        _L = L
    return _L


class SwOracle:
    """the oracle with arks_set_sliding_window's mode (and the rate-limit report when report=True)"""

    def __init__(self, tables, sliding=True, report=False):
        self.tables, self._ts = tables, tables.c_struct()
        self.h = sw_lib().ork_create(C.byref(self._ts))
        assert self.h
        self.report = report
        self.set_sliding(sliding)
        sw_lib().ork_set_ratelimit_report(self.h, int(report))

    def __del__(self):
        if getattr(self, "h", None):
            sw_lib().ork_destroy(self.h)
            self.h = None

    def set_sliding(self, on):
        self.sliding = bool(on)
        sw_lib().ork_set_sliding_window(self.h, int(bool(on)))

    def reload(self, tables):
        ts = tables.c_struct()
        assert sw_lib().ork_reload(self.h, C.byref(ts)) == 0
        self.tables, self._ts = tables, ts

    def set_precharge(self, on):
        sw_lib().ork_set_precharge(self.h, int(bool(on)))

    def set_estimates(self, est):
        self._est = np.ascontiguousarray(est, np.uint32)
        sw_lib().ork_set_estimates(self.h, abi.ptr(self._est, abi.u32p), len(self._est))

    def request_batch(self, b):
        r = RequestResult.empty(b.n, report=self.report, sliding=self.sliding)
        bs, rs = b.c_struct(), r.c_struct()
        assert sw_lib().ork_request_batch(self.h, C.byref(bs), C.byref(rs)) == 0
        return r

    def response_batch(self, b):
        r = ResponseResult.empty(b.n)
        bs, rs = b.c_struct(), r.c_struct()
        assert sw_lib().ork_response_batch(self.h, C.byref(bs), C.byref(rs)) == 0
        return r

    def _snap(self, f, now):
        out = np.zeros((self.tables.n_qos, 4), np.int64)
        getattr(sw_lib(), f)(self.h, int(now), abi.ptr(out, abi.i64p))
        return out

    def snapshot_rate(self, now):
        return self._snap("ork_snapshot_rate", now)

    def snapshot_rate_prev(self, now):
        return self._snap("ork_snapshot_rate_prev", now)

    def snapshot_metrics(self):
        out = np.zeros((self.tables.n_qos, abi.METRIC_COLS), np.int64)
        sw_lib().ork_snapshot_metrics(self.h, abi.ptr(out, abi.i64p))
        return out

    def snapshot_quota(self):
        out = np.zeros((self.tables.n_quotas, 3), np.int64)
        sw_lib().ork_snapshot_quota(self.h, abi.ptr(out, abi.i64p))
        return out


def sliding_times(c, p, left, w, limit, req):
    a, b = C.c_uint32(), C.c_uint32()
    sw_lib().ork_sliding_times(c, p, left, w, limit, req, C.byref(a), C.byref(b))
    return a.value, b.value


def reqs(token, n, now, model="m"):
    return RH.reqs(token, n, now, model)


def resp_body(total):
    return b'{"model":"m","usage":{"prompt_tokens":1,"completion_tokens":1,"total_tokens":%d}}' % total


# ---- 1. the hand scenario (DESIGN.md §5) ---------------------------------------------------------------------------------------
def test_hand_scenario_rpm_10_both_modes():
    t = RH.small([("rpm", 10)])
    times = (MIN0 + 59, MIN0 + 60, MIN0 + 90, MIN0 + 120)
    admitted = {}
    for sliding in (False, True):
        o = SwOracle(t, sliding=sliding)
        admitted[sliding] = [int((o.request_batch(reqs("tk", 10, now)).reason == abi.R_OK).sum()) for now in times]
    assert admitted[False] == [10, 10, 0, 10]  # the fixed window: 20 requests inside two seconds
    assert admitted[True] == [10, 0, 5, 5]
    # the numbers behind them: at 60 s est = 0 + floor(10 * 60 / 60) = 10; at 90 s floor(10 * 30 / 60) = 5; at 120 s prev = 5, e = 0
    o = SwOracle(t, sliding=True, report=True)
    o.request_batch(reqs("tk", 10, MIN0 + 59))
    a = o.request_batch(reqs("tk", 2, MIN0 + 60))
    assert a.reason.tolist() == [abi.R_RATE_LIMIT] * 2 and a.cur_usage.tolist() == [10, 10] and a.limit_max.tolist() == [10, 10]
    assert o.snapshot_rate(MIN0 + 60)[0, 0] == 0 and o.snapshot_rate_prev(MIN0 + 60)[0, 0] == 10
    # reset: floor(10 (60 - d) / 60) = 0 from d = 55; retry: <= 9 from d = 1 (one second later est = 9)
    assert RH.figs(a, 0)[0] == (0, 10, 0) and a.rl_reset[0].tolist() == [55, 0] and a.rl_retry.tolist() == [1, 1]
    b = o.request_batch(reqs("tk", 6, MIN0 + 90))
    assert b.reason.tolist() == [0] * 5 + [abi.R_RATE_LIMIT] and int(b.cur_usage[5]) == 10
    # the 429: C = 5, P = 10, e = 30: E(d) = 5 + floor(10 (30 - d) / 60) <= 9 from d = 0? E(0) = 10, E(1) = 9 -> 1
    assert int(b.rl_retry[5]) == 1 and int(b.rl_retry[0]) == 0
    # reset of the last admitted row: C = 5, P = 10 -> 5 until 30 s, then floor(5 (90 - d) / 60) = 0 from d = 79
    assert b.rl_reset[4].tolist() == [79, 0]
    c = o.request_batch(reqs("tk", 6, MIN0 + 120))
    assert c.reason.tolist() == [0] * 5 + [abi.R_RATE_LIMIT]
    assert o.snapshot_rate_prev(MIN0 + 120)[0, 0] == 5 and o.snapshot_rate(MIN0 + 120)[0, 0] == 5


def test_retry_without_an_admitting_time_is_reset():
    # rpm 0: nothing ever admits, retry-after names the time the estimate reaches 0
    assert sliding_times(3, 7, 20, 60, 0, 1) == sliding_times(3, 7, 20, 60, -5, 1)
    # C = 3, P = 7, W - e = 20: E(d) >= 3 for d < 20, then floor(3 (80 - d) / 60), which is 0 from d = 61
    assert sliding_times(3, 7, 20, 60, 0, 1) == (61, 61) == linear(3, 7, 20, 60, 0, 1)


# ---- 2. the oracle against a serial model of Redis keys ------------------------------------------------------------------------
def wrap(x):
    return (x + I64) % (1 << 64) - I64


def window_start(now, rule):
    return now - (now + 62135596800) % WIN[rule]


class RedisModel:
    """GET / INCRBY on keys (ns, user, model, rule, window start); the limiter of check.go with the estimate in place of cur"""

    def __init__(self, qos_rules, keys, sliding):
        self.kv, self.rules, self.keys, self.sliding = {}, qos_rules, keys, sliding

    def get(self, q, rule, ws):
        return self.kv.get(self.keys[q] + (rule, ws), 0)

    def incr(self, q, rule, ws, n):
        k = self.keys[q] + (rule, ws)
        self.kv[k] = wrap(self.kv.get(k, 0) + n)

    def est(self, q, rule, now):
        ws, w = window_start(now, rule), WIN[rule]
        cur = self.get(q, rule, ws)
        if not self.sliding:
            return cur
        return wrap(cur + self.get(q, rule, ws - w) * (w - (now - ws)) // w)

    def requests(self, now, qs, est=None):
        out, pending = [], []
        for i, q in enumerate(qs):
            row = (abi.R_OK, 0, 0, 0)
            for j, (rule, lim) in enumerate(self.rules[q]):
                e = self.est(q, rule, now)
                if wrap(e + (1 if rule < 2 else 0)) > lim:
                    row = (abi.R_RATE_LIMIT, j, e, lim)
                    break
            if row[0] == abi.R_OK:
                for rule, _ in self.rules[q]:
                    if rule < 2:
                        self.incr(q, rule, window_start(now, rule), 1)
                    elif est is not None and est[i]:
                        pending.append((q, rule, int(est[i])))
            out.append(row)
        for q, rule, n in pending:
            self.incr(q, rule, window_start(now, rule), n)
        return out

    def responses(self, now, rows):
        for q, total in rows:
            if total:
                for rule, _ in self.rules[q]:
                    if rule >= 2:
                        self.incr(q, rule, window_start(now, rule), total)

    def snapshot(self, now, back):
        return np.array([[self.get(q, r, window_start(now, r) - back * WIN[r]) for r in range(4)] for q in range(len(self.rules))],
                        np.int64)


def model_tables(rng, n_tok):
    toks, rules = [], []
    big = [I64 - 1, I64 - 2, -3, 0, 1]
    for i in range(n_tok):
        rl = []
        for _ in range(int(rng.integers(1, 5))):
            rule = int(rng.integers(0, 4))
            lim = int(rng.choice(big)) if rng.random() < 0.15 else int(rng.integers(0, 40 if rule < 2 else 4000))
            rl.append((rule, lim))
        toks.append(simple_token(f"u{i}", "ns", f"t{i}", "m", [(RULES[r], v) for r, v in rl]))
        rules.append(rl)
    return Tables(toks, [], [simple_endpoint("m", "ns")]), rules


def time_steps(rng, start, n):
    """adjacent and skipping roll-overs, e = 0 and e = W - 1 of minutes and days"""
    now, out = start, []
    for _ in range(n):
        k = rng.random()
        if k < 0.25:
            now += int(rng.integers(0, 20))
        elif k < 0.45:
            now = now - now % 60 + 60 * int(rng.integers(1, 3))  # e = 0 of the next (or the one after) minute
        elif k < 0.6:
            now = now - now % 60 + 59 + (60 if now % 60 == 59 else 0)  # e = W - 1
        elif k < 0.7:
            now += int(rng.integers(121, 400))  # a skipped minute
        elif k < 0.8:
            now = now - now % 86400 + 86400 * int(rng.integers(1, 3)) - int(rng.integers(0, 2))  # day edge, e = W - 1 or 0
        else:
            now += int(rng.integers(20, 70))
        out.append(now)
    return out


@pytest.mark.parametrize("seed", range(6))
def test_oracle_sliding_mode_equals_a_serial_model_of_redis_keys(seed):
    rng = np.random.default_rng(seed)
    n_tok = 12
    t, rules = model_tables(rng, n_tok)
    keys = [("ns", f"u{i}", "m") for i in range(n_tok)]
    sliding = seed % 3 != 2  # a third of the logs with the mode off: the fixed window
    o = SwOracle(t, sliding=sliding)
    o.set_precharge(True)
    m = RedisModel(rules, keys, sliding)
    for step, now in enumerate(time_steps(rng, NOW, 60)):
        if rng.random() < 0.6:
            n = int(rng.integers(1, 40))
            qs = [int(x) for x in rng.integers(0, n_tok, n)]
            est = rng.integers(0, 50, n).astype(np.uint32) if rng.random() < 0.4 else None
            if est is not None:
                o.set_estimates(est)
            b = RequestBatch.from_lists([b'{"model":"m","messages":[]}'] * n, [f"t{q}".encode() for q in qs], now)
            a = o.request_batch(b)
            want = m.requests(now, qs, est)
            got = list(zip(a.reason.tolist(), a.detail.tolist(), a.cur_usage.tolist(), a.limit_max.tolist()))
            assert got == want, (seed, step)
        else:
            n = int(rng.integers(1, 10))
            rows = []
            for _ in range(n):
                k = rng.random()
                total = int(rng.integers(-50, 500)) if k < 0.8 else int(rng.choice([I64 - 7, -I64 + 3, 2**62]))
                rows.append((int(rng.integers(0, n_tok)), total))
            o.response_batch(ResponseBatch.from_lists([resp_body(x) for _, x in rows], [q for q, _ in rows],
                                                      [abi.RESP_END_OF_STREAM] * n, now))
            m.responses(now, rows)
        assert np.array_equal(o.snapshot_rate(now), m.snapshot(now, 0)), (seed, step)
        assert np.array_equal(o.snapshot_rate_prev(now), m.snapshot(now, 1)), (seed, step)


# ---- 3. reset / retry: the bisection against a linear scan ----------------------------------------------------------------------
def linear(c, p, left, w, limit, req):
    c, p = max(c, 0), max(p, 0)

    def E(d):
        if d < left:
            return c + p * (left - d) // w
        if d < left + w:
            return c * (left + w - d) // w
        return 0
    ds = range(left + w + 1)
    reset = next(d for d in ds if E(d) == 0)
    retry = next((d for d in ds if E(d) + req <= limit), reset)
    return reset, retry


@pytest.mark.parametrize("w", [60, 86400])
def test_reset_and_retry_bisection_equals_a_linear_scan(w):
    rng = np.random.default_rng(w)
    cases = [(0, 0, 1, 0, 1), (0, 0, w, 0, 0), (5, 10, w, 10, 1), (I64 - 1, I64 - 1, 1, 0, 1), (-4, -9, w, 3, 1),
             (1, 0, 1, 0, 0), (10, 10, w, -1, 0)]
    for _ in range(400 if w == 60 else 12):
        big = rng.random() < 0.2
        c = int(rng.integers(-5, I64 - 1)) if big else int(rng.integers(-5, 3 * w))
        p = int(rng.integers(-5, I64 - 1)) if rng.random() < 0.2 else int(rng.integers(-5, 3 * w))
        lim = int(rng.integers(-2, max(c, 1) + 5)) if not big else int(rng.integers(-2, I64 - 1))
        cases.append((c, p, int(rng.integers(1, w + 1)), lim, int(rng.integers(0, 2))))
    for c, p, left, lim, req in cases:
        assert sliding_times(c, p, left, w, lim, req) == linear(c, p, left, w, lim, req), (c, p, left, w, lim, req)


# ---- 4. the shaping: reset and retry replace the window end ------------------------------------------------------------------
def test_headers_under_the_sliding_window():
    t = RH.small([("rpm", 10), ("tpm", 100)])
    e = np.array([0, 1], np.uint8)
    hs = replies.ratelimit_headers(abi.R_RATE_LIMIT, 0, 0, MIN0 + 60, e, [10, 100], [0, 100], t, rl_reset=[55, 0], rl_retry=1)
    assert hs == [("retry-after", "1"), ("x-ratelimit-limit-requests", "10"), ("x-ratelimit-remaining-requests", "0"),
                  ("x-ratelimit-reset-requests", "55s"), ("x-ratelimit-limit-tokens", "100"),
                  ("x-ratelimit-remaining-tokens", "100"), ("x-ratelimit-reset-tokens", "0s")]
    hs = dict(replies.ratelimit_headers(abi.R_OK, 0, 0, MIN0, e, [10, 100], [3, 1], t, rl_reset=[3600 + 61, 86399], rl_retry=0))
    assert (hs["x-ratelimit-reset-requests"], hs["x-ratelimit-reset-tokens"]) == ("1h1m1s", "23h59m59s") and "retry-after" not in hs
    st, h, v, msg = replies.request_error_reply(abi.R_RATE_LIMIT, 0, 10, 10, MIN0 + 60, t, 0, b"tk", "m", rl_retry=1)
    assert msg == '{"ruleName":"rpm","overLimit":true,"currentUsage":10,"limitMax":10,"expiresAt":"%s"}' % replies._rfc3339(MIN0 + 61)
    # without the sliding window: the window end, as before
    st, h, v, msg2 = replies.request_error_reply(abi.R_RATE_LIMIT, 0, 10, 10, MIN0 + 60, t, 0, b"tk", "m")
    assert replies._rfc3339(MIN0 + 120) in msg2


def test_process_flag_is_the_library_switch():
    from arks_b200 import __main__ as M

    class Rec:
        def __init__(self):
            self.calls = []

        def set_sliding_window(self, on):
            self.calls.append(on)

    class Cb:
        def __init__(self):
            self.b = Rec()

    for argv, want in (([], []), (["--ratelimiter.sliding-window"], [True])):
        a = M.parse_args(argv)
        e, cb = Rec(), Cb()
        M.configure_sliding_window(e, cb, a)
        assert e.calls == want and cb.b.calls == want
        e = Rec()
        M.configure_sliding_window(e, None, a)
        assert e.calls == want


# ---- GPU ------------------------------------------------------------------------------------------------------------------------
def same_sliding_report(a, b, where):
    RH.same_report(a, b, where)
    for k in ("rl_reset", "rl_retry"):
        x, y = getattr(a, k), getattr(b, k)
        assert np.array_equal(x, y), (where, k, np.flatnonzero((x != y).reshape(len(x), -1).any(1))[:8])


def same_state(g, o, now, where):
    assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), where
    assert np.array_equal(g.snapshot_rate_prev(now), o.snapshot_rate_prev(now)), where
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), where


def edge_times():
    d = RH.day_edge()
    # minute and day windows, adjacent roll-overs at e = 0 and e = W - 1, a skipped minute, a skipped day
    return (d - 121, d - 61, d - 60, d - 30, d - 1, d, d + 59, d + 60, d + 300, d + 2 * 86400 + 30)


def answer(g, o, a, now, total=45):
    ok = np.flatnonzero(a.reason == abi.R_OK)
    if len(ok):
        rb = ResponseBatch.from_lists([resp_body(total)] * len(ok), a.qos[ok], [abi.RESP_END_OF_STREAM] * len(ok), now)
        c, d = g.handle_response_body(rb), o.response_batch(rb)
        assert np.array_equal(c.reason, d.reason) and np.array_equal(c.counted, d.counted)


@pytest.mark.gpu
@pytest.mark.parametrize("report", [True, False])
@pytest.mark.parametrize("n", [1200, 3000, 8192])  # warp path (<= 2048), exact engine alone, two-stage fast path (>= 4096)
def test_gpu_sliding_equals_the_oracle(gwmod, n, report):
    t = RH.gpu_tables()
    g = gwmod.Gateway(0, 16384, 32 << 20)
    g.load_tables(t)
    g.enable_metrics(True)
    g.set_ratelimit_report(report)
    g.set_sliding_window(True)
    o = SwOracle(t, sliding=True, report=report)
    seen = set()
    for step, now in enumerate(edge_times()):
        req = RH.gpu_traffic(t, n, now, seed=300 * n + step)
        a, want = g.handle_request_body(req), o.request_batch(req)
        RH.same_decisions(a, want, (n, step))
        if report:
            same_sliding_report(a, want, (n, step))
            seen |= {int(x) for x in a.rl_retry[a.reason == abi.R_RATE_LIMIT]}
        else:
            assert a.rl_entry is None and a.rl_reset is None
        same_state(g, o, now, (n, step))
        assert np.array_equal(g.snapshot_metrics(), o.snapshot_metrics()), (n, step)
        answer(g, o, a, now)
        same_state(g, o, now, (n, step))
    if report:
        assert len(seen) > 3  # retry times other than the window end


@pytest.mark.gpu
def test_gpu_hot_groups_straddling_their_limit(gwmod):
    """255 / 256 / 257 / 258 arrivals of one qos entry against an estimate that leaves room for some of them"""
    lims = (256, 255, 300, 257)
    t = Tables([simple_token(f"h{i}", "ns", f"hot{i}", "m", [("rpm", lim), ("tpm", 10**6), ("rpd", 10**6)])
                for i, lim in enumerate(lims)], [], [simple_endpoint("m", "ns")])
    g = gwmod.Gateway(0, 4096, 8 << 20)
    g.load_tables(t)
    g.set_ratelimit_report(True)
    g.set_sliding_window(True)
    o = SwOracle(t, sliding=True, report=True)
    for step, now in enumerate((MIN0 + 50, MIN0 + 65, MIN0 + 100, MIN0 + 125)):
        toks = sum(([f"hot{i}".encode()] * s for i, s in enumerate((255, 256, 257, 258))), [])
        rng = np.random.default_rng(step)
        toks = [toks[i] for i in rng.permutation(len(toks))]
        b = RequestBatch.from_lists([b'{"model":"m","messages":[]}'] * len(toks), toks, now)
        a, want = g.handle_request_body(b), o.request_batch(b)
        RH.same_decisions(a, want, step)
        same_sliding_report(a, want, step)
        same_state(g, o, now, step)
        if step:
            k = [int(((a.qos == q) & (a.reason == abi.R_OK)).sum()) for q in range(4)]
            assert any(0 < x < s for x, s in zip(k, (255, 256, 257, 258))), k  # some group straddles its limit


@pytest.mark.gpu
def test_gpu_sliding_with_precharge_and_metering(gwmod):
    from arks_b200 import bpe
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    t = RH.gpu_tables(seed=5)
    g = gwmod.Gateway(0, 16384, 32 << 20)
    g.load_tables(t)
    g.load_bpe(bpe.load_tokenizer(text))
    g.set_precharge(True)
    g.set_stream_metering(True)
    g.set_ratelimit_report(True)
    g.set_sliding_window(True)
    o = SwOracle(t, sliding=True, report=True)
    o.set_precharge(True)
    for step, (n, now) in enumerate(((1500, MIN0 + 30), (9000, MIN0 + 70), (600, MIN0 + 119), (2000, MIN0 + 180))):
        req = RH.gpu_traffic(t, n, now, seed=50 + step)
        a = g.handle_request_body(req)
        o.set_estimates(a.bpe_count)
        want = o.request_batch(req)
        RH.same_decisions(a, want, step)
        same_sliding_report(a, want, step)
        same_state(g, o, now, step)
        answer(g, o, a, now)


@pytest.mark.gpu
def test_gpu_prev_follows_its_key_across_a_generation_swap(gwmod):
    t1 = RH.gpu_tables(n_small=300, seed=6)
    # the next generation: one token added in front (every index moves), one removed, the rest kept
    from unittest import mock
    with mock.patch.object(RH, "Tables", lambda *lists: lists):  # the CRD lists behind RH.gpu_tables
        toks, quotas, eps = RH.gpu_tables(n_small=300, seed=6, front=[simple_token("new", "ns", "tnew", "m", [("rpm", 2)])])
    t2 = Tables([x for x in toks if x["metadata"]["name"] != "u7"], quotas, eps)
    g = gwmod.Gateway(0, 16384, 32 << 20)
    g.load_tables(t1)
    g.set_ratelimit_report(True)
    g.set_sliding_window(True)
    o = SwOracle(t1, sliding=True, report=True)
    for step, now in enumerate((MIN0 + 10, MIN0 + 40, MIN0 + 70, MIN0 + 95, MIN0 + 130)):
        if step == 3:  # prev holds the minute before: it has to follow its key
            g.commit_tables(g.prepare_tables(t2))
            o.reload(t2)
        t = t2 if step >= 3 else t1
        req = RH.gpu_traffic(t, 2500, now, seed=70 + step)
        a, want = g.handle_request_body(req), o.request_batch(req)
        RH.same_decisions(a, want, step)
        same_sliding_report(a, want, step)
        same_state(g, o, now, step)
        answer(g, o, a, now)


@pytest.mark.gpu
def test_gpu_switching_on_at_any_batch_is_exact(gwmod):
    """prev is kept while the switch is off, so a context switched on at batch k decides from then on exactly as the oracle,
    which keeps its older keys whatever the mode"""
    t = RH.gpu_tables(seed=8)
    times = edge_times()[:7]
    for k in (2, 5):
        g = gwmod.Gateway(0, 16384, 32 << 20)
        g.load_tables(t)
        o = SwOracle(t, sliding=False)
        for s, now in enumerate(times):
            if s == k:
                g.set_sliding_window(True)
                o.set_sliding(True)
            req = RH.gpu_traffic(t, 2000, now, seed=90 + s)
            a, want = g.handle_request_body(req), o.request_batch(req)
            RH.same_decisions(a, want, (k, s))
            same_state(g, o, now, (k, s))
            answer(g, o, a, now)


@pytest.mark.gpu
def test_gpu_switched_off_changes_nothing(gwmod):
    t = RH.gpu_tables(seed=4)
    never, off, toggled = (gwmod.Gateway(0, 16384, 32 << 20) for _ in range(3))
    for g in (never, off, toggled):
        g.load_tables(t)
        g.enable_metrics(True)
        g.set_ratelimit_report(True)
    off.set_sliding_window(False)
    toggled.set_sliding_window(True)
    toggled.set_sliding_window(False)
    d = RH.day_edge()
    for step, (n, now) in enumerate(((700, d - 61), (9000, d - 1), (3000, d + 2), (1500, d + 200))):
        req = RH.gpu_traffic(t, n, now, seed=17 + step)
        l0 = [g.launch_count for g in (never, off, toggled)]
        outs = [g.handle_request_body(req, RequestResult.empty(n, report=True, sliding=True)) for g in (never, off, toggled)]
        launches = [g.launch_count - x for g, x in zip((never, off, toggled), l0)]
        assert launches[0] == launches[1] == launches[2], launches
        for r in outs[1:]:
            RH.same_decisions(outs[0], r, step)
            RH.same_report(outs[0], r, step)
            assert np.array_equal(outs[0].bpe_count, r.bpe_count)
        for r in outs:  # a batch run without the sliding window leaves reset / retry alone
            assert (r.rl_reset == 0xEEEEEEEE).all() and (r.rl_retry == 0xEEEEEEEE).all()
        for g in (off, toggled):
            assert np.array_equal(never.snapshot_rate(now), g.snapshot_rate(now))
            assert np.array_equal(never.snapshot_rate_prev(now), g.snapshot_rate_prev(now))
            assert np.array_equal(never.snapshot_metrics(), g.snapshot_metrics())
        ok = np.flatnonzero(outs[0].reason == abi.R_OK)
        rb = ResponseBatch.from_lists([RH.RESP] * len(ok), outs[0].qos[ok], [abi.RESP_END_OF_STREAM] * len(ok), now)
        for g in (never, off, toggled):
            g.handle_response_body(rb)


def test_cpp_and_python_shapers_agree_under_the_sliding_window():
    RH_in_subprocess("check_sliding_shapers_agree")


def RH_in_subprocess(fn):
    code = f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_sliding_window as T; T.{fn}()"
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT)


def check_sliding_shapers_agree():
    from arks_b200 import cpphost
    t = Tables(RH.FX["tokens"] + [simple_token("v", "ns", "tk2", "qwen-7b", [("tpd", 9), ("rpd", 3), ("rpm", 1), ("tpm", 4)])],
               RH.FX["quotas"], RH.FX["endpoints"] + [simple_endpoint("qwen-7b", "ns")])
    h = RH.ShimHost(t)
    try:
        gen = h.b.request(b"tk2", b'{"model":"qwen-7b"}').gen
        rng = np.random.default_rng(11)
        for k in range(400):
            reason = int(rng.choice([0, 8, 9, 1, 7]))
            detail, q, now = int(rng.integers(0, 4)), int(rng.integers(0, 2)), int(NOW + rng.integers(-10**6, 10**6))
            ent = tuple(int(x) if rng.random() < 0.8 else RH.NONE for x in rng.integers(0, 4, 2))
            lim, rem = [int(x) for x in rng.integers(0, 10**9, 2)], [int(x) for x in rng.integers(0, 10**6, 2)]
            sliding = k % 4 != 3
            reset = [int(x) for x in rng.integers(0, 2 * 86400, 2)]
            retry = int(rng.integers(0, 2 * 86400)) if reason == abi.R_RATE_LIMIT else 0
            d = cpphost.RequestDecision()
            d.reason, d.detail, d.qos, d.now_unix, d.gen, d.rl_sliding = reason, detail, q, now, gen, int(sliding)
            for j in range(2):
                d.rl_entry[j], d.rl_limit[j], d.rl_remaining[j], d.rl_reset[j] = ent[j], lim[j], rem[j], reset[j]
            d.rl_retry = retry
            want = replies.ratelimit_headers(reason, detail, q, now, list(ent), lim, rem, t, *((reset, retry) if sliding else ()))
            assert h.b.ratelimit_headers(d) == want, (reason, detail, q, now, ent, sliding)
    finally:
        h.close()
