"""Pricing-based quotas (include/arks_gateway.h: ARKS_QT_COST, arks_set_endpoint_price): a `cost` ArksQuota item, checked at
request time like every item and billed prompt_tokens x p_prompt + completion_tokens x p_completion at the prices of the
ArksEndpoint each qos entry resolves to.

CPU: the hand scenario of DESIGN.md §5 with its numbers; the test-side oracle (tests/cost_oracle.c) against a serial model of
Redis keys written here, on seeded event logs; table validation on the snapshot-check route; the provider; both shapers.
GPU: every scan path against the oracle with cost items, config 4 with price policies at full size, generation swaps, stream
metering, the pre-charge, quota sharing refused, the four-column sync, and the launch count."""
import copy
import ctypes as C
import datetime
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from arks_b200 import abi, cpphost, replies, traffic
from arks_b200.abi import ArksRequestBatch, ArksRequestResult, ArksResponseBatch, ArksResponseResult, ArksTables
from arks_b200.abi import RequestBatch, RequestResult, ResponseBatch, ResponseResult
from arks_b200.tables import Tables, endpoint_pricing, simple_endpoint, simple_quota, simple_token

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BUILD = os.path.join(HERE, "_build")
FX = json.load(open(os.path.join(HERE, "golden", "quickstart.json")))
NOW = 1_700_000_020
M64 = 1 << 64
QT = abi.QUOTA_TYPES


def wrap(x: int) -> int:
    """int64 modulo 2^64, as every counter adds"""
    return (x + (1 << 63)) % M64 - (1 << 63)


# ---- the oracle with cost items ---------------------------------------------------------------------------------------------
def _stale(out, srcs):
    return not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs)


def cost_oracle_path() -> str:
    os.makedirs(BUILD, exist_ok=True)
    out = os.path.join(BUILD, "libarks_oracle_cost.so")
    od = os.path.join(ROOT, "oracle")
    srcs = [os.path.join(HERE, "cost_oracle.c"), os.path.join(ROOT, "include", "arks_gateway.h")] + \
        [os.path.join(od, f) for f in os.listdir(od) if f.endswith((".c", ".h"))]
    if _stale(out, srcs):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-Wl,-Bsymbolic", "-o", out,
                               os.path.join(HERE, "cost_oracle.c"), os.path.join(od, "ork_json.c")])
    return out


_L = None


def cost_lib():
    global _L
    if _L is None:
        L = C.CDLL(cost_oracle_path())
        vp = C.c_void_p
        L.ork_create.restype = vp
        L.ork_create.argtypes = [C.POINTER(ArksTables)]
        L.ork_destroy.argtypes = [vp]
        L.ork_reload.argtypes = [vp, C.POINTER(ArksTables)]
        L.ork_set_precharge.argtypes = [vp, C.c_int]
        L.ork_set_precharge.restype = None
        L.ork_set_estimates.argtypes = [vp, abi.u32p, C.c_uint32]
        L.ork_set_estimates.restype = None
        L.ork_request_batch.argtypes = [vp, C.POINTER(ArksRequestBatch), C.POINTER(ArksRequestResult)]
        L.ork_response_batch.argtypes = [vp, C.POINTER(ArksResponseBatch), C.POINTER(ArksResponseResult)]
        L.ork_snapshot_rate.argtypes = [vp, C.c_int64, abi.i64p]
        L.ork_snapshot_quota.argtypes = [vp, abi.i64p]
        L.ork_snapshot_quota_cost.argtypes = [vp, abi.i64p]
        L.ork_set_endpoint_price.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_char_p, C.c_uint32, C.c_int64, C.c_int64]
        L.ork_meter_charge.argtypes = [vp, C.c_uint32, abi.i32p, abi.i64p, C.c_int, C.c_int64]
        L.ork_meter_charge.restype = None
        L.ork_sync_quota_usage.argtypes = [vp, C.c_uint32, C.POINTER(C.c_uint32), abi.i64p, C.c_int]
        L.ork_sync_quota_usage4.argtypes = [vp, C.c_uint32, C.POINTER(C.c_uint32), abi.i64p, C.c_int]
        _L = L
    return _L


class CostOracle:
    """the oracle with `cost` items; prices are read at create / reload, like the library reads them at prepare"""

    def __init__(self, tables, prices=None):
        self.tables, self._ts = tables, tables.c_struct()
        self.h = cost_lib().ork_create(C.byref(self._ts))
        if not self.h:
            raise ValueError("the cost oracle refused the tables")
        if prices:
            for (ns, name), (p, c) in prices.items():
                self.set_price(ns, name, p, c)
            self.reload(tables)

    def __del__(self):
        if getattr(self, "h", None):
            cost_lib().ork_destroy(self.h)
            self.h = None

    def set_price(self, ns, name, p, c):
        a, b = ns.encode(), name.encode()
        assert cost_lib().ork_set_endpoint_price(self.h, a, len(a), b, len(b), int(p), int(c)) == 0

    def reload(self, tables):
        ts = tables.c_struct()
        assert cost_lib().ork_reload(self.h, C.byref(ts)) == 0
        self.tables, self._ts = tables, ts

    def set_precharge(self, on):
        cost_lib().ork_set_precharge(self.h, int(bool(on)))

    def set_estimates(self, est):
        self._est = np.ascontiguousarray(est, np.uint32)
        cost_lib().ork_set_estimates(self.h, abi.ptr(self._est, abi.u32p), len(self._est))

    def request_batch(self, b):
        r = RequestResult.empty(b.n)
        bs, rs = b.c_struct(), r.c_struct()
        assert cost_lib().ork_request_batch(self.h, C.byref(bs), C.byref(rs)) == 0
        return r

    def response_batch(self, b):
        r = ResponseResult.empty(b.n)
        bs, rs = b.c_struct(), r.c_struct()
        assert cost_lib().ork_response_batch(self.h, C.byref(bs), C.byref(rs)) == 0
        return r

    def meter(self, qos, counts, side, now):
        q, c = np.ascontiguousarray(qos, np.int32), np.ascontiguousarray(counts, np.int64)
        cost_lib().ork_meter_charge(self.h, len(q), abi.ptr(q, abi.i32p), abi.ptr(c, abi.i64p), side, int(now))

    def snapshot_rate(self, now):
        out = np.zeros((self.tables.n_qos, 4), np.int64)
        cost_lib().ork_snapshot_rate(self.h, int(now), abi.ptr(out, abi.i64p))
        return out

    def snapshot_quota(self):
        out = np.zeros((self.tables.n_quotas, 3), np.int64)
        cost_lib().ork_snapshot_quota(self.h, abi.ptr(out, abi.i64p))
        return out

    def snapshot_quota_cost(self):
        out = np.zeros(self.tables.n_quotas, np.int64)
        cost_lib().ork_snapshot_quota_cost(self.h, abi.ptr(out, abi.i64p))
        return out

    def sync_quota_usage(self, present, used, restore=False):
        """Gateway.sync_quota_usage's convention: used [n, 3] (the cost column ignored) or [n, 4]"""
        f = cost_lib().ork_sync_quota_usage4 if used.shape[1] == 4 else cost_lib().ork_sync_quota_usage
        action = np.zeros(self.tables.n_quotas, np.uint8)
        for q in range(self.tables.n_quotas):
            p = C.c_uint32(int(present[q]))
            u = np.ascontiguousarray(used[q], np.int64)
            action[q] = f(self.h, q, C.byref(p), abi.ptr(u, abi.i64p), int(restore))
            present[q], used[q] = p.value, u
        return action


# ---- traffic helpers --------------------------------------------------------------------------------------------------------
def req_batch(rows, now):
    """rows: [(token, model, stream)]"""
    bodies = [(b'{"model":"%s","stream":true,"stream_options":{"include_usage":true},"messages":[]}' if s else
               b'{"model":"%s","messages":[]}') % m.encode() for t, m, s in rows]
    return RequestBatch.from_lists(bodies, [t.encode() for t, _, _ in rows], now)


def usage_body(p, c, t=None):
    t = p + c if t is None else t
    return b'{"model":"m","usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}' % (p, c, t)


def usage_chunk(p, c, t=None):
    t = p + c if t is None else t
    return b'data: {"choices":[],"usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}\n\n' % (p, c, t)


def resp_batch(rows, now):
    """rows: [(qos index, usage (p, c, t), stream)]"""
    bodies = [(usage_chunk if s else usage_body)(*u) for _, u, s in rows]
    flags = [abi.RESP_STREAM if s else abi.RESP_END_OF_STREAM for _, _, s in rows]
    return ResponseBatch.from_lists(bodies, [q for q, _, _ in rows], flags, now)


def quickstart_cost(items, extra_tokens=(), extra_endpoints=()):
    """the quickstart tenant with its quota's items replaced by `items`"""
    q = copy.deepcopy(FX["quotas"])
    q[0]["spec"]["quotas"] = [{"type": t, "value": v} for t, v in items]
    return Tables(FX["tokens"] + list(extra_tokens), q, FX["endpoints"] + list(extra_endpoints))


# ---- 1. the hand scenario ---------------------------------------------------------------------------------------------------
def test_hand_scenario_with_written_down_numbers():
    """quickstart tenant, qwen-7b priced prompt 2 / completion 8: the README response (25 / 20 / 45) bills 25*2 + 20*8 = 210"""
    price = {("default", "qwen-7b"): (2, 8)}
    llama = {"arksEndpoint": {"name": "llama"}, "rateLimits": [], "quota": {"name": "basic-quota"}}
    tok = copy.deepcopy(FX["tokens"][0])
    tok["spec"]["qos"].append(llama)  # an unpriced model on the same quota
    t = Tables([tok], [simple_quota("basic-quota", "default", [("prompt", 100000), ("total", 600000), ("cost", 210)])],
               FX["endpoints"] + [simple_endpoint("llama", "default")])
    o = CostOracle(t, price)
    a = o.request_batch(req_batch([("sk-test123456", "qwen-7b", False)], NOW))
    assert a.reason[0] == abi.R_OK
    o.response_batch(resp_batch([(0, (25, 20, 45), False)], NOW))
    assert o.snapshot_quota_cost().tolist() == [210]
    assert o.snapshot_quota().tolist() == [[25, 0, 45]]
    # cost == limit admits
    a = o.request_batch(req_batch([("sk-test123456", "qwen-7b", False)], NOW + 1))
    assert a.reason[0] == abi.R_OK
    # the unpriced model bills 0 ...
    o.response_batch(resp_batch([(1, (1000, 1000, 2000), False)], NOW + 1))
    assert o.snapshot_quota_cost().tolist() == [210]
    # ... limit + 1 is denied by the cost item (index 2) with the cost figures, on both models of the shared quota
    o.response_batch(resp_batch([(0, (0, 0, 1), False), (0, (1, 0, 1), False)], NOW + 1))  # total 1, prompt 0: nothing; then 2
    assert o.snapshot_quota_cost().tolist() == [212]
    t2 = Tables([tok], [simple_quota("basic-quota", "default", [("prompt", 100000), ("total", 600000), ("cost", 211)])],
                FX["endpoints"] + [simple_endpoint("llama", "default")])
    o.reload(t2)
    a = o.request_batch(req_batch([("sk-test123456", "qwen-7b", False), ("sk-test123456", "llama", False)], NOW + 2))
    assert a.reason.tolist() == [abi.R_QUOTA, abi.R_QUOTA]
    assert a.detail.tolist() == [2, 2] and a.cur_usage.tolist() == [212, 212] and a.limit_max.tolist() == [211, 211]
    # two cost items bill twice
    t3 = quickstart_cost([("cost", 10**9), ("total", 10**9), ("cost", 10**9)])
    o3 = CostOracle(t3, price)
    o3.request_batch(req_batch([("sk-test123456", "qwen-7b", False)], NOW))
    o3.response_batch(resp_batch([(0, (25, 20, 45), False)], NOW))
    assert o3.snapshot_quota_cost().tolist() == [420]
    assert o3.snapshot_quota().tolist() == [[0, 0, 45]]


def test_cost_figures_come_before_later_token_items_and_after_earlier_ones():
    price = {("default", "qwen-7b"): (1, 1)}
    o = CostOracle(quickstart_cost([("prompt", 5), ("cost", 3), ("total", 4)]), price)
    o.response_batch(resp_batch([(0, (2, 2, 4), False)], NOW))  # prompt 2, cost 4, total 4
    a = o.request_batch(req_batch([("sk-test123456", "qwen-7b", False)], NOW))
    assert (a.reason[0], a.detail[0], a.cur_usage[0], a.limit_max[0]) == (abi.R_QUOTA, 1, 4, 3)
    o.response_batch(resp_batch([(0, (4, 0, 4), False)], NOW))  # prompt 6 > 5: the earlier item wins
    a = o.request_batch(req_batch([("sk-test123456", "qwen-7b", False)], NOW))
    assert (a.reason[0], a.detail[0], a.cur_usage[0], a.limit_max[0]) == (abi.R_QUOTA, 0, 6, 5)


# ---- 2. the oracle against a serial model of Redis keys ------------------------------------------------------------------------
WIN = (60, 86400, 60, 86400)


class RedisModel:
    """ArksToken / ArksQuota / ArksEndpoint objects and Redis: rate keys (ns, user, model, rule, window start) and four quota keys
    (ns, quota, type) per ArksQuota, `cost` the fourth. Prices are read when a configuration is loaded"""

    def __init__(self, tokens, quotas, endpoints, prices):
        self.rate, self.quota, self.price_map = {}, {}, dict(prices)
        self.precharge, self.est = False, None
        self.load(tokens, quotas, endpoints)

    def load(self, tokens, quotas, endpoints):
        self.tok = {}
        for t in tokens:
            ns, user = t["metadata"].get("namespace", "default"), t["metadata"]["name"]
            if t["spec"]["token"] in self.tok:
                continue
            self.tok[t["spec"]["token"]] = (ns, user, [(q["arksEndpoint"]["name"], (q.get("quota") or {}).get("name", ""),
                                                        [(abi.RULES[r["type"]], int(r["value"])) for r in q.get("rateLimits") or []])
                                                       for q in t["spec"].get("qos") or []])
        self.quotas = {}
        for q in quotas:
            self.quotas.setdefault((q["metadata"].get("namespace", "default"), q["metadata"]["name"]),
                                   [(QT[i["type"]], int(i["value"])) for i in q["spec"]["quotas"]])
        self.eps = {(e["metadata"].get("namespace", "default"), e["metadata"]["name"]) for e in endpoints}
        self.prices = {k: v for k, v in self.price_map.items() if k in self.eps}

    def entry(self, key):
        ns, user, model = key
        for tk, (n, u, qos) in self.tok.items():
            if (n, u) == (ns, user):
                for m, qn, rls in qos:
                    if m == model:
                        return m, qn, rls
        return None

    def request(self, rows, now):
        out, pend = [], []
        for i, (token, model, _) in enumerate(rows):
            if token not in self.tok:
                out.append((abi.R_TOKEN_NOT_FOUND, 0, 0, 0))
                continue
            ns, user, qos = self.tok[token]
            e = next((x for x in qos if x[0] == model), None)
            if e is None:
                out.append((abi.R_MODEL_NOT_IN_TOKEN, 0, 0, 0))
                continue
            if (ns, model) not in self.eps:
                out.append((abi.R_NO_MODEL_BACKENDS, 0, 0, 0))
                continue
            _, qn, rls = e
            key = (ns, user, model)
            res = None
            for j, (rule, lim) in enumerate(rls):
                cur = self.rate.get(key + (rule, now - now % WIN[rule]), 0)
                if wrap(cur + (1 if rule < 2 else 0)) > lim:
                    res = (abi.R_RATE_LIMIT, j, cur, lim)
                    break
            if res is None and qn:
                if (ns, qn) not in self.quotas:
                    res = (abi.R_QUOTA_CONFIG, 0, 0, 0)
                else:
                    for j, (ty, lim) in enumerate(self.quotas[(ns, qn)]):
                        cur = self.quota.get((ns, qn, ty), 0)
                        if cur > lim:
                            res = (abi.R_QUOTA, j, cur, lim)
                            break
            if res is None:
                res = (abi.R_OK, 0, 0, 0)
                for rule, _ in rls:
                    if rule < 2:
                        self._add_rate(key + (rule, now - now % WIN[rule]), 1)
                    elif self.precharge and self.est is not None and self.est[i] not in (0, 0xFFFFFFFF):
                        pend.append((key + (rule, now - now % WIN[rule]), int(self.est[i])))
            out.append(res)
        for k, v in pend:
            self._add_rate(k, v)
        self.est = None
        return out

    def _add_rate(self, k, v):
        self.rate[k] = wrap(self.rate.get(k, 0) + v)

    def _add_quota(self, k, v):
        self.quota[k] = wrap(self.quota.get(k, 0) + v)

    def response(self, rows, now, precharged=None):
        """rows: [(qos key or None, (p, c, t))]"""
        for i, (key, (p, c, t)) in enumerate(rows):
            e = self.entry(key) if key else None
            if e is None or t == 0:
                continue
            _, qn, rls = e
            for rule, _ in rls:
                if rule >= 2:
                    self._add_rate(key + (rule, now - now % WIN[rule]), t - (int(precharged[i]) if precharged is not None else 0))
            self._bill(key, qn, {0: p, 1: c, 2: t}, p, c)

    def _bill(self, key, qn, tokens, p, c):
        ns = key[0]
        if not qn or (ns, qn) not in self.quotas:
            return
        pp, pc = self.prices.get((ns, key[2]), (0, 0))
        for ty, _ in self.quotas[(ns, qn)]:
            self._add_quota((ns, qn, ty), p * pp + c * pc if ty == QT["cost"] else tokens.get(ty, 0))

    def meter(self, rows, side, now):
        """N5: [(qos key, count)]: the count on tpm / tpd, on the side's and the total item, at the side's price"""
        for key, n in rows:
            e = self.entry(key)
            if e is None or n == 0:
                continue
            _, qn, rls = e
            for rule, _ in rls:
                if rule >= 2:
                    self._add_rate(key + (rule, now - now % WIN[rule]), n)
            self._bill(key, qn, {side: n, 2: n}, n if side == 0 else 0, n if side == 1 else 0)

    def quota_rows(self, tables):
        out = []
        for q in range(tables.n_quotas):
            k = (tables.strings[tables.quota_ns_str[q]].decode(), tables.strings[tables.quota_name_str[q]].decode())
            out.append([self.quota.get(k + (ty,), 0) for ty in range(4)])
        return np.array(out, np.int64).reshape(-1, 4)


def qos_keys(tables):
    return [(tables.token_namespace[tables.qos_token[q]], tables.token_user[tables.qos_token[q]], tables.qos_model_name[q])
            for q in range(tables.n_qos)]


def random_config(rng, n_ns=4, drop_endpoint=False):
    """several namespaces, each with users whose qos entries for 3 models share one or two quotas with mixed items"""
    tokens, quotas, endpoints = [], [], []
    for k in range(n_ns):
        ns = "ns%d" % k
        for m in ("m0", "m1", "m2"):
            if not (drop_endpoint and k == 0 and m == "m1"):
                endpoints.append(simple_endpoint(m, ns))
        for qn in ("qa", "qb"):
            items = []
            for _ in range(int(rng.integers(1, 5))):
                ty = ["prompt", "response", "total", "cost"][int(rng.integers(0, 4))]
                items.append({"type": ty, "value": int(rng.choice([rng.integers(0, 3000), rng.integers(-5, 5), 2**63 - 1]))})
            quotas.append({"metadata": {"namespace": ns, "name": qn}, "spec": {"quotas": items}})
        for u in range(3):
            qos = []
            for m in ("m0", "m1", "m2"):
                qos.append({"arksEndpoint": {"name": m}, "quota": {"name": ["qa", "qb", ""][int(rng.integers(0, 3)) if u else 0]},
                            "rateLimits": [{"type": r, "value": int(rng.integers(2, 50) * (1000 if r[0] == "t" else 1))}
                                           for r in ("rpm", "tpm", "rpd", "tpd") if rng.random() < 0.6]})
            tokens.append({"metadata": {"namespace": ns, "name": "u%d" % u}, "spec": {"token": "sk-%d-%d" % (k, u), "qos": qos}})
    return tokens, quotas, endpoints


def random_prices(rng, n_ns=4, big=False):
    out = {}
    for k in range(n_ns):
        for m in ("m0", "m1", "m2"):
            if rng.random() < 0.8:
                hi = (1 << 62) if big else 5000
                out[("ns%d" % k, m)] = (int(rng.integers(0, hi)), int(rng.integers(0, hi)))
    return out


def compare(o, model, tables, now):
    got = np.concatenate([o.snapshot_quota(), o.snapshot_quota_cost()[:, None]], axis=1)
    assert np.array_equal(got, model.quota_rows(tables))
    keys = qos_keys(tables)
    want = np.array([[model.rate.get(keys[q] + (r, now - now % WIN[r]), 0) for r in range(4)] for q in range(tables.n_qos)],
                    np.int64).reshape(-1, 4)
    assert np.array_equal(o.snapshot_rate(now), want)


@pytest.mark.parametrize("seed", range(6))
def test_oracle_matches_a_model_of_redis_keys(seed):
    rng = np.random.default_rng(seed)
    big = seed % 2 == 1  # prices near 2^62: products and sums wrap
    tokens, quotas, endpoints = random_config(rng)
    prices = random_prices(rng, big=big)
    t = Tables(tokens, quotas, endpoints)
    o, model = CostOracle(t, prices), RedisModel(tokens, quotas, endpoints, prices)
    if seed >= 4:  # the pre-charge on: quotas (and the cost key) untouched by it
        o.set_precharge(True)
        model.precharge = True
    toks = ["sk-%d-%d" % (k, u) for k in range(4) for u in range(3)] + ["sk-unknown"]
    now = NOW
    n_cost_denials = 0
    for step in range(40):
        now += int(rng.choice([0, 1, 7, 61]))
        ev = rng.random()
        if ev < 0.1:  # price changes, a reload, maybe an endpoint deleted
            new = random_prices(rng, big=big)
            for k in set(prices) | set(new):
                p = new.get(k, (0, 0))
                o.set_price(k[0], k[1], *p)
                model.price_map[k] = p
            prices = new
            tokens, quotas, endpoints = random_config(np.random.default_rng([seed, step]), drop_endpoint=rng.random() < 0.5)
            t = Tables(tokens, quotas, endpoints)
            o.reload(t)
            model.load(tokens, quotas, endpoints)
            continue
        rows = [(toks[int(rng.integers(0, len(toks)))], ["m0", "m1", "m2", "mx"][int(rng.integers(0, 4))], False)
                for _ in range(int(rng.integers(1, 40)))]
        est = rng.integers(0, 300, len(rows)).astype(np.uint32)
        o.set_estimates(est)
        model.est = est
        r = o.request_batch(req_batch(rows, now))
        want = model.request(rows, now)
        got = list(zip(r.reason.tolist(), r.detail.tolist(), r.cur_usage.tolist(), r.limit_max.tolist()))
        assert got == want, (seed, step)
        keys = qos_keys(t)
        for i, (reason, detail, _, _) in enumerate(want):
            if reason == abi.R_QUOTA:
                ns, user, m = keys[r.qos[i]]
                qn = model.entry((ns, user, m))[1]
                n_cost_denials += model.quotas[(ns, qn)][detail][0] == QT["cost"]
        # responses of admitted rows and some rows whose qos entry is gone; usage may be negative or near int64's ends
        resp, mrows, pre = [], [], []
        for i in np.flatnonzero(r.reason == abi.R_OK):
            u = [int(x) for x in rng.integers(0, 3000, 2)]
            if rng.random() < 0.15:
                u = [int(rng.choice([-(1 << 63), (1 << 63) - 1, -5, 1 << 40])) for _ in range(2)]
            tot = wrap(u[0] + u[1]) if rng.random() < 0.9 else 0
            q = int(r.qos[i]) if rng.random() < 0.9 else -1  # ARKS_R_QOS_GONE
            resp.append((q, (u[0], u[1], tot), False))
            mrows.append((keys[q] if q >= 0 else None, (u[0], u[1], tot)))
            pre.append(int(est[i]) if seed >= 4 else 0)
        if resp:
            b = resp_batch(resp, now)
            if seed >= 4:
                b.precharged = np.array(pre, np.uint32)
            o.response_batch(b)
            model.response(mrows, now, np.array(pre) if seed >= 4 else None)
        # metered streams (N5): a prompt count and a chunk count per admitted row, given by the test
        adm = [int(x) for x in r.qos[r.reason == abi.R_OK]]
        if adm and rng.random() < 0.5:
            for side in (0, 1):
                cnt = [int(x) for x in rng.integers(0, 5000, len(adm))]
                o.meter(adm, cnt, side, now)
                model.meter([(keys[q], c) for q, c in zip(adm, cnt)], side, now)
        compare(o, model, t, now)
    assert n_cost_denials > 0 or seed % 2, seed


# ---- 3. table validation ----------------------------------------------------------------------------------------------------
def test_type_3_is_accepted_and_type_4_refused_on_both_routes():
    import hostmachine as hm
    from hostmachine import ConfigStore
    good = quickstart_cost([("prompt", 1), ("cost", 5)])
    assert hm.tables_shape_error(good.c_struct()) is None
    bad = quickstart_cost([("prompt", 1), ("cost", 5)])
    bad.qitem_type[1] = 4
    assert "unknown quota type" in hm.tables_shape_error(bad.c_struct())
    bad.qitem_type[1] = 3
    bad.rl_rule[0] = 4
    assert "unknown rate-limit rule" in hm.tables_shape_error(bad.c_struct())
    # the object store's flatten
    st = ConfigStore()
    st.upsert("quota", simple_quota("q", "ns", [("total", 1), ("cost", 2)]))
    assert hm.tables_shape_error(st.flatten().c_struct()) is None
    ty, val = np.array([2, 4], np.uint8), np.array([1, 2], np.int64)  # a type no ArksQuota spells: straight through the C call
    hm.lib().hm_store_upsert_quota(st.h, b"ns", 2, b"q4", 2, abi.ptr(ty, abi.u8p), abi.ptr(val, abi.i64p), 2)
    assert "unknown quota type" in hm.tables_shape_error(st.flatten().c_struct())
    # the oracle refuses type 4 as well
    with pytest.raises(ValueError):
        CostOracle(_with_type(good, 4))


def _with_type(t, ty):
    t = copy.deepcopy(t)
    t.qitem_type[-1] = ty
    return t


def test_prices_are_validated():
    assert endpoint_pricing(simple_endpoint("m", "ns")) == (0, 0)
    assert endpoint_pricing(simple_endpoint("m", "ns", pricing=(2500, 10000))) == (2500, 10000)
    for bad in ((-1, 0), (0, -7), (1.5, 0), ("3", 0), (True, 0), (0, 1 << 63)):
        with pytest.raises(ValueError):
            endpoint_pricing(simple_endpoint("m", "ns", pricing=bad))
    with pytest.raises(ValueError):
        endpoint_pricing({"metadata": {"name": "m"}, "spec": {"pricing": [1, 2]}})
    t = Tables([], [], [simple_endpoint("m", "ns", pricing=(1, 2)), simple_endpoint("m", "ns", pricing=(3, 4)),
                        simple_endpoint("n", "ns")])
    assert t.endpoint_price == {("ns", "m"): (1, 2)}  # the first object wins; unpriced endpoints are not listed


# ---- 4. the provider --------------------------------------------------------------------------------------------------------
class FakeGateway:
    """the config-plane methods the provider calls, recorded; counters and the sync from the cost oracle"""

    def __init__(self):
        self.calls, self.prices, self.tables, self.o = [], {}, None, None
        self.eps, self.quotas, self.tokens = {}, {}, {}

    def upsert_token(self, ns, name, token, qos):
        self.calls.append(("token", ns, name))

    def upsert_quota(self, ns, name, items):
        self.calls.append(("quota", ns, name, tuple(items)))

    def upsert_endpoint(self, ns, name, weights):
        self.calls.append(("endpoint", ns, name))

    def set_endpoint_price(self, ns, name, p, c):
        if p < 0 or c < 0:
            raise ValueError("negative price")
        self.calls.append(("price", ns, name, p, c))
        if (p, c) == (0, 0):
            self.prices.pop((ns, name), None)
        else:
            self.prices[(ns, name)] = (p, c)

    def delete_object(self, kind, ns, name):
        self.calls.append(("delete", kind, ns, name))

    def sync_quota_usage(self, present, used, restore=False):
        self.sync_shape = used.shape
        return self.o.sync_quota_usage(present, used, restore=restore)


def _ev(kind, obj, ty="ADDED"):
    o = copy.deepcopy(obj)
    o["kind"] = kind
    return {"type": ty, "object": o}


def test_provider_prices_endpoints_and_keeps_the_configuration_on_malformed_pricing():
    from arks_b200.provider import ArksProvider
    g = FakeGateway()
    p = ArksProvider(g, publish=lambda names: None)
    assert p.apply(_ev("ArksEndpoint", simple_endpoint("m", "ns", pricing=(2500, 10000))))
    assert g.prices == {("ns", "m"): (2500, 10000)}
    assert p.apply(_ev("ArksEndpoint", simple_endpoint("plain", "ns")))
    assert not [c for c in g.calls if c[0] == "price" and c[2] == "plain"]  # unpriced: no call
    # a price change alone is a change of what the request path reads
    assert p.apply(_ev("ArksEndpoint", simple_endpoint("m", "ns", pricing=(3000, 10000)), "MODIFIED"))
    assert g.prices == {("ns", "m"): (3000, 10000)}
    # malformed pricing: refused, the previous object and price stay
    for bad in ((-1, 5), (1.5, 2), ("x", 1)):
        n = len(g.calls)
        assert not p.apply(_ev("ArksEndpoint", simple_endpoint("m", "ns", pricing=bad), "MODIFIED"))
        assert len(g.calls) == n and p.rejected[-1][:2] == ("endpoint", ("ns", "m"))
    assert g.prices == {("ns", "m"): (3000, 10000)}
    assert p.objects["endpoint"][("ns", "m")]["spec"]["pricing"] == {"prompt": 3000, "completion": 10000}
    # the price removed from the spec, then the endpoint deleted
    assert p.apply(_ev("ArksEndpoint", simple_endpoint("m", "ns"), "MODIFIED"))
    assert g.prices == {}
    assert p.apply(_ev("ArksEndpoint", simple_endpoint("m", "ns", pricing=(1, 1)), "MODIFIED"))
    assert p.apply(_ev("ArksEndpoint", simple_endpoint("m", "ns"), "DELETED"))
    assert g.prices == {} and g.calls[-2:] == [("price", "ns", "m", 0, 0), ("delete", "endpoint", "ns", "m")]
    # a cost item in a quota goes through like the other types
    assert p.apply(_ev("ArksQuota", simple_quota("q", "ns", [("total", 5), ("cost", 7)])))
    assert g.calls[-1] == ("quota", "ns", "q", ((2, 5), (3, 7)))
    assert not p.apply(_ev("ArksQuota", simple_quota("q2", "ns", [("dollars", 5)])))


def test_provider_status_loop_writes_the_cost_entry_and_restores_it():
    from arks_b200.provider import ArksProvider
    t = quickstart_cost([("total", 10**9), ("cost", 10**9)])
    g = FakeGateway()
    g.o = CostOracle(t, {("default", "qwen-7b"): (2, 8)})
    g.tables = t
    clock = datetime.datetime(2026, 1, 2, 3, 4, 5, tzinfo=datetime.timezone.utc)
    p = ArksProvider(g, publish=lambda names: None, clock=lambda: clock)
    q = copy.deepcopy(FX["quotas"][0])
    q["spec"]["quotas"] = [{"type": "total", "value": 10**9}, {"type": "cost", "value": 10**9}]
    p.objects["quota"][("default", "basic-quota")] = q
    g.o.request_batch(req_batch([("sk-test123456", "qwen-7b", False)], NOW))
    g.o.response_batch(resp_batch([(0, (25, 20, 45), False)], NOW))
    out = p.sync_quota_status()
    assert g.sync_shape == (1, 4)
    assert out == [{"namespace": "default", "name": "basic-quota", "status": {"quotaStatus": [
        {"type": "total", "used": 45, "lastUpdateTime": "2026-01-02T03:04:05Z"},
        {"type": "cost", "used": 210, "lastUpdateTime": "2026-01-02T03:04:05Z"}]}}]
    # restart: the counters are gone, restore-on-start raises them to the CR, the cost key included
    g.o = CostOracle(t, {("default", "qwen-7b"): (2, 8)})
    assert p.sync_quota_status(restore=True) == []
    assert g.o.snapshot_quota_cost().tolist() == [210] and g.o.snapshot_quota().tolist() == [[0, 0, 45]]
    # reference mode: a store behind the CR is zeroed, every item of the quota (the cost key too)
    g.o.response_batch(resp_batch([(0, (1, 1, 2), False)], NOW))
    q["status"]["quotaStatus"][1]["used"] = 10**6
    p.sync_quota_status()
    assert g.o.snapshot_quota_cost().tolist() == [0] and g.o.snapshot_quota().tolist() == [[0, 0, 0]]


# ---- 5. the shapers ---------------------------------------------------------------------------------------------------------
def _in_subprocess(fn):
    code = f"import sys; sys.path[:0] = [{HERE!r}, {ROOT!r}]; import test_cost_quota as T; T.{fn}()"
    subprocess.check_call([sys.executable, "-c", code], cwd=ROOT)


def test_cpp_and_python_shapers_agree_on_a_cost_denial():
    _in_subprocess("check_shapers_agree")


def check_shapers_agree():
    from test_cpp_host import CpuEngine
    plain = Tables([simple_token("alice", "team-a", "sk-x", "qwen-7b", [("rpm", 5)], "q-main")],
                   [simple_quota("q-main", "team-a", [("prompt", 100), ("total", 600)])], [simple_endpoint("qwen-7b", "team-a")])
    t = Tables([simple_token("alice", "team-a", "sk-x", "qwen-7b", [("rpm", 5)], "q-main")],
               [simple_quota("q-main", "team-a", [("prompt", 100), ("cost", 2500), ("total", 600)])],
               [simple_endpoint("qwen-7b", "team-a", pricing=(2, 8))])
    eng = CpuEngine(plain, max_batch=16, max_bytes=1 << 16)  # the shim's oracle has no cost items: the names carry them
    try:
        eng.b.set_names(t)
        body = b'{"model":"qwen-7b","messages":[]}'
        k = body.find(b'"model":"') + 9
        for detail, cur, lim in ((1, 2501, 2500), (1, 9 * 10**18, 2500), (0, 101, 100), (2, 601, 600)):
            d = cpphost.RequestDecision()
            d.reason, d.detail, d.cur_usage, d.limit_max, d.now_unix, d.qos = abi.R_QUOTA, detail, cur, lim, NOW, 0
            d.model_off, d.model_len = k, 7
            got = eng.b.request_error_reply(d, b"sk-x", body)
            want = replies.request_error_reply(abi.R_QUOTA, detail, cur, lim, NOW, t, 0, b"sk-x", "qwen-7b")
            assert got == want, (got, want)
            ty = ["prompt", "cost", "total"][detail]
            assert want[0] == 429 and want[1] == "x-error-quota"
            assert '{"Key":"type","Value":"%s"}' % ty in want[3] and '"currentUsage":%d' % cur in want[3]
    finally:
        eng.close()


# ---- GPU ----------------------------------------------------------------------------------------------------------------------
def priced_objects(w, seed, cost_lo=0, cost_hi=4000, cost_frac=0.3, unpriced_frac=0.1):
    """workload `w`'s objects with price policies: each quota gets a mix of cost-only, cost + total or all four items (some with
    a tight cost limit), each tenant endpoint its own prices (a few unpriced)"""
    rng = np.random.default_rng(seed)
    tokens, quotas, endpoints = copy.deepcopy(w.objects)
    prices = {}
    for t, (q, e) in enumerate(zip(quotas, endpoints)):
        tight = rng.random() < cost_frac
        lim = int(rng.integers(cost_lo, cost_hi)) if tight else int(rng.integers(10**9, 10**12))
        items = q["spec"]["quotas"]
        mix = t % 3
        if mix == 0:
            q["spec"]["quotas"] = [{"type": "cost", "value": lim}]
        elif mix == 1:
            q["spec"]["quotas"] = [{"type": "cost", "value": lim}, items[2]]
        else:
            q["spec"]["quotas"] = items[:2] + [{"type": "cost", "value": lim}, items[2]]
        if rng.random() >= unpriced_frac:
            p = (int(rng.integers(0, 50)), int(rng.integers(0, 200)))
            e["spec"]["pricing"] = {"prompt": p[0], "completion": p[1]}
            prices[(e["metadata"]["namespace"], e["metadata"]["name"])] = p
    return tokens, quotas, endpoints, prices


def same(a, b, what):
    for k, v in a.fields().items():
        assert np.array_equal(v, b.fields()[k]), (what, k)


def same_state(g, o, now, what):
    assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), what
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), what
    assert np.array_equal(g.snapshot_quota_cost(), o.snapshot_quota_cost()), what


@pytest.mark.gpu
@pytest.mark.parametrize("sse", [False, True], ids=["json", "sse"])
def test_gpu_every_scan_path_with_cost_items(gwmod, sse):
    w = traffic.Workload(n_tenants=1500, seed=41, zipf_alpha=1.1)
    tokens, quotas, endpoints, prices = priced_objects(w, 5)
    t = Tables(tokens, quotas, endpoints)
    g = gwmod.Gateway(0, 16384, 64 << 20)
    g.load_tables(t)
    o = CostOracle(t, prices)
    now = NOW
    cost_first = 0
    for step, n in enumerate((300, 2048, 2049, 4095, 4096, 12000, 2048, 300)):
        now += 1
        req = w.request_batch(n, now, seed=100 + step, stream_frac=0.5 if sse else 0.0, n_templates=64)
        a, b = g.handle_request_body(req), o.request_batch(req)
        same(a, b, ("request", n))
        for i in np.flatnonzero(a.reason == abi.R_QUOTA):
            qt = int(t.qos_quota[a.qos[i]])
            cost_first += int(t.qitem_type[t.quota_item_off[qt] + a.detail[i]]) == abi.QT_COST
        resp = w.response_batch(a, now, seed=200 + step, noise_frac=0.02)
        c, d = g.handle_response_body(resp), o.response_batch(resp)
        same(c, d, ("response", n))
        same_state(g, o, now, n)
    assert cost_first > 0


@pytest.mark.gpu
def test_gpu_hot_tenant_with_cost_items(gwmod):
    """one tenant with more than kHotGroup (256) arrivals in a batch: rank_hot_groups_kernel ranks it"""
    w = traffic.Workload(n_tenants=200, seed=3, zipf_alpha=2.0)
    tokens, quotas, endpoints, prices = priced_objects(w, 9, cost_frac=0.5, cost_lo=0, cost_hi=100)
    t = Tables(tokens, quotas, endpoints)
    g = gwmod.Gateway(0, 16384, 64 << 20)
    g.load_tables(t)
    o = CostOracle(t, prices)
    for step, n in enumerate((8192, 1500, 8192)):
        req = w.request_batch(n, NOW + step, seed=7 + step, n_templates=32)
        a, b = g.handle_request_body(req), o.request_batch(req)
        same(a, b, ("request", step))
        assert np.bincount(a.qos[a.qos >= 0]).max() > 256
        resp = w.response_batch(a, NOW + step, seed=17 + step)
        same(g.handle_response_body(resp), o.response_batch(resp), ("response", step))
        same_state(g, o, NOW + step, step)


@pytest.mark.gpu
def test_gpu_config4_with_price_policies_at_full_size(gwmod):
    w = traffic.Workload(n_tenants=100_000, seed=0xC4, zipf_alpha=1.1)
    tokens, quotas, endpoints, prices = priced_objects(w, 44, cost_frac=0.2, cost_hi=3000)
    t = Tables(tokens, quotas, endpoints)
    assert t.n_quotas == 100_000 and len(set(prices.values())) > 1000
    g = gwmod.Gateway(0, 65536, 96 << 20)
    g.load_tables(t)
    o = CostOracle(t, prices)
    cost_first = 0
    for step in range(3):
        now = NOW + 7 * step
        req = w.request_batch(32768, now, seed=300 + step, n_templates=256)
        a, b = g.handle_request_body(req), o.request_batch(req)
        same(a, b, ("request", step))
        for i in np.flatnonzero(a.reason == abi.R_QUOTA):
            qt = int(t.qos_quota[a.qos[i]])
            cost_first += int(t.qitem_type[t.quota_item_off[qt] + a.detail[i]]) == abi.QT_COST
        resp = w.response_batch(a, now, seed=400 + step, varied=True, n_templates=256)
        same(g.handle_response_body(resp), o.response_batch(resp), ("response", step))
        same_state(g, o, now, step)
    assert cost_first > 100


@pytest.mark.gpu
def test_gpu_generation_swap_carries_cost_and_applies_new_prices(gwmod):
    price = {("default", "qwen-7b"): (2, 8)}
    llama = {"arksEndpoint": {"name": "llama"}, "rateLimits": [], "quota": {"name": "basic-quota"}}
    tok = copy.deepcopy(FX["tokens"][0])
    tok["spec"]["qos"].append(llama)
    q = [simple_quota("basic-quota", "default", [("total", 10**9), ("cost", 10**9)]), simple_quota("other", "default", [("cost", 1)])]
    eps = FX["endpoints"] + [simple_endpoint("llama", "default", pricing=(100, 100))]
    t = Tables([tok], q, eps)
    assert t.endpoint_price == {("default", "llama"): (100, 100)}
    g = gwmod.Gateway(0, 1024, 1 << 20)
    g.set_endpoint_price("default", "qwen-7b", 2, 8)
    g.load_tables(t)  # also pushes llama's spec.pricing
    o = CostOracle(t, {**price, ("default", "llama"): (100, 100)})
    a = g.handle_request_body(req_batch([("sk-test123456", "qwen-7b", False)], NOW))
    gen0 = g.generation
    rows = [(0, (25, 20, 45), False), (1, (1, 1, 2), False)]
    g.handle_response_body(resp_batch(rows, NOW))
    o.response_batch(resp_batch(rows, NOW))
    assert g.snapshot_quota_cost().tolist() == [210 + 200, 0]
    # a price change: nothing until the next generation
    g.set_endpoint_price("default", "qwen-7b", 3, 5)
    g.handle_response_body(resp_batch([(0, (1, 1, 2), False)], NOW))
    o.response_batch(resp_batch([(0, (1, 1, 2), False)], NOW))
    assert g.snapshot_quota_cost().tolist() == [420, 0]
    # next generation: the quotas in another order, llama's endpoint deleted; cost carried by key
    t2 = Tables([tok], q[::-1], FX["endpoints"])
    g.load_tables(t2)
    o.set_price("default", "qwen-7b", 3, 5)
    o.reload(t2)
    assert g.snapshot_quota_cost().tolist() == [0, 420]
    # an old-generation row is billed at the current prices; the deleted endpoint bills 0
    b = resp_batch([(0, (10, 10, 20), False), (1, (10, 10, 20), False)], NOW + 1)
    b.gen = np.array([gen0, g.generation], np.uint32)
    r = g.handle_response_body(b)
    assert r.reason.tolist() == [abi.R_OK, abi.R_OK]
    o.response_batch(resp_batch([(0, (10, 10, 20), False), (1, (10, 10, 20), False)], NOW + 1))
    assert g.snapshot_quota_cost().tolist() == [0, 420 + 80]
    assert np.array_equal(g.snapshot_quota_cost(), o.snapshot_quota_cost())
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota())
    # a qos entry that is gone bills nothing
    t3 = Tables([simple_token("x", "default", "sk-x", "qwen-7b", [])], q, FX["endpoints"])
    g.load_tables(t3)
    b = resp_batch([(0, (10, 10, 20), False)], NOW + 2)
    b.gen = np.array([gen0], np.uint32)
    assert g.handle_response_body(b).reason.tolist() == [abi.R_QOS_GONE]
    assert g.snapshot_quota_cost().tolist() == [500, 0]  # t3 lists the quotas in the first order again
    assert a.reason[0] == abi.R_OK


@pytest.mark.gpu
def test_gpu_stream_metering_bills_cost_and_precharge_leaves_it(gwmod):
    from arks_b200 import bpe
    tok, text = bpe.standin_tokenizer(20_000, cache_dir=BUILD)
    w = traffic.Workload(n_tenants=300, seed=23)
    tokens, quotas, endpoints, prices = priced_objects(w, 2, cost_frac=0.0)
    t = Tables(tokens, quotas, endpoints)
    g = gwmod.Gateway(0, 65536, 96 << 20)
    g.load_tables(t)
    g.load_bpe(bpe.load_tokenizer(text))
    price = np.zeros((t.n_qos, 2), np.int64)
    for qi, (ns, _, m) in enumerate(qos_keys(t)):
        price[qi] = prices.get((ns, m), (0, 0))
    ncost = np.array([int(np.sum(t.qitem_type[t.quota_item_off[q]:t.quota_item_off[q + 1]] == abi.QT_COST))
                      for q in range(t.n_quotas)])
    want = np.zeros(t.n_quotas, np.int64)

    def charge(qos, counts, side):
        for q, c in zip(qos, counts):
            qt = int(t.qos_quota[q])
            if qt >= 0:
                want[qt] = wrap(int(want[qt]) + int(c) * int(price[q, side]) * int(ncost[qt]))

    # the pre-charge alone: the cost column does not move at request time
    g.set_precharge(True)
    a = g.handle_request_body(w.request_batch(2000, NOW, seed=1))
    assert np.all(g.snapshot_quota_cost() == 0)
    g.set_precharge(False)
    # metered streams: the prompt's count at p_prompt, every chunk's at p_completion (body length when uncounted)
    g.set_stream_metering(True)
    for step, n in enumerate((700, 3000, 9000)):
        now = NOW + 1 + step
        req = w.request_batch(n, now, seed=40 + step, stream_frac=0.6)
        bodies = [bytes(req.bodies[req.body_off[i]:req.body_off[i] + req.body_len[i]]).replace(
            b',"stream_options":{"include_usage":true}', b"") if i % 2 else
            bytes(req.bodies[req.body_off[i]:req.body_off[i] + req.body_len[i]]) for i in range(req.n)]
        toks = [bytes(req.tokens[req.token_off[i]:req.token_off[i + 1]]) for i in range(req.n)]
        req = RequestBatch.from_lists(bodies, toks, now, pick_rand=req.pick_rand)
        a = g.handle_request_body(req)
        met = np.flatnonzero((a.flags & abi.FLAG_METERED) != 0)
        assert len(met) > 0.1 * n
        cnt = np.where(a.bpe_count[met] == 0xFFFFFFFF, req.body_len[met], a.bpe_count[met])
        charge(a.qos[met], cnt, 0)
        resp = w.response_batch(a, now, seed=70 + step)
        owner = np.repeat(np.flatnonzero(a.reason == abi.R_OK), np.where(a.flags[a.reason == abi.R_OK] & 1, 4, 1))
        flags = [int(f) | (abi.RESP_METERED if a.flags[owner[k]] & abi.FLAG_METERED else 0) for k, f in enumerate(resp.flags)]
        resp.flags = np.array(flags, np.uint8)
        c = g.handle_response_body(resp)
        mk = np.flatnonzero((resp.flags & (abi.RESP_STREAM | abi.RESP_METERED)) == (abi.RESP_STREAM | abi.RESP_METERED))
        mk = mk[c.reason[mk] == abi.R_OK]
        cnt = np.where(c.bpe_count[mk] == 0xFFFFFFFF, resp.body_len[mk], c.bpe_count[mk])
        charge(resp.qos[mk], cnt, 1)
        # the rows that are not metered are billed as counted responses
        cnt_rows = np.flatnonzero(c.counted == 1)
        for k in cnt_rows:
            q = int(resp.qos[k])
            qt = int(t.qos_quota[q])
            if qt >= 0:
                u = c.usage[k]
                want[qt] = wrap(int(want[qt]) + (int(u[0]) * int(price[q, 0]) + int(u[1]) * int(price[q, 1])) * int(ncost[qt]))
        assert np.array_equal(g.snapshot_quota_cost(), want), step
    assert want.any()


@pytest.mark.gpu
def test_gpu_quota_sharing_is_refused_in_both_orders(gwmod):
    t = quickstart_cost([("total", 5), ("cost", 5)])
    g = gwmod.Gateway(0, 1024, 1 << 20, share_quota=True)
    with pytest.raises(gwmod.ArksError, match="cost"):
        g.load_tables(t)
    g.load_tables(quickstart_cost([("total", 5)]))  # without a cost item sharing works as before
    g2 = gwmod.Gateway(0, 1024, 1 << 20)
    g2.load_tables(t)
    with pytest.raises(gwmod.ArksError, match="cost"):
        g2._ck(gwmod.lib().arks_enable_quota_sharing(g2._h, 1))


@pytest.mark.gpu
@pytest.mark.parametrize("restore", [False, True])
def test_gpu_sync_in_four_and_three_columns(gwmod, restore):
    w = traffic.Workload(n_tenants=2000, seed=8)
    tokens, quotas, endpoints, prices = priced_objects(w, 3)
    t = Tables(tokens, quotas, endpoints)
    rng = np.random.default_rng(int(restore))
    for cols in (4, 3):
        g = gwmod.Gateway(0, 8192, 32 << 20)
        g.load_tables(t)
        o = CostOracle(t, prices)
        req = w.request_batch(6000, NOW, seed=1, n_templates=64)
        a, b = g.handle_request_body(req), o.request_batch(req)
        resp = w.response_batch(a, NOW, seed=2)
        g.handle_response_body(resp)
        o.response_batch(resp)
        n = t.n_quotas
        present = rng.integers(0, 16 if cols == 4 else 8, n).astype(np.uint32)
        cur = np.concatenate([g.snapshot_quota(), g.snapshot_quota_cost()[:, None]], axis=1)[:, :cols]
        used = (cur + rng.integers(-3000, 3000, (n, cols)) * (rng.random((n, cols)) < 0.5)).astype(np.int64)
        p1, u1, p2, u2 = present.copy(), used.copy(), present.copy(), used.copy()
        cost_before = g.snapshot_quota_cost()
        act_g = g.sync_quota_usage(p1, u1, restore=restore)
        act_o = o.sync_quota_usage(p2, u2, restore=restore)
        assert np.array_equal(act_g, act_o) and np.array_equal(p1, p2) and np.array_equal(u1, u2), cols
        assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), cols
        assert np.array_equal(g.snapshot_quota_cost(), o.snapshot_quota_cost()), cols
        assert (act_g & 2).any()
        if cols == 3:  # the three-column call leaves the cost column alone
            assert np.array_equal(g.snapshot_quota_cost(), cost_before) and cost_before.any()


@pytest.mark.gpu
def test_gpu_cost_items_add_no_launch(gwmod):
    w = traffic.Workload(n_tenants=500, seed=12)
    tokens, quotas, endpoints, prices = priced_objects(w, 4)
    deltas = []
    for t in (w.tables, Tables(tokens, quotas, endpoints)):
        g = gwmod.Gateway(0, 16384, 64 << 20)
        g.load_tables(t)
        d = []
        for n in (500, 3000, 9000):
            req = w.request_batch(n, NOW, seed=n, stream_frac=0.3, n_templates=32)
            before = g.launch_count
            a = g.handle_request_body(req)
            d.append(g.launch_count - before)
            resp = w.response_batch(a, NOW, seed=n + 1)
            before = g.launch_count
            g.handle_response_body(resp)
            d.append(g.launch_count - before)
        before = g.launch_count
        g.load_tables(t)
        d.append(g.launch_count - before)
        deltas.append(d)
    assert deltas[0] == deltas[1]
