"""Admission (limit_admit_kernel, rank_hot_groups_kernel) and the generation history at their fixed capacities.

kHotGroup = 256: a qos entry with up to 256 arrivals in a batch is ranked by walking its member list, from 257 on it is
listed in hot_list and ranked by a block sweep over the batch in int4 tiles. The tests put a tenant at exactly 255, 256,
257 and 258 arrivals, several hot tenants with different `k` in one batch (duplicated rules whose room is not a multiple
of their count, k = 0 by tpm, by quota and by a missing ArksQuota, k >= n), at batch sizes on the warp path, the exact
engine alone and the fast path, with sizes that are not multiples of 4 or 1 024 and hot members at the first and last row.

Two referees, neither of them the device: the oracle (orklib), and SerialLimiter below — a dict of counters, requests
applied in index order, the first over-limit entry of the list denies, every request-type entry +1 on admit — so that
the closed form `k = min_j max(0, (limit_j - cur_j - 1) / cnt_j + 1)` and the hot-group ranks are checked against
something that is not ork_core.c.

ARKS_GEN_HISTORY = 16: a response row carrying a generation at most 16 publications old is re-mapped to the current
index of its (namespace, user, model) key and billed there; the 17th publication makes it ARKS_R_QOS_GONE."""
import numpy as np
import pytest

import orklib
from arks_b200 import abi
from arks_b200.abi import RequestBatch, ResponseBatch
from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token

pytestmark = pytest.mark.gpu
NOW = 1_700_000_040  # second 0 of a minute: now + 59 is the same rpm window, now + 60 the next
assert NOW % 60 == 0
HOT_GROUP = 256       # arks_gateway.cu kHotGroup
I64_MAX = 2**63 - 1
WINDOW = {"rpm": 60, "rpd": 86400, "tpm": 60, "tpd": 86400}


class SerialLimiter:
    """the limiter one request at a time. tenants: {bearer token: (limits [(rule, value)], quota)}; quota is None (no
    quota), "missing" (the ArksQuota does not exist) or (items [(type, value)], used {type: int})"""

    def __init__(self, tenants):
        self.tenants = tenants
        self.cur = {}  # (token, rule) -> (window start, value)

    def value(self, tok, rule, now):
        w, v = self.cur.get((tok, rule), (0, 0))
        return v if w == now - now % WINDOW[rule] else 0

    def request(self, tok, now):
        """-> (reason, detail, current usage, limit)"""
        limits, quota = self.tenants[tok]
        for j, (rule, lim) in enumerate(limits):
            c = self.value(tok, rule, now)
            if c + (1 if rule[0] == "r" else 0) > lim:
                return abi.R_RATE_LIMIT, j, c, lim
        if quota == "missing":
            return abi.R_QUOTA_CONFIG, 0, 0, 0
        if quota is not None:
            for j, (ty, lim) in enumerate(quota[0]):
                if quota[1].get(ty, 0) > lim:
                    return abi.R_QUOTA, j, quota[1].get(ty, 0), lim
        for rule, _ in limits:
            if rule[0] == "r":
                self.cur[(tok, rule)] = (now - now % WINDOW[rule], self.value(tok, rule, now) + 1)
        return 0, 0, 0, 0

    def batch(self, toks, now):
        return [self.request(t, now) for t in toks]


def make(gwmod, tenants, max_batch=8192):
    """tenants as for SerialLimiter -> (gateway, oracle, serial limiter); every tenant reads model "m" """
    toks, quotas = [], []
    for i, (tok, (limits, quota)) in enumerate(tenants.items()):
        qn = "" if quota is None else "absent" if quota == "missing" else "q%d" % i
        toks.append(simple_token("u%d" % i, "ns", tok.decode(), "m", limits, qn))
        if isinstance(quota, tuple):
            quotas.append(simple_quota(qn, "ns", quota[0]))
    t = Tables(toks, quotas, [simple_endpoint("m", "ns")])
    g = gwmod.Gateway(0, max_batch, 16 << 20)
    g.load_tables(t)
    o = orklib.Oracle(t)
    qi = 0
    for tok, (limits, quota) in tenants.items():  # quota usage that is already there
        if isinstance(quota, tuple):
            used = [quota[1].get(k, 0) for k in ("prompt", "response", "total")]
            g.set_quota_usage(qi, used); o.set_quota_usage(qi, used)
            qi += 1
    return g, o, SerialLimiter(tenants)


def submit(g, o, s, toks, now, ctx):
    req = RequestBatch.from_lists([b'{"model":"m"}'] * len(toks), list(toks), now)
    a = g.handle_request_body(req)
    b = o.request_batch(req)
    for k, v in a.fields().items():
        w = b.fields()[k]
        if not np.array_equal(v, w):
            bad = np.flatnonzero(v != w)
            raise AssertionError(f"{ctx} field {k}: {len(bad)} rows differ from the oracle, first {bad[:5]}: gpu={v[bad[:5]]} oracle={w[bad[:5]]}")
    assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), ctx + ": rate counters differ"
    want = s.batch(toks, now)
    got = list(zip(a.reason.tolist(), a.detail.tolist(), a.cur_usage.tolist(), a.limit_max.tolist()))
    bad = [i for i in range(len(toks)) if got[i] != want[i]]
    assert not bad, (ctx, len(bad), [(i, toks[i], got[i], want[i]) for i in bad[:5]])
    return a


def mixed_order(groups, n, seed, order):
    """`groups`: {token: arrivals}; the rest of the n rows are spread over cold tenants tk-c0 .. tk-c7"""
    toks = [t for t, k in groups.items() for _ in range(k)]
    toks += [b"tk-c%d" % (i % 8) for i in range(n - len(toks))]
    assert len(toks) == n
    if order == "shuffled":
        return [toks[i] for i in np.random.default_rng(seed).permutation(n)]
    return toks  # sorted: the first group owns the first rows; the caller puts a hot one last too


COLD = {b"tk-c%d" % i: ([("rpm", 10**9)], None) for i in range(8)}
# the warp path, the exact engine alone, the fast path; 1 025 / 1 027 / 4 099: tile tails of rank_hot_groups_kernel
SIZES = [1025, 1027, 2048, 2500, 4096, 4099]


@pytest.mark.parametrize("arrivals", [HOT_GROUP - 1, HOT_GROUP, HOT_GROUP + 1, HOT_GROUP + 2])
def test_kHotGroup_256_arrivals_of_one_tenant(gwmod, arrivals):
    """kHotGroup: 255 and 256 arrivals are ranked by the member-list walk, 257 and 258 by rank_hot_groups_kernel; an rpm
    limit that admits 1, 255, 256, 257 of them, all of them, none of them. Exactly the first `limit` arrivals in batch order
    are admitted, the others get detail 0, currentUsage = limit, limitMax = limit."""
    for limit in (1, HOT_GROUP - 1, HOT_GROUP, HOT_GROUP + 1, 10**6, 0, I64_MAX):
        tenants = dict(COLD)
        tenants[b"tk-hot"] = ([("rpm", limit)], None)
        g, o, s = make(gwmod, tenants)
        now = NOW
        for n, order in ((arrivals, "sorted"), (1027, "shuffled"), (2500, "shuffled"), (4099, "shuffled"), (4099, "sorted")):
            toks = mixed_order({b"tk-hot": arrivals}, n, 11, order)
            if order == "sorted" and n > arrivals:  # hot members at the first AND the last index of the batch
                toks[1], toks[-1] = toks[-1], toks[1]
            a = submit(g, o, s, toks, now, f"arrivals={arrivals} limit={limit} n={n} {order}")
            hot = np.array([t == b"tk-hot" for t in toks])
            assert int((a.reason[hot] == 0).sum()) == min(arrivals, limit)
            assert np.all(a.reason[~hot] == 0)
            first = np.flatnonzero(hot)[:min(arrivals, limit)]
            assert np.all(a.reason[first] == 0)  # in arrival order
            now += 60


def hot_tenants():
    t = dict(COLD)
    t[b"tk-a"] = ([("rpm", 300), ("tpm", 10**9), ("rpd", 10**6)], None)
    t[b"tk-dup"] = ([("rpm", 9 + 600), ("rpm", 5 + 600), ("rpd", 10**5)], None)     # room not a multiple of cnt = 2
    t[b"tk-tpm"] = ([("rpm", 10**6), ("tpm", -1)], None)                            # 0 > -1: k = 0 by a token rule
    t[b"tk-quota"] = ([("rpm", 10**6)], ([("prompt", 10**6), ("total", 50)], {"total": 51}))  # k = 0 by quota item 1
    t[b"tk-noq"] = ([("rpm", 10**6)], "missing")                                    # k = 0: ArksQuota missing
    t[b"tk-all"] = ([("rpm", 10**6), ("rpd", 10**7)], None)                         # k >= n
    return t


@pytest.mark.parametrize("n", SIZES)
def test_several_hot_groups_with_different_k(gwmod, n):
    """several groups beyond kHotGroup in one batch, each with its own k: duplicated rules (`room / cnt` not whole), k = 0
    by an over-limit tpm, by quota and by a missing ArksQuota, k >= n_g; shuffled by a seeded permutation and sorted with a
    hot tenant on the first and on the last rows; the same batch again in the same window (cur != 0) and after the
    minute rolls over."""
    g, o, s = make(gwmod, hot_tenants())
    per = max(HOT_GROUP + 1, min(700, n // 7))
    groups = {b"tk-dup": per, b"tk-tpm": HOT_GROUP + 1, b"tk-quota": HOT_GROUP + 2, b"tk-noq": HOT_GROUP + 1}
    if n > 2000:
        groups.update({b"tk-a": per + 3, b"tk-all": per})
    else:
        groups[b"tk-noq"] = 100  # four groups of 257 do not fit 1 025 rows: this one is ranked by its member list
    for order in ("shuffled", "sorted"):
        toks = mixed_order(groups, n, n, order)
        if order == "sorted":
            toks = toks[groups[b"tk-dup"]:] + toks[:groups[b"tk-dup"]]  # tk-tpm first ... cold ... tk-dup last
        now = NOW + (0 if order == "shuffled" else 7200)
        submit(g, o, s, toks, now, f"n={n} {order} first")
        submit(g, o, s, toks, now + 59, f"n={n} {order} same window")
        submit(g, o, s, toks, now + 60, f"n={n} {order} next minute")


def test_limits_0_1_int64_max_and_a_negative_tpm_counter(gwmod):
    """limits 0, 1 and 2^63 - 1 on a hot group; a tpm counter driven negative by a usage of INT64_MIN (gjson's int64(f) of
    an out-of-range float) and the request batch that follows it: cur + 0 > limit is false for every limit >= 0."""
    tenants = dict(COLD)
    tenants[b"tk-0"] = ([("rpm", 0)], None)
    tenants[b"tk-1"] = ([("rpd", 1), ("rpm", 5)], None)
    tenants[b"tk-max"] = ([("rpm", I64_MAX), ("rpd", I64_MAX)], None)
    tenants[b"tk-neg"] = ([("tpm", 0), ("rpm", 300)], None)
    g, o, s = make(gwmod, tenants)
    groups = {b"tk-0": 300, b"tk-1": 300, b"tk-max": 300, b"tk-neg": 400}
    toks = mixed_order(groups, 2500, 5, "shuffled")
    submit(g, o, s, toks, NOW, "limits first")
    submit(g, o, s, toks, NOW + 1, "limits second")
    qos_neg = list(tenants).index(b"tk-neg")
    resp = ResponseBatch.from_lists([b'{"model":"m","usage":{"prompt_tokens":1,"completion_tokens":1,"total_tokens":1e30}}'],
                                    [qos_neg], [abi.RESP_END_OF_STREAM], NOW + 120)
    c, d = g.handle_response_body(resp), o.response_batch(resp)
    assert np.array_equal(c.usage, d.usage) and c.usage[0, 2] == -2**63
    assert np.array_equal(g.snapshot_rate(NOW + 120), o.snapshot_rate(NOW + 120))
    assert g.snapshot_rate(NOW + 120)[qos_neg].min() == -2**63
    a = submit(g, o, s, toks, NOW + 121, "after the negative counter")
    assert int((a.reason[np.array([t == b"tk-neg" for t in toks])] == 0).sum()) == 300


@pytest.mark.parametrize("publications", [15, 16, 17])
def test_ARKS_GEN_HISTORY_16_publications(gwmod, publications):
    """ARKS_GEN_HISTORY: a stream admitted at generation g, then 15 / 16 / 17 table publications that each shift the qos
    indices, then its response with gen = g. resolve_qos walks `current - g` re-maps and 16 are kept: 15 and 16 bill the
    same (namespace, user, model) key at its current index, 17 is ARKS_R_QOS_GONE and no counter moves."""
    def tables(k):  # k tenants sorted in front of "zz-user": its qos index moves by one with every publication
        toks = [simple_token("aa%02d" % i, "ns", "tk-aa%02d" % i, "m", [("rpm", 10**6)]) for i in range(k)]
        toks.append(simple_token("zz-user", "ns", "tk-zz", "m", [("rpm", 10**6), ("tpm", 10**9)]))
        return Tables(toks, [], [simple_endpoint("m", "ns")])
    g = gwmod.Gateway(0, 64, 1 << 20)
    g.load_tables(tables(0))
    a = g.handle_request_body(RequestBatch.from_lists([b'{"model":"m"}'], [b"tk-zz"], NOW))
    assert a.reason[0] == 0
    q0, g0 = int(a.qos[0]), g.generation
    for k in range(1, publications + 1):
        g.load_tables(tables(k))
    o = orklib.Oracle(tables(publications))
    a = g.handle_request_body(RequestBatch.from_lists([b'{"model":"m"}'], [b"tk-zz"], NOW + 1))
    q_now = int(a.qos[0])
    assert q_now != q0 and g.generation == g0 + publications
    before = g.snapshot_rate(NOW + 1).copy()
    body = b'{"model":"m","usage":{"prompt_tokens":3,"completion_tokens":4,"total_tokens":7}}'
    c = g.handle_response_body(ResponseBatch.from_lists([body], [q0], [abi.RESP_END_OF_STREAM], NOW + 2, gen=[g0]))
    after = g.snapshot_rate(NOW + 2)
    if publications <= abi.GEN_HISTORY:
        d = o.response_batch(ResponseBatch.from_lists([body], [q_now], [abi.RESP_END_OF_STREAM], NOW + 2))
        assert c.reason[0] == d.reason[0] != abi.R_QOS_GONE and tuple(c.usage[0]) == (3, 4, 7) and c.counted[0]
        moved = np.argwhere(after != before)
        assert moved.size and set(moved[:, 0].tolist()) == {q_now} and (after - before)[q_now].max() == 7
    else:
        assert c.reason[0] == abi.R_QOS_GONE and not c.counted[0]
        assert np.array_equal(after, before)
