"""Randomised parity soak on a GPU box: ROUNDS rounds of mixed traffic (client-application requests, three completion
dialects, SSE chunks, fuzzed documents, malformed / unauthorised requests, window roll-overs, table reloads) through the
C ABI, every decision and every counter compared with the oracle. Usage: python tests/harness/gpu_soak.py [rounds] [seed]"""
import sys
import numpy as np
import os
_R = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, _R); sys.path.insert(0, os.path.join(_R, "tests"))
import __graft_entry__ as ge; ge.build()
import orklib
from jsonfuzz import Gen
from arks_b200 import abi, traffic
from arks_b200.abi import RequestBatch, ResponseBatch
from arks_b200.gateway import Gateway

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 20
seed = int(sys.argv[2]) if len(sys.argv) > 2 else 1
rng = np.random.default_rng(seed)
w = traffic.Workload(n_tenants=400, seed=seed)
g = Gateway(0, 16384, 48 << 20); g.load_tables(w.tables); g.enable_metrics(True)
o = orklib.Oracle(w.tables)
gen = Gen(seed)
now = 1_700_000_000
def same(a, b, what):
    for k, v in a.fields().items():
        assert np.array_equal(v, b.fields()[k]), (what, k, np.flatnonzero(np.any(np.atleast_2d((v != b.fields()[k]).reshape(len(v), -1)), axis=1))[:5] if v.ndim > 1 else np.flatnonzero(v != b.fields()[k])[:5])
n_req = n_resp = 0
for r in range(rounds):
    n = int(rng.choice([37, 700, 5000, 16000]))
    req = w.request_batch(n, now, seed=int(rng.integers(1 << 30)), stream_frac=float(rng.random()) * 0.6, noise_frac=0.12,
                          varied=bool(rng.random() < 0.7), n_templates=0 if n < 6000 else 3000)
    if rng.random() < 0.5:  # splice fuzzed documents in
        bodies = [bytes(req.bodies[req.body_off[i]:req.body_off[i] + req.body_len[i]]) for i in range(req.n)]
        toks = [bytes(req.tokens[req.token_off[i]:req.token_off[i + 1]]) for i in range(req.n)]
        for i in rng.integers(0, req.n, req.n // 10):
            bodies[int(i)] = gen.request()
        req = RequestBatch.from_lists(bodies, toks, now, pick_rand=req.pick_rand)
    a, b = g.handle_request_body(req), o.request_batch(req)
    same(a, b, f"round {r} request")
    n_req += req.n
    resp = w.response_batch(a, now + 1, seed=int(rng.integers(1 << 30)), noise_frac=0.1, varied=bool(rng.random() < 0.7))
    if resp.n:
        bodies = [bytes(resp.bodies[resp.body_off[i]:resp.body_off[i] + resp.body_len[i]]) for i in range(resp.n)]
        fl = resp.flags.copy()
        for i in rng.integers(0, resp.n, resp.n // 10):
            i = int(i)
            bodies[i] = gen.sse_chunk() if fl[i] & abi.RESP_STREAM else gen.response()
        fl = np.where(fl & abi.RESP_STREAM, fl | rng.choice([0, 2, 4, 6], resp.n).astype(np.uint8), fl)
        kinds = [None] if rng.random() < 0.4 else [0, 1]     # mixed batch, or split into JSON-only / SSE-only batches
        for kind in kinds:
            sel = np.arange(resp.n) if kind is None else np.flatnonzero(((fl & abi.RESP_STREAM) != 0) == bool(kind))
            for lo in range(0, len(sel), 16384):
                part = sel[lo:lo + 16384]
                if len(part) == 0:
                    continue
                rb = ResponseBatch.from_lists([bodies[i] for i in part], resp.qos[part], fl[part], now + 1)
                same(g.handle_response_body(rb), o.response_batch(rb), f"round {r} response kind {kind}")
                n_resp += rb.n
    assert np.array_equal(g.snapshot_rate(now + 1), o.snapshot_rate(now + 1)), f"round {r}: rate counters"
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), f"round {r}: quota usage"
    assert np.array_equal(g.snapshot_metrics(), o.snapshot_metrics()), f"round {r}: metrics"
    if rng.random() < 0.2:
        g.load_tables(w.tables); o.reload(w.tables)
    now += int(rng.choice([3, 20, 61, 61, 3600, 86400]))
print(f"soak ok: {rounds} rounds, {n_req} requests, {n_resp} responses, seed {seed}")
