"""GPU parity: the CUDA path, called through the C ABI, against the oracle on the same seeded inputs.
Bit-exact on every output array (reason, detail, flags, qos, token, pick, currentUsage, limitMax, usage ints,
counted) and on the counter snapshots (rate windows, quota usage) after every batch."""
import numpy as np
import pytest

import orklib
from arks_b200 import abi, traffic
from arks_b200.abi import RequestBatch, ResponseBatch
from arks_b200.tables import Tables, simple_endpoint, simple_quota, simple_token
from jsonfuzz import Gen

pytestmark = pytest.mark.gpu
NOW = 1_700_000_000


def pair(gwmod, tables, max_batch=4096, max_bytes=16 << 20):
    g = gwmod.Gateway(0, max_batch, max_bytes)
    g.load_tables(tables)
    return g, orklib.Oracle(tables)


def same(a, b, ctx=""):
    for k, v in a.fields().items():
        w = b.fields()[k]
        if not np.array_equal(v, w):
            bad = np.nonzero(np.any(np.atleast_2d((v != w).reshape(len(v), -1)), axis=1) if v.ndim > 1 else (v != w))[0]
            raise AssertionError(f"{ctx} field {k}: {len(bad)} mismatches, first at {bad[:5]}: gpu={v[bad[:5]]} oracle={w[bad[:5]]}")


def state_same(g, o, now):
    assert np.array_equal(g.snapshot_rate(now), o.snapshot_rate(now)), "rate counters differ"
    assert np.array_equal(g.snapshot_quota(), o.snapshot_quota()), "quota usage differs"


def test_quickstart_config1(gwmod):
    import json, os
    fx = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "quickstart.json")))
    t = Tables(fx["tokens"], fx["quotas"], fx["endpoints"], {("default", "qwen-7b"): ["arks-application-qwen-7b"]})
    g, o = pair(gwmod, t)
    req = RequestBatch.from_lists([fx["request_body"].encode()] * 7, [b"sk-test123456"] * 7, NOW, pick_rand=np.arange(7))
    a = g.handle_request_body(req)
    same(a, o.request_batch(req), "quickstart")
    assert a.reason.tolist() == [0] * 5 + [abi.R_RATE_LIMIT] * 2
    assert g.request_headers(a, 0) == {"model": "qwen-7b", "namespace": "default", "username": "example-token"}
    resp = ResponseBatch.from_lists([fx["response_body"].encode()], [0], [abi.RESP_END_OF_STREAM], NOW + 1)
    c = g.handle_response_body(resp)
    same(c, o.response_batch(resp))
    assert c.usage[0].tolist() == [25, 20, 45]
    assert g.snapshot_rate(NOW + 1)[0].tolist() == [5, 5, 45, 45]
    assert g.snapshot_quota()[0].tolist() == [25, 20, 45]
    state_same(g, o, NOW + 1)


def test_waves_with_noise_and_window_rollover(gwmod):
    w = traffic.Workload(n_tenants=300, seed=3)
    g, o = pair(gwmod, w.tables, 4096, 16 << 20)
    now = NOW
    for wave in range(9):
        req = w.request_batch(3000, now, seed=100 + wave, stream_frac=0.3, noise_frac=0.15, varied=bool(wave & 1))
        a = g.handle_request_body(req)
        same(a, o.request_batch(req), f"wave {wave} request")
        state_same(g, o, now)
        resp = w.response_batch(a, now + 3, seed=200 + wave, noise_frac=0.1, varied=bool(wave & 1))
        if resp.n > 4096:
            resp = ResponseBatch(resp.bodies, resp.body_off[:4096], resp.body_len[:4096], resp.qos[:4096], resp.flags[:4096], resp.now_unix)
        c = g.handle_response_body(resp)
        same(c, o.response_batch(resp), f"wave {wave} response")
        state_same(g, o, now + 3)
        now += [7, 25, 40, 61, 3, 86400, 59, 1, 30][wave]  # several minute roll-overs and one day roll-over


def test_hot_tenant_crosses_limit_inside_a_batch(gwmod):
    toks = [simple_token("hot", "ns0", "tk-hot", "m", [("rpm", 37), ("tpm", 10**9), ("rpd", 50), ("tpd", 10**9)]),
            simple_token("dup", "ns1", "tk-dup", "m", [("rpm", 9), ("rpm", 5), ("rpd", 100)]),
            simple_token("cold", "ns2", "tk-cold", "m", [("rpm", 10**6)])]
    eps = [simple_endpoint("m", ns) for ns in ("ns0", "ns1", "ns2")]
    g, o = pair(gwmod, Tables(toks, [], eps))
    rng = np.random.default_rng(5)
    for rnd in range(4):
        who = rng.choice([b"tk-hot", b"tk-dup", b"tk-cold"], size=1500, p=[0.5, 0.2, 0.3])
        req = RequestBatch.from_lists([b'{"model":"m"}'] * 1500, list(who), NOW + 20 * rnd)
        a = g.handle_request_body(req)
        same(a, o.request_batch(req), f"round {rnd}")
        state_same(g, o, NOW + 20 * rnd)


def test_quota_shapes(gwmod):
    toks = [simple_token("a", "ns", "ta", "m", [("rpm", 100)], "shared"),
            simple_token("b", "ns", "tb", "m", [("tpm", 50)], "shared"),
            simple_token("c", "ns", "tc", "m", [], "absent"),           # ArksQuota missing -> 500 x-error-quota
            simple_token("d", "ns", "td", "m", [], ""),                 # no quota
            {"metadata": {"name": "e", "namespace": "ns"},
             "spec": {"token": "te", "qos": [{"arksEndpoint": {"name": "m2"}, "rateLimits": [{"type": "rpd", "value": 3}]},
                                             {"arksEndpoint": {"name": "m"}, "quota": {"name": "promptonly"}}]}}]
    quotas = [simple_quota("shared", "ns", [("prompt", 120), ("total", 1000), ("total", 400)]),
              simple_quota("promptonly", "ns", [("prompt", 60)])]
    eps = [simple_endpoint("m", "ns"), simple_endpoint("m2", "ns")]
    g, o = pair(gwmod, Tables(toks, quotas, eps))
    rng = np.random.default_rng(9)
    now = NOW
    for rnd in range(6):
        who = rng.choice([b"ta", b"tb", b"tc", b"td", b"te"], size=400)
        bodies = [b'{"model":"m2"}' if (t == b"te" and rng.random() < 0.5) else b'{"model":"m"}' for t in who]
        req = RequestBatch.from_lists(bodies, list(who), now)
        a = g.handle_request_body(req)
        same(a, o.request_batch(req), f"round {rnd}")
        ok = np.nonzero(a.reason == 0)[0][:200]
        rb = [b'{"model":"m","usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}'
              % (p, c, p + c) for p, c in rng.integers(0, 9, (len(ok), 2))]
        if len(ok):
            resp = ResponseBatch.from_lists(rb, a.qos[ok], [abi.RESP_END_OF_STREAM] * len(ok), now + 1)
            same(g.handle_response_body(resp), o.response_batch(resp), f"round {rnd} resp")
        state_same(g, o, now + 1)
        now += 13


@pytest.mark.parametrize("seed", [41, 42])
def test_fuzzed_request_bodies(gwmod, seed):
    w = traffic.Workload(n_tenants=8, seed=1)
    g, o = pair(gwmod, w.tables)
    gen = Gen(seed)
    bodies = [gen.request() for _ in range(4000)]
    toks = [w.token_strings[i % 8] for i in range(4000)]
    req = RequestBatch.from_lists(bodies, toks, NOW)
    same(g.handle_request_body(req), o.request_batch(req), "fuzz")
    state_same(g, o, NOW)


@pytest.mark.parametrize("seed", [51, 52])
def test_fuzzed_response_bodies_and_sse(gwmod, seed):
    w = traffic.Workload(n_tenants=8, seed=1)
    g, o = pair(gwmod, w.tables)
    gen = Gen(seed)
    bodies, flags = [], []
    while len(bodies) < 4000:
        if gen.r.random() < 0.5:
            b, f = gen.response(), abi.RESP_END_OF_STREAM
        else:
            b, f = gen.sse_chunk(), abi.RESP_STREAM
        bodies.append(b)
        flags.append(f if gen.r.random() < 0.97 else 0)
    resp = ResponseBatch.from_lists(bodies, [i % 8 for i in range(4000)], flags, NOW)
    same(g.handle_response_body(resp), o.response_batch(resp), "fuzz resp")
    state_same(g, o, NOW)


@pytest.mark.parametrize("seed", [61, 62])
def test_all_sse_batches_event_parallel_kernel(gwmod, seed):
    """Homogeneous SSE batches take scan_sse_kernel (events cut out by SseSplit, one lane per event). Feed it real-server
    shaped chunks, fuzzed chunks (CR LF, event: lines, multi-line data -> the sequential fallback inside the same
    kernel), chunks with hundreds of tiny events (per-warp event list overflows) and unaligned event starts."""
    w = traffic.Workload(n_tenants=8, seed=1)
    g, o = pair(gwmod, w.tables, 8192, 32 << 20)
    gen = Gen(seed)
    r = gen.r
    usage_ev = b'{"id":"c","choices":[],"usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}'
    delta_ev = b'{"id":"c","object":"chat.completion.chunk","choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":null}],"usage":null}'
    bodies = []
    while len(bodies) < 6000:
        k = r.random()
        if k < 0.35:
            b = gen.sse_chunk()
            if r.random() < 0.5:
                b = b.replace(b"\r\n", b"\n")
        elif k < 0.8:  # what servers send: a few content deltas, sometimes the usage frame and [DONE]
            parts = [b": " + b"k" * r.randint(0, 20) + b"\n\n"] if r.random() < 0.3 else []
            for _ in range(r.randint(1, 8)):
                parts.append(b"data: " + delta_ev % (b"w" * r.randint(0, 40)) + b"\n\n")
            if r.random() < 0.5:
                p, c = r.randint(0, 5000), r.randint(0, 5000)
                parts.append(b"data: " + usage_ev % (p, c, p + c) + b"\n\n")
                if r.random() < 0.3:
                    parts.append(b"data: " + delta_ev % b"after" + b"\n\n")
            if r.random() < 0.5:
                parts.append(b"data: [DONE]\n\n")
                if r.random() < 0.3:
                    parts.append(b"data: {not json\n\n")
            if r.random() < 0.1:
                parts.insert(r.randint(0, len(parts)), b"data: {\"error\":{\"message\":\"boom\"}}\n\n")
            b = b"".join(parts)
            if r.random() < 0.1:
                b = b[:r.randint(0, len(b))]
        elif k < 0.9:  # many tiny events: 32 of these overflow the warp's event list
            n = r.randint(20, 400)
            b = b"".join(b"data: {}\n\n" if r.random() < 0.9 else b"data: " + usage_ev % (1, 2, 3) + b"\n\n" for _ in range(n))
        else:
            b = b"data: " + delta_ev % (b"x" * r.randint(100, 3000)) + b"\n\n" + b"data: " + usage_ev % (7, 8, 15) + b"\n\n"
        bodies.append(b)
    for lo in range(0, 6000, 3000):
        part = bodies[lo:lo + 3000]
        resp = ResponseBatch.from_lists(part, [i % 8 for i in range(len(part))], [abi.RESP_STREAM] * len(part), NOW + lo)
        same(g.handle_response_body(resp), o.response_batch(resp), f"all-sse {lo}")
        state_same(g, o, NOW + lo)


def test_edges_empty_large_reload_and_time(gwmod):
    w = traffic.Workload(n_tenants=16, seed=2)
    g, o = pair(gwmod, w.tables, 512, 8 << 20)
    # empty batch
    e = RequestBatch.from_lists([], [], NOW)
    assert g.handle_request_body(e).reason.shape == (0,)
    # zero-length body, 64 KiB and 1 MiB bodies, a body that is only whitespace
    rng = np.random.default_rng(1)
    big = traffic.chat_request_body(rng, 65536)
    huge = traffic.chat_request_body(rng, 1 << 20)
    req = RequestBatch.from_lists([b"", big, huge, b"   \n", big[:-1]], [w.token_strings[i] for i in range(5)], NOW)
    same(g.handle_request_body(req), o.request_batch(req), "edges")
    # SetUsage / IncrUsage surface
    g.set_quota_usage(3, [5, 6, 7]); o.set_quota_usage(3, [5, 6, 7])
    g.incr_quota_usage(3, [1, 1, 1]); o.incr_quota_usage(3, [1, 1, 1])
    state_same(g, o, NOW)
    # endpoint weight churn (config 5): picks follow the new weights
    g.update_endpoint_weights(2, [0, 0, 9]); o.update_endpoint_weights(2, [0, 0, 9])
    req = w.request_batch(400, NOW + 1, seed=8)
    same(g.handle_request_body(req), o.request_batch(req), "after weight update")
    # reload with one tenant removed and limits changed: counters carried over by key
    w2 = traffic.Workload(n_tenants=15, seed=2)
    g.load_tables(w2.tables); o.reload(w2.tables)
    state_same(g, o, NOW + 1)
    req = w2.request_batch(400, NOW + 2, seed=9)
    same(g.handle_request_body(req), o.request_batch(req), "after reload")
    # the clock must not fall into an earlier window
    with pytest.raises(gwmod.ArksError) as ei:
        g.handle_request_body(w2.request_batch(4, NOW - 120, seed=1))
    assert ei.value.code == abi.E_TIME_WENT_BACK


def test_full_size_wave_64k(gwmod):
    """BASELINE config 2 at full size: 65 536 x 1 KiB requests over 10 000 tenants, three waves, vs the oracle;
    plus the size-independent invariants (admissions never exceed a window's limit; counters == admissions)."""
    w = traffic.Workload(n_tenants=10_000, seed=0xA2C5)
    g, o = pair(gwmod, w.tables, 65536, 80 << 20)
    now = NOW
    admitted_per_tenant = np.zeros(10_000, np.int64)
    for wave in range(3):
        req = w.request_batch(65536, now, seed=300 + wave, n_templates=2048, varied=wave != 1)
        a = g.handle_request_body(req)
        same(a, o.request_batch(req), f"wave {wave}")
        ok = a.reason == 0
        np.add.at(admitted_per_tenant, a.token[ok], 1)
        rate = g.snapshot_rate(now)
        assert np.array_equal(rate[:, 0], admitted_per_tenant)          # rpm counter == admissions this minute
        lim = w.tables.rl_value.reshape(-1, 4)[:, 0]
        assert np.all(rate[:, 0] <= lim)
        resp = w.response_batch(a, now + 2, seed=400 + wave, varied=wave != 1, n_templates=2048)
        n = min(resp.n, 65536)
        resp = ResponseBatch(resp.bodies, resp.body_off[:n], resp.body_len[:n], resp.qos[:n], resp.flags[:n], resp.now_unix)
        c = g.handle_response_body(resp)
        same(c, o.response_batch(resp), f"wave {wave} resp")
        assert np.array_equal(c.usage[:, 0] + c.usage[:, 1], c.usage[:, 2])
        state_same(g, o, now + 2)
        now += 10  # NOW % 60 == 20: all three waves stay inside one minute window


def test_async_pipelined_submits_match_serial_oracle(gwmod):
    """Two batches in flight (slot ping-pong) still apply in call order: same results as the serial oracle."""
    w = traffic.Workload(n_tenants=200, seed=11)
    g, o = pair(gwmod, w.tables, 2048, 8 << 20)
    now = NOW
    reqs = [w.request_batch(1500, now + 3 * k, seed=600 + k, stream_frac=0.2, noise_frac=0.1) for k in range(6)]
    outs = [abi.RequestResult.empty(r.n) for r in reqs]
    inflight = None
    for k, r in enumerate(reqs):
        g.select_slot(k % 2)
        g.submit_request_async(r)
        if inflight is not None:
            g.wait_request(inflight % 2, outs[inflight])
        inflight = k
    g.wait_request(inflight % 2, outs[inflight])
    for k, r in enumerate(reqs):
        same(outs[k], o.request_batch(r), f"async batch {k}")
    state_same(g, o, now + 15)


def test_two_stage_scan_fuzzed_and_plain_documents(gwmod):
    """Batches of 4 096 rows and more go through the fast path (mask_scan.cuh) first and the exact engine for what it declines
    (arks_b200/csrc/mask_scan.cuh). Hostile documents, plain ones and bodies longer than the resident window in ONE batch:
    the verdicts must not depend on which path a row took, and both paths must have been taken."""
    w = traffic.Workload(n_tenants=8, seed=1)
    g, o = pair(gwmod, w.tables, 16384, 48 << 20)
    gen = Gen(91)
    rng = np.random.default_rng(91)
    bodies = [gen.request() for _ in range(5000)]
    bodies += [traffic.chat_request_body_varied(rng, 900, stream=bool(rng.random() < 0.3)) for _ in range(4000)]
    bodies += [traffic.chat_request_body(rng, int(s)) for s in rng.integers(1900, 2300, 300)]  # around the 2 KiB window
    bodies += [b"", b"{}", b'{"model":"qwen-7b"}', traffic.chat_request_body(rng, 70000)]
    order = rng.permutation(len(bodies))
    bodies = [bodies[i] for i in order]
    req = RequestBatch.from_lists(bodies, [w.token_strings[i % 8] for i in range(len(bodies))], NOW,
                                  pick_rand=rng.integers(0, 1 << 63, len(bodies), dtype=np.uint64))
    a = g.handle_request_body(req)
    declined = g.last_declined
    same(a, o.request_batch(req), "two-stage requests")
    state_same(g, o, NOW)
    assert 2000 < declined < len(bodies) - 4000, declined  # the hostile ones went to the exact engine, the plain ones did not
    # complete response bodies (a homogeneous JSON batch takes the two-stage path too)
    rb, flags = [], []
    while len(rb) < 5000:
        rb.append(gen.response())
        flags.append(abi.RESP_END_OF_STREAM if gen.r.random() < 0.97 else 0)
    for _ in range(4000):
        rb.append(traffic.chat_response_body_varied(rng, int(rng.integers(50, 401)), int(rng.integers(1, 513)), 600))
        flags.append(abi.RESP_END_OF_STREAM)
    order = rng.permutation(len(rb))
    resp = ResponseBatch.from_lists([rb[i] for i in order], [int(i) % 8 if i % 97 else -1 for i in range(len(rb))], [flags[i] for i in order], NOW + 1)
    c = g.handle_response_body(resp)
    declined = g.last_declined
    same(c, o.response_batch(resp), "two-stage responses")
    state_same(g, o, NOW + 1)
    assert 1500 < declined < len(rb) - 3500, declined
    # the bench workload itself: nothing declined
    wave = w.request_batch(8192, NOW + 2, seed=5, varied=True)
    same(g.handle_request_body(wave), o.request_batch(wave), "plain wave")
    assert g.last_declined == 0
    # the same bodies packed on 16-byte boundaries (all the ABI asks for): half of them start in the middle of a 32-byte
    # sector and are read with two bounds-checked 16-byte loads instead of one whole-sector read
    bb, bo, bl = abi.pack_blobs(bodies, align=16)
    assert (bo % 32 == 16).sum() > 1000
    req16 = RequestBatch(bb, bo, bl, req.tokens, req.token_off, NOW + 3, req.pick_rand)
    same(g.handle_request_body(req16), o.request_batch(req16), "two-stage requests, 16-byte packing")
    state_same(g, o, NOW + 3)


@pytest.mark.parametrize("seed", [95, 96])
def test_latency_path_warp_per_body_fuzzed(gwmod, seed):
    """Micro-batches (up to 2 048 rows) take the warp-per-body latency path (arks_b200/csrc/warp_scan.cuh) in front of the exact
    engine: hostile and plain documents, bodies around the resident window, every batch size from 1 up."""
    w = traffic.Workload(n_tenants=8, seed=1)
    g, o = pair(gwmod, w.tables, 4096, 16 << 20)
    gen = Gen(seed)
    rng = np.random.default_rng(seed)
    now = NOW
    for n in (1, 2, 31, 33, 64, 700, 2048):
        bodies = [gen.request() if rng.random() < 0.5 else traffic.chat_request_body_varied(rng, 900, stream=bool(rng.random() < 0.3))
                  for _ in range(n)]
        if n >= 64:
            bodies[5] = traffic.chat_request_body(rng, 2047)
            bodies[6] = traffic.chat_request_body(rng, 2049)
            bodies[7] = b""
        req = RequestBatch.from_lists(bodies, [w.token_strings[i % 8] for i in range(n)], now, pick_rand=rng.integers(0, 1 << 63, n, dtype=np.uint64))
        a = g.handle_request_body(req)
        assert g.last_declined >= 0  # the batch took the two-stage (latency) path
        same(a, o.request_batch(req), f"warp path requests n={n}")
        rb, flags = [], []
        while len(rb) < n:
            rb.append(gen.response() if rng.random() < 0.5 else traffic.chat_response_body_varied(rng, 10, 20, 600))
            flags.append(abi.RESP_END_OF_STREAM if rng.random() < 0.95 else 0)
        resp = ResponseBatch.from_lists(rb, [int(i) % 8 if i % 13 else -1 for i in range(n)], flags, now + 1)
        c = g.handle_response_body(resp)
        same(c, o.response_batch(resp), f"warp path responses n={n}")
        state_same(g, o, now + 1)
        now += 3
