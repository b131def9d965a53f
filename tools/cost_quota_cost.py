#!/usr/bin/env python
"""What `cost` quota items (ARKS_QT_COST) cost on bench.py's config-2 step: one request wave of 65 536 rows and its response
wave, run resident in HBM, on 10 000 uniform tenants.

Two contexts hold the same workload: `plain`, the config-2 tables as they are, and `cost`, the same tables with a cost item
appended to every quota (a limit no tenant reaches, so decisions stay the same) and every tenant endpoint priced. Both get
the same staged waves and are stepped alternately in one process. Per context: the whole step (request + response kernels,
CUDA events on the library's stream, median), the admission interval and the response scan interval from the library's own
events (arks_last_kernel_ms, median of separate profiled steps), the launches per step, and whether the request results and
the token counters are equal (they must be: only the cost column differs). The card's name and power limit are printed with
the numbers; one JSON line."""
import copy
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

import __graft_entry__ as ge  # noqa: E402

ge.build()
from arks_b200 import traffic  # noqa: E402
from arks_b200.gateway import Gateway  # noqa: E402
from arks_b200.tables import Tables  # noqa: E402
from bench import pin_batch  # noqa: E402

NOW0 = 1_700_000_000
DAY = 86_400
WAVE = 65_536


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def cost_tables(w, seed=5):
    rng = np.random.default_rng(seed)
    tokens, quotas, endpoints = copy.deepcopy(w.objects)
    for q in quotas:
        q["spec"]["quotas"].append({"type": "cost", "value": 1 << 62})
    for e in endpoints:
        e["spec"]["pricing"] = {"prompt": int(rng.integers(100, 5000)), "completion": int(rng.integers(100, 20000))}
    return Tables(tokens, quotas, endpoints)


def measure(steps=41):
    w = traffic.Workload(10_000, seed=0xA2C5)
    req = pin_batch(w.request_batch(WAVE, NOW0, seed=41, varied=True))
    gs = {}
    for name, t in (("plain", w.tables), ("cost", cost_tables(w))):
        g = Gateway(0, WAVE, int(WAVE * 1100 * 1.05))
        g.load_tables(t)
        gs[name] = g
    res = {n: g.handle_request_body(req) for n, g in gs.items()}
    resp = pin_batch(w.response_batch(res["plain"], NOW0 + 1, seed=42, body_size=600, varied=True))
    for n, g in gs.items():
        g.handle_response_body(resp)
    equal = all(np.array_equal(v, res["cost"].fields()[k]) for k, v in res["plain"].fields().items())
    for g in gs.values():
        g.stage_request(req)
        g.stage_response(resp)
    now = NOW0 + DAY
    step_ms = {n: [] for n in gs}
    admit_ms = {n: [] for n in gs}
    resp_ms = {n: [] for n in gs}
    launches = {}
    order = list(gs)
    for i in range(3 + steps):  # alternating order (the first three rounds warm up)
        now += DAY  # fresh windows each step, like bench.py
        for n in order if i % 2 == 0 else order[::-1]:
            g = gs[n]
            ext = torch.cuda.ExternalStream(g.stream_handle)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            l0 = g.launch_count
            e0.record(ext)
            g.run_request(now)
            g.run_response(now + 1)
            e1.record(ext)
            e1.synchronize()
            launches[n] = g.launch_count - l0
            g.set_profiling(True)
            g.run_request(now)
            k_req = g.last_kernel_ms()
            g.run_response(now + 1)
            k_resp = g.last_kernel_ms()
            g.set_profiling(False)
            torch.cuda.synchronize()
            if i >= 3:
                step_ms[n].append(e0.elapsed_time(e1))
                admit_ms[n].append(k_req[1])
                resp_ms[n].append(k_resp[0])
    equal &= bool(np.array_equal(gs["plain"].snapshot_quota(), gs["cost"].snapshot_quota()))
    equal &= bool(np.array_equal(gs["plain"].snapshot_rate(now), gs["cost"].snapshot_rate(now)))
    billed = bool((gs["cost"].snapshot_quota_cost() != 0).any()) and not (gs["plain"].snapshot_quota_cost() != 0).any()
    med = lambda d: {n: round(float(np.median(v)), 4) for n, v in d.items()}
    spread = lambda d: {n: [round(float(np.min(v)), 4), round(float(np.max(v)), 4)] for n, v in d.items()}
    return {"workload": "config-2", "request_rows": WAVE, "response_rows": int(resp.n), "steps_per_context": steps,
            "step_ms_median": med(step_ms), "step_ms_min_max": spread(step_ms),
            "rank_hot_plus_limit_admit_ms": med(admit_ms), "response_scan_ms": med(resp_ms),
            "step_delta_ms": round(float(np.median(step_ms["cost"]) - np.median(step_ms["plain"])), 4),
            "launches_per_step": launches, "decisions_and_token_counters_equal": bool(equal), "cost_billed": billed,
            "card": card()}


if __name__ == "__main__":
    print(json.dumps(measure()), flush=True)
