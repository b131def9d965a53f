#!/usr/bin/env python
"""What the sliding window (arks_set_sliding_window) costs on a request step of 65 536 rows, with the rate-limit report off and
on, on two workloads:

  config-2   10 000 uniform tenants (bench.py's request wave)
  zipf       100 000 tenants with Zipf(1.1) popularity (bench_configs.py config 4): the largest groups exceed kHotGroup

For each, four contexts hold the same tables and the same staged batch (sliding off / on x report off / on) and are stepped
alternately in one process, 30 s apart, so that every window has a previous one. Per mode: the rank_hot + limit_admit interval
from the library's own events (arks_last_kernel_ms, median of the profiled steps), the whole request step (run + result fetch,
wall clock, median) timed without the events, and whether the outputs that must be equal are: the report changes no decision
or counter in either window kind. The card's name and power limit are printed with the numbers; one JSON line per workload."""
import dataclasses
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

import __graft_entry__ as ge  # noqa: E402

ge.build()
from arks_b200 import abi, traffic  # noqa: E402
from arks_b200.gateway import Gateway  # noqa: E402
from bench import pin_batch  # noqa: E402

NOW0 = 1_700_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def workload(name, wave):
    if name == "config-2":
        w = traffic.Workload(10_000, seed=0xA2C5)
    else:
        w = traffic.Workload(100_000, seed=0xA2C6, zipf_alpha=1.1)
    req = w.request_batch(wave, NOW0, seed=41, n_templates=2048, varied=True)
    tok = np.frombuffer(req.tokens[:req.token_off[-1]], np.uint8).reshape(wave, -1)
    _, counts = np.unique(tok, axis=0, return_counts=True)
    return w, pin_batch(req), int(counts.max())


MODES = ("fixed", "sliding", "fixed+report", "sliding+report")


def same(a, b):
    return all(np.array_equal(v, b.fields()[k]) for k, v in a.fields().items())


def measure(name, wave=65536, steps=21):
    w, req, largest = workload(name, wave)
    gs = {}
    for mode in MODES:
        g = Gateway(0, wave, int(wave * 1100 * 1.05))
        g.load_tables(w.tables)
        if "report" in mode:
            g.set_ratelimit_report(True)
        if mode.startswith("sliding"):
            g.set_sliding_window(True)
        gs[mode] = g
    now = NOW0
    res = {m: gs[m].handle_request_body(req) for m in gs}  # a first window's worth of counts
    now += 60
    res = {m: gs[m].handle_request_body(dataclasses.replace(req, now_unix=now)) for m in gs}
    equal = same(res["fixed"], res["fixed+report"]) and same(res["sliding"], res["sliding+report"])
    equal &= res["sliding+report"].rl_reset is not None and res["fixed+report"].rl_reset is None
    differs = not same(res["fixed"], res["sliding"])  # the previous window's share denies more
    for g in gs.values():
        g.stage_request(req)
    kern = {m: [] for m in gs}
    wall = {m: [] for m in gs}
    out = {m: abi.RequestResult.empty(wave, report="report" in m, sliding=m.startswith("sliding")) for m in gs}
    for i in range(3 + steps):  # alternating order (the first three rounds warm up)
        now += 30  # every other step starts a new minute: prev is always there
        for m in MODES if i % 2 == 0 else MODES[::-1]:
            g = gs[m]
            torch.cuda.synchronize()
            t0 = time.perf_counter()  # the whole step, events off; the fetch waits for the device
            g.run_request(now)
            g.fetch_request(wave, out[m])
            t1 = time.perf_counter()
            g.set_profiling(True)  # then the same step once more with the library's kernel events
            g.run_request(now)
            g.fetch_request(wave, out[m])
            k = g.last_kernel_ms()
            g.set_profiling(False)
            if i >= 3:
                kern[m].append(k[1])
                wall[m].append((t1 - t0) * 1e3)
        equal &= same(out["fixed"], out["fixed+report"]) and same(out["sliding"], out["sliding+report"])
    for a, b in (("fixed", "fixed+report"), ("sliding", "sliding+report")):
        equal &= bool(np.array_equal(gs[a].snapshot_rate(now), gs[b].snapshot_rate(now)))
        equal &= bool(np.array_equal(gs[a].snapshot_rate_prev(now), gs[b].snapshot_rate_prev(now)))
    med = {m: (float(np.median(kern[m])), float(np.median(wall[m]))) for m in gs}
    return {"workload": name, "rows": wave, "largest_group": largest, "steps_per_mode": steps,
            "rank_hot_plus_limit_admit_ms": {m: round(med[m][0], 4) for m in gs},
            "request_step_ms": {m: round(med[m][1], 3) for m in gs},
            "admit_delta_ms": {"report off": round(med["sliding"][0] - med["fixed"][0], 4),
                               "report on": round(med["sliding+report"][0] - med["fixed+report"][0], 4)},
            "outputs_equal": bool(equal), "sliding_decides_differently": bool(differs), "card": card()}


if __name__ == "__main__":
    for name in ("config-2", "zipf"):
        print(json.dumps(measure(name)), flush=True)
