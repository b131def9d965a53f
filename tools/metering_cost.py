#!/usr/bin/env python
"""What stream metering (N5, arks_set_stream_metering) costs on a config-3 shaped step: 65 536 streams, each a request and
4 SSE chunks of ~1 KiB, with the BPE counter on. Three measurements, one JSON line each:

  reference   stream:true + include_usage, metering off: the chunks are billed by their upstream `usage`
  metered     the same traffic without include_usage, metering on, every chunk marked ARKS_RESP_METERED
  meter       meter_charge_kernel alone, from the library's own events (arks_last_kernel_ms), next to the BPE kernels

Step times are CUDA events around whole steps on the library's stream (inputs resident in HBM). The card's name and power
limit are printed with the numbers."""
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

import __graft_entry__ as ge  # noqa: E402

ge.build()
from arks_b200 import abi, bpe, traffic  # noqa: E402
from arks_b200.abi import RequestBatch, ResponseBatch  # noqa: E402
from arks_b200.gateway import Gateway  # noqa: E402
from bench import pin_batch  # noqa: E402
from bench_configs import timed  # noqa: E402

NOW0, DAY = 1_700_000_000, 86_400


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def rows(b):
    return [bytes(b.bodies[b.body_off[i]:b.body_off[i] + b.body_len[i]]) for i in range(b.n)]


def variant(w, tables, metered, wave, steps):
    g = Gateway(0, wave, int(wave * 1100 * 1.05))
    g.load_tables(w.tables)
    g.load_bpe(tables)
    req = w.request_batch(wave, NOW0, seed=31, stream_frac=1.0, n_templates=2048, varied=True)
    if metered:
        bodies = [re.sub(rb',\s*"stream_options":\{"include_usage":true\}', b"", b) for b in rows(req)]
        toks = [bytes(req.tokens[req.token_off[i]:req.token_off[i + 1]]) for i in range(req.n)]
        req = RequestBatch.from_lists(bodies, toks, NOW0, pick_rand=req.pick_rand)
        g.set_stream_metering(True)
    req = pin_batch(req)
    a = g.handle_request_body(req)
    ok = a.reason == abi.R_OK
    assert ok.mean() > 0.9 and bool(np.all(a.flags[ok] & abi.FLAG_METERED)) == metered
    allresp = w.response_batch(a, NOW0 + 1, seed=32)
    flags = allresp.flags | (abi.RESP_METERED if metered else 0)
    idx, parts, chunks = np.arange(allresp.n), [], rows(allresp)
    for c in range(4):  # chunk c of every stream -> response batch c
        sel = idx[c::4]
        parts.append(pin_batch(ResponseBatch.from_lists([chunks[i] for i in sel], allresp.qos[sel], flags[sel], NOW0 + 1)))
    g.select_slot(0); g.stage_request(req)
    for c, p in enumerate(parts):
        g.select_slot(c); g.stage_response(p)
    state = {"now": NOW0 + DAY}

    def step(i):
        g.select_slot(0); g.run_request(state["now"])
        for c in range(4):
            g.select_slot(c); g.run_response(state["now"] + 1)
        state["now"] += DAY
    ms = timed(g, step, steps)
    # per-kernel times of one profiled step: request [scan, admit, fast, bpe, (meter)], response [scan, fast, bpe, (meter)]
    g.set_profiling(True)
    k_req, k_resp = [], []
    for _ in range(5):
        g.select_slot(0); g.run_request(state["now"]); k_req.append(g.last_kernel_ms())
        for c in range(4):
            g.select_slot(c); g.run_response(state["now"] + 1); k_resp.append(g.last_kernel_ms())
        state["now"] += DAY
    g.set_profiling(False)
    kq, kr = np.median(np.array(k_req), axis=0), np.median(np.array(k_resp), axis=0)
    out = {"ms_per_step": ms, "streams_per_s": wave / ms * 1e3, "bpe_request_ms": float(kq[3]), "bpe_chunk_batch_ms": float(kr[2])}
    if metered:
        out.update(meter_request_us=float(kq[4]) * 1e3, meter_chunk_batch_us=float(kr[3]) * 1e3)
    return out


def main(wave=65536, steps=20):
    tok, text = bpe.standin_tokenizer(151_643, cache_dir=os.path.join(tempfile.gettempdir(), "arks_bench"))
    tables = bpe.load_tokenizer(text)
    w = traffic.Workload(10_000, seed=0xA2C5)
    gpu = card()
    shape = f"{wave} streams x (1 request + 4 SSE chunks of ~1 KiB), BPE on"
    ref = variant(w, tables, False, wave, steps)
    met = variant(w, tables, True, wave, steps)
    print(json.dumps({"variant": "reference (include_usage, metering off)", "shape": shape, "gpu": gpu, **ref}), flush=True)
    print(json.dumps({"variant": "metered (no include_usage, metering on)", "shape": shape, "gpu": gpu, **met}), flush=True)
    print(json.dumps({"variant": "meter kernels alone", "gpu": gpu, "request_batch_us": met["meter_request_us"],
                      "chunk_batch_us": met["meter_chunk_batch_us"],
                      "step_overhead_ms": met["ms_per_step"] - ref["ms_per_step"]}), flush=True)


if __name__ == "__main__":
    main()
