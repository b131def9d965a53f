#!/usr/bin/env python
"""What per-model vocabularies (arks_load_bpe_vocab, arks_bind_model_vocab) cost the BPE kernels on a 65 536-body config-2
wave. Slot 0 holds bench.py's 151 k-merge Qwen2 stand-in, slot 1 a Llama 3 style stand-in of the same size (numbers in runs
of up to three, `ignore_merges`); model llama-3 is bound to slot 1. Device time of the BPE kernels per wave
(arks_last_kernel_ms, median of 15 profiled waves), one JSON line per case:

  single      one vocabulary, no binding: the kernels every context without the new calls runs (the reference point)
  slot0       two vocabularies bound, every row names qwen-7b (slot 0): the split kernel + both slots' kernels
  mixed       rows alternate between qwen-7b and llama-3 (50 / 50)
  slot1       every row names llama-3 (slot 1)

The card's name and power limit are printed with the numbers."""
import copy
import json
import os
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
from arks_b200.abi import RequestBatch  # noqa: E402
from arks_b200.gateway import Gateway  # noqa: E402
from arks_b200.tables import Tables  # noqa: E402
from bench import pin_batch  # noqa: E402

NOW0, DAY = 1_700_000_000, 86_400
LLAMA = "llama-3"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def two_model_tables(w):
    """the config-2 objects with a second model: every token has a qos entry for llama-3 too, every namespace its endpoint"""
    tokens, quotas, endpoints = copy.deepcopy(w.objects)
    for t in tokens:
        q = copy.deepcopy(t["spec"]["qos"][0])
        q["arksEndpoint"]["name"] = LLAMA
        t["spec"]["qos"].append(q)
    endpoints += [dict(copy.deepcopy(e), metadata=dict(e["metadata"], name=LLAMA)) for e in endpoints]
    return Tables(tokens, quotas, endpoints)


def wave_with_models(base, which):
    """`base` with each row's model set by which(i): 0 qwen-7b, 1 llama-3"""
    bodies = [bytes(base.bodies[base.body_off[i]:base.body_off[i] + base.body_len[i]]) for i in range(base.n)]
    bodies = [b.replace(b'"model":"qwen-7b"', b'"model":"llama-3"') if which(i) else b for i, b in enumerate(bodies)]
    toks = [bytes(base.tokens[base.token_off[i]:base.token_off[i + 1]]) for i in range(base.n)]
    return pin_batch(RequestBatch.from_lists(bodies, toks, NOW0, pick_rand=base.pick_rand))


_now = [NOW0 + DAY]


def bpe_ms(g, req, waves=15):
    g.select_slot(0)
    g.stage_request(req)
    g.set_profiling(True)
    t = []
    for i in range(3 + waves):
        g.run_request(_now[0])
        k = g.last_kernel_ms()
        if i >= 3:
            t.append(k[3])
        _now[0] += DAY
    g.set_profiling(False)
    return float(np.median(t)), float(np.min(t)), float(np.max(t))


def main(wave=65536):
    cache = os.path.join(tempfile.gettempdir(), "arks_bench")
    _, qtext = bpe.standin_tokenizer(151_643, cache_dir=cache)
    _, ltext = bpe.standin_tokenizer(151_643, cache_dir=cache, pattern=bpe.LLAMA3_PATTERN, ignore_merges=True)
    qt, lt = bpe.load_tokenizer(qtext), bpe.load_tokenizer(ltext)
    w = traffic.Workload(10_000, seed=0xA2C5)
    tables = two_model_tables(w)
    base = w.request_batch(wave, NOW0, seed=31, n_templates=4096, varied=True, stream_frac=0.2)
    gpu = card()
    shape = f"{wave}-body config-2 request wave (varied bodies, 4 096 templates)"
    single = Gateway(0, wave, int(wave * 1100 * 1.05))
    single.load_tables(tables)
    single.load_bpe(qt)
    req0 = wave_with_models(base, lambda i: 0)
    a = single.handle_request_body(req0)
    assert (a.reason == abi.R_OK).mean() > 0.8
    out = {"single": bpe_ms(single, req0)}
    single.close()
    g = Gateway(0, wave, int(wave * 1100 * 1.05))
    g.load_bpe(qt)
    g.load_bpe_vocab(1, lt)
    g.bind_model_vocab(LLAMA, 1)
    g.load_tables(tables)
    for name, which in (("slot0", lambda i: 0), ("mixed", lambda i: i & 1), ("slot1", lambda i: 1)):
        out[name] = bpe_ms(g, wave_with_models(base, which))
    for name, (med, lo, hi) in out.items():
        print(json.dumps({"case": name, "shape": shape, "gpu": gpu, "bpe_ms_median": med, "bpe_ms_min": lo, "bpe_ms_max": hi}),
              flush=True)
    print(json.dumps({"mixed_ms": out["mixed"][0], "slot0_plus_slot1_ms": out["slot0"][0] + out["slot1"][0],
                      "mean_of_slot0_slot1_ms": (out["slot0"][0] + out["slot1"][0]) / 2}), flush=True)


if __name__ == "__main__":
    main()
