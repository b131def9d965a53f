"""The oracle of stream metering (N5, include/arks_gateway.h: arks_set_stream_metering), composed from the C oracle's reference
decisions. TEST INFRASTRUCTURE.

The metering policy is additive to the reference path, so it is stated here on top of orklib.Oracle instead of inside it:
  - a stream:true request without include_usage is decided like any other: the oracle decides the same body with
    `"stream_options":{"include_usage":true}` appended as its last member (the model span does not move); admitted rows get
    FLAG_METERED;
  - the prompt of an admitted metered row is charged after the batch (its micro-batch commits), a chunk of a metered stream
    answered ARKS_R_OK when it is processed. A charge of `c` tokens is applied by the oracle itself, as one synthetic complete
    response with usage (prompt c, completion 0, total c) or (0, c, c) on the row's qos entry: that is exactly c on every
    tpm / tpd entry and c on the quota items of the prompt (response) and total types. ARKS_RESP_COMPLETED keeps it out of
    the token-usage series, and the one response-message count it adds is taken back, so the metrics are corrected here;
  - a metered chunk is decoded by the oracle's SSE decoder alone: its usage is reported, never billed (counted = 0);
  - the counts come from the test (`counts`, the oracle has no tokenizer); a row without one (None, ARKS_BPE_UNCOUNTED) is
    billed its body length; the N4 pre-charge estimates of metered rows are withheld from the oracle.
The appended member must be the body's only stream_options: bodies that already carry one are not modelled."""
from __future__ import annotations

import numpy as np

import orklib
from arks_b200 import abi
from arks_b200.abi import RequestBatch, ResponseBatch

UNCOUNTED = 0xFFFFFFFF
METERED_CHUNK = abi.RESP_STREAM | abi.RESP_METERED
_INCLUDE_USAGE = b',"stream_options":{"include_usage":true}'


def rows(b) -> list[bytes]:
    return [bytes(b.bodies[b.body_off[i]:b.body_off[i] + b.body_len[i]]) for i in range(b.n)]


def is_metered_request(body: bytes) -> bool:
    """stream:true without stream_options.include_usage:true, in a body the reference decodes"""
    err, _, stream, so, iu = orklib.parse_request_body(body)
    return err == 0 and stream == 2 and not (so and iu == 2)


def _usage_body(prompt: int, completion: int) -> bytes:
    return b'{"model":"m","usage":{"prompt_tokens":%d,"completion_tokens":%d,"total_tokens":%d}}' % (prompt, completion,
                                                                                                      prompt + completion)


class MeteredOracle:
    def __init__(self, tables):
        self.tables = tables
        self.o = orklib.Oracle(tables)
        self.meter = False
        self.precharge = False
        self.metrics = np.zeros((tables.n_qos, abi.METRIC_COLS), np.int64)  # correction of the oracle's series

    def set_stream_metering(self, on: bool):
        self.meter = bool(on)

    def set_precharge(self, on: bool):
        self.precharge = bool(on)
        self.o.set_precharge(on)

    def _charge(self, qos, amounts, side, now):
        """`amounts` tokens on the rows' qos entries; side 0 prompt, 1 completion"""
        sel = [k for k, c in enumerate(amounts) if c]
        if not sel:
            return
        bodies = [_usage_body(amounts[k], 0) if side == 0 else _usage_body(0, amounts[k]) for k in sel]
        q = [int(qos[k]) for k in sel]
        self.o.response_batch(ResponseBatch.from_lists(bodies, q, [abi.RESP_END_OF_STREAM | abi.RESP_COMPLETED] * len(sel), now))
        for k in sel:
            self.metrics[qos[k], abi.METRIC_MESSAGES] -= 1
            self.metrics[qos[k], abi.METRIC_USAGE + side] += amounts[k]

    def request_batch(self, b: RequestBatch, counts=None):
        bodies = rows(b)
        metered = np.array([self.meter and is_metered_request(x) for x in bodies], bool)
        if self.precharge and counts is not None:
            self.o.set_estimates(np.where(metered, 0, np.asarray(counts, np.uint32)))
        if metered.any():
            for i in np.flatnonzero(metered):
                k = bodies[i].rindex(b"}")
                bodies[i] = bodies[i][:k] + _INCLUDE_USAGE + bodies[i][k:]
            toks = [bytes(b.tokens[b.token_off[i]:b.token_off[i + 1]]) for i in range(b.n)]
            b2 = RequestBatch.from_lists(bodies, toks, b.now_unix, pick_rand=b.pick_rand)
        else:
            b2 = b
        r = self.o.request_batch(b2)
        ok = metered & (r.reason == abi.R_OK)
        r.flags[ok] |= abi.FLAG_METERED
        sel = np.flatnonzero(ok)
        amounts = [int(b.body_len[i]) if counts is None or int(counts[i]) == UNCOUNTED else int(counts[i]) for i in sel]
        self._charge(r.qos[sel], amounts, 0, b.now_unix)
        return r

    def response_batch(self, b: ResponseBatch, counts=None):
        r = abi.ResponseResult.empty(b.n)
        metered = (np.asarray(b.flags) & METERED_CHUNK) == METERED_CHUNK
        bodies = rows(b)
        plain = np.flatnonzero(~metered)
        if len(plain):
            sub = ResponseBatch.from_lists([bodies[i] for i in plain], b.qos[plain], b.flags[plain], b.now_unix)
            if b.precharged is not None:
                sub.precharged = np.ascontiguousarray(b.precharged[plain], np.uint32)
            got = self.o.response_batch(sub)
            r.reason[plain], r.counted[plain], r.usage[plain] = got.reason, got.counted, got.usage
        charge_q, charge_c = [], []
        for i in np.flatnonzero(metered):
            q = int(b.qos[i])
            r.counted[i] = 0
            if q < 0 or q >= self.tables.n_qos:
                r.reason[i], r.usage[i] = abi.R_QOS_GONE, 0
                continue
            rc, u = orklib.parse_sse_chunk(bodies[i])
            r.reason[i] = abi.R_STREAMING if rc else abi.R_OK
            r.usage[i] = 0 if rc else u
            c = 0 if rc else int(b.body_len[i]) if counts is None or int(counts[i]) == UNCOUNTED else int(counts[i])
            self.metrics[q, abi.METRIC_MESSAGES] += 1  # every response-body message, billed or not
            charge_q.append(q)
            charge_c.append(c)
        self._charge(charge_q, charge_c, 1, b.now_unix)
        return r

    def snapshot_rate(self, now):
        return self.o.snapshot_rate(now)

    def snapshot_quota(self):
        return self.o.snapshot_quota()

    def snapshot_metrics(self):
        return self.o.snapshot_metrics() + self.metrics
