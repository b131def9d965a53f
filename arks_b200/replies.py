"""What the reference puts on the wire for a failed request / response phase (SURVEY.md §8a A13): HTTP status, the
x-error-* header WITH THE VALUE the Go code sends, and the `error.message` of the JSON body. Python twin of
host/cpp's RequestErrorReply / ResponseErrorReply (same table; tests/test_error_replies.py holds both to
tests/golden/error_replies.json).

  handle_request.go:48-56,97-171,199-205   check.go:76-104,140-152   handle_response.go:125-181,215-223
  ratelimiter/types.go:98-114 (RateLimitResponse.JSON)   quota/types.go:41-55 (QuotaResult.JSON)   util.go:40-77

Not a function of the request stream in the reference, hence fixed here: `expiresAt` of a 429 (wall clock + Redis TTL with
jitter; here the end of the rule's window), the wording of third-party decoder errors (x-error-streaming /
x-error-response-unmarshal messages), and the member order of the body's inner map.
"""
from __future__ import annotations

import json
import time

from . import abi

WINDOW = {"rpm": 60, "tpm": 60, "rpd": 86400, "tpd": 86400}  # ratelimiter/rate_limiter.go:31-68


def _rfc3339(unix_s: int) -> str:
    return time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime(unix_s))


def _go_str(s: str) -> str:
    """encoding/json string (inside the message, which is itself a JSON document)"""
    return json.dumps(s, ensure_ascii=False)


def _utf8(r: int) -> bytes:
    if r > 0x10FFFF or 0xD800 <= r <= 0xDFFF:
        r = 0xFFFD
    return chr(r).encode("utf-8")


_SIMPLE = {ord("b"): b"\b", ord("f"): b"\f", ord("n"): b"\n", ord("r"): b"\r", ord("t"): b"\t"}


def decode_model(raw: bytes, escaped: bool) -> str:
    """the model name out of its raw span (arks_request_result.model_off / model_len): jsoniter's ReadString on bytes the
    parser already accepted -- escapes are decoded (a lone surrogate becomes U+FFFD, a pair one code point), every other
    byte is copied as it is, valid UTF-8 or not. Bytes that are not UTF-8 travel as surrogate escapes in the str and come
    out as the same bytes on the wire (Go strings are byte strings: `RawValue: []byte(...)`, util.go:40-77)."""
    if not escaped:
        return raw.decode("utf-8", "surrogateescape")

    def hex4(i):
        v = 0
        for c in raw[i:i + 4]:
            v = v * 16 + (c - 48 if c <= 57 else (c | 0x20) - 97 + 10)
        return v
    o, i, n = bytearray(), 0, len(raw)
    while i < n:
        c = raw[i]
        i += 1
        if c != 0x5C or i >= n:
            o.append(c)
            continue
        e = raw[i]
        i += 1
        while True:
            if e != 0x75:  # not \u
                o += _SIMPLE.get(e, bytes([e]))
                break
            r = hex4(i)
            i += 4
            if r < 0xD800 or r > 0xDFFF or i >= n or raw[i] != 0x5C:
                o += _utf8(r)
                break
            i += 1
            e = raw[i] if i < n else 0x5C
            i += 1 if i < n else 0
            if e != 0x75:  # the next escape is decoded on its own
                o += _utf8(r)
                continue
            r2 = hex4(i)
            i += 4
            if r < 0xDC00 and 0xDC00 <= r2 < 0xE000:
                o += _utf8((((r - 0xD800) << 10) | (r2 - 0xDC00)) + 0x10000)
            else:
                o += _utf8(r) + _utf8(r2)
            break
    return bytes(o).decode("utf-8", "surrogateescape")


def window_end(now_unix: int, rule: str) -> int:
    """end of the fixed window of `rule` that holds now_unix: the 429 body's expiresAt and the x-ratelimit-reset-* /
    retry-after headers. Go truncates time relative to year 1 (62135596800 s before the epoch)."""
    w = WINDOW[rule]
    return now_unix - ((now_unix + 62135596800) % w) + w


def go_duration(seconds: int) -> str:
    """time.Duration.String() of whole seconds: "1s", "59s", "1m0s", "23h59m59s" (the x-ratelimit-reset-* format)"""
    h, m, s = seconds // 3600, seconds // 60 % 60, seconds % 60
    return f"{h}h{m}m{s}s" if h else f"{m}m{s}s" if m else f"{s}s"


RATELIMIT_HEADERS = tuple(f"x-ratelimit-{w}-{k}" for k in ("requests", "tokens") for w in ("limit", "remaining", "reset"))


def ratelimit_headers(reason: int, detail: int, qos: int, now_unix: int, rl_entry, rl_limit, rl_remaining, tables, rl_reset=None,
                      rl_retry=None):
    """the headers of the rate-limit report (arks_set_ratelimit_report) for one request decision, in wire order: retry-after
    on a rate-limit 429 (until the denying entry's window ends), then limit / remaining / reset of the requests figure, then
    of the tokens figure. A figure without an entry (abi.RL_NONE) adds nothing; [] when the decision carries no report.
    Under the sliding window (arks_set_sliding_window) the decision also carries rl_reset / rl_retry, the seconds the device
    projected, and those replace the window ends."""
    if reason not in (abi.R_OK, abi.R_RATE_LIMIT, abi.R_QUOTA) or rl_entry is None or all(int(e) == abi.RL_NONE for e in rl_entry):
        return []
    names = tables.qos_rule_names[qos]
    out = []
    if reason == abi.R_RATE_LIMIT:
        out.append(("retry-after", str(int(rl_retry) if rl_retry is not None else window_end(now_unix, names[detail]) - now_unix)))
    for t, kind in enumerate(("requests", "tokens")):
        e = int(rl_entry[t])
        if e == abi.RL_NONE:
            continue
        out += [(f"x-ratelimit-limit-{kind}", str(int(rl_limit[t]))), (f"x-ratelimit-remaining-{kind}", str(int(rl_remaining[t]))),
                (f"x-ratelimit-reset-{kind}", go_duration(int(rl_reset[t]) if rl_reset is not None else window_end(now_unix, names[e]) - now_unix))]
    return out


def request_error_reply(reason: int, detail: int, cur_usage: int, limit_max: int, now_unix: int, tables, qos: int,
                        token: bytes, model: str, rl_retry=None):
    """-> (status, header, header value, message). `rl_retry`: the sliding window's retry time of a rate-limit 429
    (arks_set_sliding_window with the report), which expiresAt then names instead of the window end"""
    status, header = abi.REASON_HTTP.get(reason, (500, "x-error-rate-limit"))
    value, msg = "true", ""
    if reason == abi.R_NO_TOKEN:
        msg = "no token found in request headers"
    elif reason == abi.R_REQUEST_BODY:
        msg = "error processing request body"
    elif reason == abi.R_NO_MODEL:
        value, msg = "", "no model in request body"
    elif reason == abi.R_TOKEN_NOT_FOUND:
        value, msg = "token not found: " + token.decode("utf-8", "surrogateescape"), "error to get qos by token"
    elif reason == abi.R_MODEL_NOT_IN_TOKEN:
        value, msg = "model not found: " + model, "error to get qos by token"
    elif reason == abi.R_NO_MODEL_BACKENDS:
        value, msg = model, "model %s does not exist" % model
    elif reason == abi.R_STREAM_OPTIONS:
        value, msg = "include_usage for stream_options not set", "no stream with usage option available"
    elif reason == abi.R_RATE_LIMIT:
        rule = tables.qos_rule_names[qos][detail]
        msg = '{"ruleName":"%s","overLimit":true,"currentUsage":%d,"limitMax":%d,"expiresAt":"%s"}' % (
            rule, cur_usage, limit_max, _rfc3339(now_unix + int(rl_retry) if rl_retry is not None else window_end(now_unix, rule)))
    elif reason == abi.R_QUOTA:
        ns = tables.token_namespace[int(tables.qos_token[qos])]
        msg = ('{"Identifier":[{"Key":"namespace","Value":%s},{"Key":"quotaname","Value":%s},{"Key":"type","Value":"%s"}],'
               '"overLimit":true,"currentUsage":%d,"limitMax":%d}') % (
            _go_str(ns), _go_str(tables.qos_quota_name[qos]), tables.qos_quota_item_types[qos][detail], cur_usage, limit_max)
    elif reason == abi.R_QUOTA_CONFIG:
        msg = 'ArksQuota.arks.ai "%s" not found' % tables.qos_quota_name[qos]
    else:
        status, header, value, msg = 500, "x-error-rate-limit", "rate limit error", "rate limit error"
    return status, header, value, msg


def response_error_reply(reason: int, tables, qos: int, last_chunk: bytes):
    status, header = abi.REASON_HTTP.get(reason, (500, "x-error-response-unknown"))
    if reason in (abi.R_STREAMING, abi.R_RESPONSE_UNMARSHAL):
        msg = "error to unmarshal response"
    elif reason == abi.R_RESPONSE_UNKNOWN:
        msg = last_chunk.decode("utf-8", "surrogateescape") if last_chunk else "unknown response"
    elif reason == abi.R_QUOTA_CONFIG_RESP:
        msg = 'ArksQuota.arks.ai "%s" not found' % tables.qos_quota_name[qos]
    else:
        status, header, msg = 500, "x-error-response-unknown", "unknown response"
    return status, header, "true", msg


def error_body(message: str, status: int) -> bytes:
    """generateErrorMessage, util.go:66-77 (jsoniter ConfigFastest: no HTML escaping)"""
    return ('{"error":{"message":%s,"code":%d}}' % (json.dumps(message, ensure_ascii=False), status)).encode("utf-8", "surrogateescape")
