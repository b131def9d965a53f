"""Independent formulation of what the reference's handlers extract from a request / response / SSE chunk, built on
parsers that are NOT the oracle's: Python's `json` (tokenisation, validity, escape decoding) and openai-python's
`SSEDecoder` (the Stainless SSE decoder family openai-go's `packages/ssestream` belongs to). Only the struct-binding rules
of the Go code around those parsers are stated here (handle_request.go:87-93, handle_response.go:89-124):

  request   struct{Model string; Stream *bool; StreamOptions *struct{IncludeUsage *bool}} decoded by json-iterator:
            case-insensitive field match, last duplicate wins, null -> zero value / nil pointer, an allocated
            StreamOptions struct is reused by a later duplicate, a value of the wrong JSON type is an error
  response  struct{Model string; Usage openai.CompletionUsage}; Usage via apijson/gjson: exact keys, last duplicate wins,
            null leaves a field untouched
  sse       for each event: data prefix "[DONE]" ends the stream; invalid JSON or a top-level "error" key fails it;
            `if len(evt.Choices) == 0 { usage = evt.Usage }`

Every function returns None when a document is OUTSIDE the subset on which these independent parsers and the Go
libraries are known to agree (invalid UTF-8, lone surrogates, non-integer counters, id:/retry: lines, lone CR, ...);
the pin tests skip those and count how many documents took part. TEST INFRASTRUCTURE."""
import json
import re

I64 = (-(1 << 63), (1 << 63) - 1)


class _Reject(Exception):
    pass


def _no_const(name):
    raise ValueError("NaN / Infinity are not JSON")  # json.loads would accept them; RFC 8259 and both Go decoders do not


def loads_pairs(text: str):
    """RFC 8259 parse keeping member order and duplicates: objects come back as lists of (key, value) wrapped in Obj."""
    return json.loads(text, object_pairs_hook=Obj, parse_constant=_no_const)


class Obj(list):
    """a JSON object as its ordered (key, value) pairs"""


def _has_surrogate(s: str) -> bool:
    return any(0xD800 <= ord(c) <= 0xDFFF for c in s)


def _depth(v, d=0):
    if isinstance(v, Obj):
        return max([_depth(x, d + 1) for _, x in v] + [d + 1])
    if isinstance(v, list):
        return max([_depth(x, d + 1) for x in v] + [d + 1])
    return d


def _parse(body: bytes):
    """-> ('ok', value) | ('invalid', None) | None (outside the subset)"""
    try:
        text = body.decode("utf-8")
    except UnicodeDecodeError:
        return None
    if "\x00" in text:
        return None  # json-iterator stops at a NUL byte after the document (a quirk the oracle restates; not RFC)
    try:
        return "ok", loads_pairs(text)
    except RecursionError:
        return None
    except ValueError:
        return "invalid", None


def request_fields(body: bytes):
    """-> dict(err, model(bytes), stream, so_present, include_usage) with tri-states 0 nil / 1 false / 2 true, or None."""
    r = _parse(body)
    if r is None:
        return None
    if r[0] == "invalid":
        return None  # json-iterator is lenient in places (-01, null keys, ...): RFC-invalid input is outside the subset
    doc = r[1]
    if not isinstance(doc, Obj):
        # jsoniter's struct decoder accepts `null` at the top (zero struct) and rejects every other non-object
        return {"err": 0, "model": b"", "stream": 0, "so_present": 0, "include_usage": 0} if doc is None else {"err": 1}
    tri = lambda v: 0 if v is None else (2 if v else 1)
    model, stream, so = "", None, None
    try:
        for k, v in doc:
            kl = _fold(k)
            if kl is None:
                return None
            if kl == "model":
                if v is None:
                    model = ""
                elif isinstance(v, str):
                    if _has_surrogate(v):
                        return None
                    model = v
                else:
                    raise _Reject
            elif kl == "stream":
                if v is not None and not isinstance(v, bool):
                    raise _Reject
                stream = v
            elif kl == "stream_options":
                if v is None:
                    so = None
                elif isinstance(v, Obj):
                    if so is None:
                        so = {"iu": None}
                    for k2, v2 in v:
                        k2l = _fold(k2)
                        if k2l is None:
                            return None
                        if k2l == "include_usage":
                            if v2 is not None and not isinstance(v2, bool):
                                raise _Reject
                            so["iu"] = v2
                else:
                    raise _Reject
    except _Reject:
        return {"err": 1}
    return {"err": 0, "model": model.encode(), "stream": tri(stream), "so_present": int(so is not None),
            "include_usage": tri(so["iu"]) if so is not None else 0}


def _fold(k: str):
    """jsoniter readFieldHash lowers ASCII letters byte by byte; keys with non-ASCII or surrogates stay out of the subset
    only if they could matter (they cannot equal an ASCII field name, so they simply do not match)."""
    if _has_surrogate(k):
        return "\udc80"  # cannot match any field
    return "".join(chr(ord(c) + 32) if "A" <= c <= "Z" else c for c in k)


def _usage_into(v, usage):
    """apijson struct decode of openai.CompletionUsage over gjson's Map(): returns False if outside the subset"""
    if not isinstance(v, Obj):
        return v is None  # null: nothing decoded; any other non-object type is left to the oracle (unpinned)
    last = {}
    for k, x in v:
        last[k] = x
    for f, name in enumerate(("prompt_tokens", "completion_tokens", "total_tokens")):
        if name not in last:
            continue
        x = last[name]
        if x is None:
            continue
        if isinstance(x, bool):
            usage[f] = 1 if x else 0
        elif isinstance(x, int) and I64[0] <= x <= I64[1]:
            usage[f] = x
        else:
            return False  # floats, strings, containers, out-of-range integers: gjson specifics, outside the subset
    return True


INT64_MIN = I64[0]
_PLAIN_INT = re.compile(rb"-?[0-9]+")


def _wrap64(v: int) -> int:
    return (v + (1 << 63)) % (1 << 64) - (1 << 63)


def _gjson_parse_int(s: bytes) -> int:
    """gjson parseInt: `-?[0-9]+` read into an int64 that wraps; anything else is 0"""
    if not _PLAIN_INT.fullmatch(s):
        return 0
    return _wrap64(int(s))


def gjson_int(raw: bytes) -> int:
    """gjson Result.Int of a usage counter's raw JSON token (a number, or a string without escapes), stated with Python's
    int and float only. A plain integer is the wrapping int64 parse. Any other number is safeInt(ParseFloat(raw)) when
    |f| <= 2^53-1, else int64(f), which on amd64 is INT64_MIN outside [-2^63, 2^63) and for +-Inf. float() rounds
    correctly like ParseFloat; ParseFloat's exponent stops growing at 10000, which cannot matter for numbers of up to
    4 KiB of text, the domain this rule is stated for. A string is parseInt of its raw content."""
    if raw[:1] == b'"':
        return _gjson_parse_int(raw[1:-1])
    if _PLAIN_INT.fullmatch(raw):
        return _gjson_parse_int(raw)
    f = float(raw)
    if abs(f) <= (1 << 53) - 1:
        return int(f)
    if -(1 << 63) <= f < (1 << 63):
        return int(f)
    return INT64_MIN


def response_fields(body: bytes):
    """-> dict(err, model_len, usage[3]) or None"""
    r = _parse(body)
    if r is None:
        return None
    if r[0] == "invalid":
        return None
    doc = r[1]
    if not isinstance(doc, Obj):
        return {"err": 0, "model_len": 0, "usage": [0, 0, 0]} if doc is None else {"err": 1}
    model, usage = "", [0, 0, 0]
    for k, v in doc:
        kl = _fold(k)
        if kl == "model":
            if v is None:
                model = ""
            elif isinstance(v, str):
                if _has_surrogate(v):
                    return None
                model = v
            else:
                return {"err": 1}
        elif kl == "usage":
            if not _usage_into(v, usage):
                return None
    return {"err": 0, "model_len": len(model.encode()), "usage": usage}


def sse_split(chunk: bytes):
    """Events of one chunk by openai-python's SSEDecoder -> [(event type, data)] or None when the chunk is outside the
    subset on which that decoder and openai-go's agree: invalid UTF-8, a CR that is not part of CR LF, `id:` / `retry:`
    fields (openai-python keeps a sticky last-event-id that changes what it dispatches), lines of 64 KiB."""
    from openai._streaming import SSEDecoder
    try:
        chunk.decode("utf-8")
    except UnicodeDecodeError:
        return None
    if b"\r" in chunk.replace(b"\r\n", b"\n"):
        return None
    has_data, event_name = False, b""  # what openai-python holds when a blank line arrives
    lines = chunk.replace(b"\r\n", b"\n").split(b"\n")
    for li, line in enumerate(lines):
        if len(line) >= 65000:
            return None
        name = line.split(b":", 1)[0]
        if name in (b"id", b"retry"):
            return None
        if not line:
            # openai-go dispatches an event on EVERY blank line (an event without data then fails to unmarshal);
            # openai-python swallows a blank line when nothing is pending. Chunks with such a line are outside the subset.
            if not (has_data or event_name) and li < len(lines) - 1:
                return None
            has_data, event_name = False, b""
        elif name == b"data":
            has_data = True
        elif name == b"event":
            value = line.split(b":", 1)[1] if b":" in line else b""
            if value[:1] == b" ":
                value = value[1:]
            event_name = value  # openai-python tests the event NAME for truthiness, and a later `event` line REPLACES it
                                # (`event: message` then a bare `event` leaves nothing pending there; openai-go dispatches)
    # Go's bufio.Scanner delivers an unterminated last line as a token; openai-python's chunker does too
    return [(e.event or "", e.data) for e in SSEDecoder().iter_bytes(iter([chunk]))]


def sse_fields(chunk: bytes):
    """-> dict(err, usage[3]) or None: Stream.Next + the handler's loop (handle_response.go:113-124) over sse_split()"""
    evs = sse_split(chunk)
    if evs is None:
        return None
    usage, done = [0, 0, 0], False
    for typ, data in evs:
        if done:
            continue
        if data.startswith("[DONE]"):
            done = True
            continue
        if "\x00" in data:
            return None
        try:
            doc = loads_pairs(data)
        except RecursionError:
            return None
        except ValueError:
            return {"err": 1}
        if not isinstance(doc, Obj):
            return None  # apijson on a non-object event: unpinned
        keys = {}
        for k, v in doc:
            keys[k] = v
        if "error" in keys:
            return {"err": 1}
        if typ.startswith("thread."):
            usage = [0, 0, 0]  # the event is wrapped as {"event":..,"data":..}: no choices, zero usage
            continue
        ch = keys.get("choices")
        if isinstance(ch, list) and not isinstance(ch, Obj) and len(ch) > 0:
            continue
        u = [0, 0, 0]
        if "usage" in keys and not _usage_into(keys["usage"], u):
            return None
        usage = u
    return {"err": 0, "usage": usage}
