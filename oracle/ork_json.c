/*
 * ork_json.c — oracle: JSON / SSE decoding exactly as the reference's call sites use it.
 * TEST INFRASTRUCTURE ONLY (see arks_oracle.h).
 *
 * Call sites restated (reference tree):
 *   pkg/gateway/util.go:26-33              jsoniter.ConfigFastest.Unmarshal
 *   pkg/gateway/handle_request.go:87-104   request body  -> {model, stream, stream_options.include_usage}
 *   pkg/gateway/handle_response.go:89-93,157  response body -> {model, usage openai.CompletionUsage}
 *   pkg/gateway/handle_response.go:113-124 SSE chunk -> ssestream.Stream[openai.ChatCompletionChunk]
 *
 * The decoders themselves live in un-vendored modules (go.mod): github.com/json-iterator/go v1.1.12,
 * github.com/openai/openai-go v0.1.0-beta.3 (packages/ssestream, internal/apijson),
 * github.com/tidwall/gjson v1.14.4 and the standard library's encoding/json + bufio.Scanner.
 * Their algorithms are restated here function by function; names in comments are the upstream ones.
 * PARITY UNPINNED for this file (no upstream source or vectors in the reference tree).
 *
 * Deliberate, documented simplifications (DESIGN.md §4 "divergence list"):
 *   D1  numbers in *skipped* positions: jsoniter's trySkipNumber is restated exactly; when it defers to
 *       ReadFloat64/ReadBigFloat we validate the RFC 8259 number grammar instead of Go's ParseFloat
 *       (differs only for malformed numbers such as "+1", "1.", or magnitudes beyond float range).
 *   D2  usage counters written with a fraction/exponent are converted with strtod over the whole number +
 *       truncation (gjson Result.Int); out-of-int64-range conversions yield INT64_MIN (amd64 behaviour).
 *       strtod does not stop growing the exponent at 10000 as ParseFloat does: only numbers thousands of
 *       bytes long can tell the two apart.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "ork_internal.h"

/* =====================================================================================
 * jsoniter Iterator (iter.go, iter_str.go, iter_skip.go, iter_skip_strict.go, iter_object.go)
 * ===================================================================================== */
typedef struct {
  const uint8_t* b;
  size_t head, tail;
  int err;   /* a non-EOF error has been reported (iter.Error != nil && != io.EOF) */
  int eof;   /* iter.Error == io.EOF */
  int depth; /* incrementDepth / maxDepth = 10000 (iter.go) */
  size_t str_start; /* ReadString: first byte after the opening quote of the last string read (model span) */
} jit;

#define J_MAX_DEPTH 10000

static void j_report(jit* it) { it->err = 1; }

/* Iterator.nextToken */
static uint8_t j_next_token(jit* it) {
  while (it->head < it->tail) {
    uint8_t c = it->b[it->head++];
    if (c == ' ' || c == '\n' || c == '\t' || c == '\r') continue;
    return c;
  }
  if (!it->err) it->eof = 1;
  return 0;
}
/* Iterator.readByte */
static uint8_t j_read_byte(jit* it) {
  if (it->head == it->tail) {
    if (!it->err) it->eof = 1;
    return 0;
  }
  return it->b[it->head++];
}
/* Iterator.unreadByte: a no-op once any error (EOF included) is set */
static void j_unread(jit* it) {
  if (it->err || it->eof) return;
  it->head--;
}
static void j_skip_bytes(jit* it, const char* s) {
  for (; *s; s++) {
    if (j_read_byte(it) != (uint8_t)*s) {
      j_report(it);
      return;
    }
  }
}
static int j_inc_depth(jit* it) {
  it->depth++;
  if (it->depth <= J_MAX_DEPTH) return 1;
  j_report(it);
  return 0;
}
static void j_dec_depth(jit* it) { it->depth--; }

/* growable byte sink for decoded strings (NULL sink = discard) */
static void sink_put(ork_sink* s, uint8_t c) {
  if (!s) return;
  if (s->hash_on) { /* readFieldHash: lower-case ASCII, FNV-style 64-bit (iter_object.go) */
    if (c >= 'A' && c <= 'Z') c += 'a' - 'A';
    s->h ^= (uint64_t)c;
    s->h *= 0x1000193ull;
  } else if (s->len < s->cap) {
    s->buf[s->len] = c;
  }
  s->len++;
}
/* appendRune (iter_str.go): utf8.EncodeRune with surrogates / out of range -> U+FFFD */
static void sink_rune(ork_sink* s, uint32_t r) {
  if (r <= 0x7F) {
    sink_put(s, (uint8_t)r);
  } else if (r <= 0x7FF) {
    sink_put(s, 0xC0 | (uint8_t)(r >> 6));
    sink_put(s, 0x80 | (uint8_t)(r & 0x3F));
  } else {
    if (r > 0x10FFFF || (r >= 0xD800 && r <= 0xDFFF)) r = 0xFFFD;
    if (r <= 0xFFFF) {
      sink_put(s, 0xE0 | (uint8_t)(r >> 12));
      sink_put(s, 0x80 | (uint8_t)((r >> 6) & 0x3F));
      sink_put(s, 0x80 | (uint8_t)(r & 0x3F));
    } else {
      sink_put(s, 0xF0 | (uint8_t)(r >> 18));
      sink_put(s, 0x80 | (uint8_t)((r >> 12) & 0x3F));
      sink_put(s, 0x80 | (uint8_t)((r >> 6) & 0x3F));
      sink_put(s, 0x80 | (uint8_t)(r & 0x3F));
    }
  }
}

/* Iterator.readU4 */
static uint32_t j_read_u4(jit* it) {
  uint32_t r = 0;
  for (int i = 0; i < 4; i++) {
    uint8_t c = j_read_byte(it);
    if (it->err || it->eof) return r;
    if (c >= '0' && c <= '9')
      r = r * 16 + (c - '0');
    else if (c >= 'a' && c <= 'f')
      r = r * 16 + (c - 'a' + 10);
    else if (c >= 'A' && c <= 'F')
      r = r * 16 + (c - 'A' + 10);
    else {
      j_report(it);
      return r;
    }
  }
  return r;
}
static int is_surrogate(uint32_t r) { return r >= 0xD800 && r <= 0xDFFF; }
/* utf16.DecodeRune */
static uint32_t utf16_decode(uint32_t r1, uint32_t r2) {
  if (r1 >= 0xD800 && r1 < 0xDC00 && r2 >= 0xDC00 && r2 < 0xE000)
    return ((r1 - 0xD800) << 10 | (r2 - 0xDC00)) + 0x10000;
  return 0xFFFD;
}
/* Iterator.readEscapedChar */
static void j_read_escaped(jit* it, uint8_t c, ork_sink* s) {
  for (;;) { /* the tail call `return iter.readEscapedChar(c, str)` becomes this loop */
    switch (c) {
      case 'u': {
        uint32_t r = j_read_u4(it);
        if (is_surrogate(r)) {
          c = j_read_byte(it);
          if (it->err || it->eof) return;
          if (c != '\\') {
            j_unread(it);
            sink_rune(s, r);
            return;
          }
          c = j_read_byte(it);
          if (it->err || it->eof) return;
          if (c != 'u') {
            sink_rune(s, r);
            continue; /* readEscapedChar(c, str) */
          }
          uint32_t r2 = j_read_u4(it);
          if (it->err || it->eof) return;
          uint32_t comb = utf16_decode(r, r2);
          if (comb == 0xFFFD) {
            sink_rune(s, r);
            sink_rune(s, r2);
          } else {
            sink_rune(s, comb);
          }
        } else {
          sink_rune(s, r);
        }
        return;
      }
      case '"': sink_put(s, '"'); return;
      case '\\': sink_put(s, '\\'); return;
      case '/': sink_put(s, '/'); return;
      case 'b': sink_put(s, '\b'); return;
      case 'f': sink_put(s, '\f'); return;
      case 'n': sink_put(s, '\n'); return;
      case 'r': sink_put(s, '\r'); return;
      case 't': sink_put(s, '\t'); return;
      default: j_report(it); return;
    }
  }
}
/* Iterator.readStringSlowPath: no control-character check on this path */
static void j_read_string_slow(jit* it, ork_sink* s) {
  while (!it->err && !it->eof) {
    uint8_t c = j_read_byte(it);
    if (it->eof) break;
    if (c == '"') return;
    if (c == '\\') {
      c = j_read_byte(it);
      j_read_escaped(it, c, s);
    } else {
      sink_put(s, c);
    }
  }
  j_report(it); /* "unexpected end of input" */
}
/* Iterator.ReadString: returns 1 if the value was the literal null */
static int j_read_string(jit* it, ork_sink* s) {
  uint8_t c = j_next_token(it);
  if (c == '"') {
    it->str_start = it->head;
    for (size_t i = it->head; i < it->tail; i++) {
      c = it->b[i];
      if (c == '"') {
        for (size_t k = it->head; k < i; k++) sink_put(s, it->b[k]);
        it->head = i + 1;
        return 0;
      } else if (c == '\\') {
        break;
      } else if (c < ' ') {
        j_report(it); /* invalid control character */
        return 0;
      }
    }
    j_read_string_slow(it, s);
    return 0;
  } else if (c == 'n') {
    j_skip_bytes(it, "ull");
    return 1;
  }
  j_report(it);
  return 0;
}

static void j_skip(jit* it);

/* RFC 8259 number grammar from b[pos]; returns end or (size_t)-1. (divergence D1) */
static size_t rfc_number_end(const uint8_t* b, size_t pos, size_t tail) {
  size_t i = pos;
  if (i < tail && b[i] == '-') i++;
  if (i >= tail) return (size_t)-1;
  if (b[i] == '0') {
    i++;
  } else if (b[i] >= '1' && b[i] <= '9') {
    while (i < tail && b[i] >= '0' && b[i] <= '9') i++;
  } else {
    return (size_t)-1;
  }
  if (i < tail && b[i] == '.') {
    i++;
    if (i >= tail || b[i] < '0' || b[i] > '9') return (size_t)-1;
    while (i < tail && b[i] >= '0' && b[i] <= '9') i++;
  }
  if (i < tail && (b[i] == 'e' || b[i] == 'E')) {
    i++;
    if (i < tail && (b[i] == '+' || b[i] == '-')) i++;
    if (i >= tail || b[i] < '0' || b[i] > '9') return (size_t)-1;
    while (i < tail && b[i] >= '0' && b[i] <= '9') i++;
  }
  /* readNumberAsString would keep eating number characters and then fail to parse */
  if (i < tail) {
    uint8_t c = b[i];
    if ((c >= '0' && c <= '9') || c == '+' || c == '-' || c == '.' || c == 'e' || c == 'E') return (size_t)-1;
  }
  return i;
}
static void j_number_fallback(jit* it, size_t start) {
  size_t e = rfc_number_end(it->b, start, it->tail);
  if (e == (size_t)-1) {
    j_report(it);
    return;
  }
  it->head = e;
}
/* Iterator.skipNumber / trySkipNumber (iter_skip_strict.go); `start` = index of the first char */
static void j_skip_number(jit* it, size_t start) {
  int dot = 0;
  for (size_t i = it->head; i < it->tail; i++) {
    uint8_t c = it->b[i];
    if (c >= '0' && c <= '9') continue;
    if (c == '.') {
      if (dot) {
        j_report(it);
        return;
      }
      if (i + 1 == it->tail) {
        j_number_fallback(it, start);
        return;
      }
      c = it->b[i + 1];
      if (c < '0' || c > '9') {
        j_report(it);
        return;
      }
      dot = 1;
      continue;
    }
    if (c == ',' || c == ']' || c == '}' || c == ' ' || c == '\t' || c == '\n' || c == '\r') {
      if (it->head == i) {
        j_number_fallback(it, start);
        return;
      }
      it->head = i;
      return;
    }
    j_number_fallback(it, start);
    return;
  }
  j_number_fallback(it, start);
}
/* Iterator.skipString / trySkipString */
static void j_skip_string(jit* it) {
  for (size_t i = it->head; i < it->tail; i++) {
    uint8_t c = it->b[i];
    if (c == '"') {
      it->head = i + 1;
      return;
    } else if (c == '\\') {
      break;
    } else if (c < ' ') {
      j_report(it);
      return;
    }
  }
  /* unreadByte(); ReadString() == slow path from the start of the string */
  j_read_string_slow(it, NULL);
}
/* Iterator.skipObject == ReadObjectCB(func{ Skip() }) (iter_object.go) */
static void j_skip_object(jit* it) {
  /* '{' already consumed */
  if (!j_inc_depth(it)) return;
  uint8_t c = j_next_token(it);
  if (c == '"') {
    j_unread(it);
    j_read_string(it, NULL);
    c = j_next_token(it);
    if (c != ':') j_report(it);
    if (it->err) return;
    j_skip(it);
    if (it->err) return;
    c = j_next_token(it);
    while (c == ',') {
      j_read_string(it, NULL); /* NB: accepts the literal null as a key, like upstream */
      c = j_next_token(it);
      if (c != ':') j_report(it);
      if (it->err) return;
      j_skip(it);
      if (it->err) return;
      c = j_next_token(it);
    }
    if (c != '}') {
      j_report(it);
      return;
    }
    j_dec_depth(it);
    return;
  }
  if (c == '}') {
    j_dec_depth(it);
    return;
  }
  j_report(it);
}
/* Iterator.skipArray == ReadArrayCB(func{ Skip() }) (iter_array.go) */
static void j_skip_array(jit* it) {
  if (!j_inc_depth(it)) return;
  uint8_t c = j_next_token(it);
  if (c != ']') {
    j_unread(it);
    j_skip(it);
    if (it->err) return;
    c = j_next_token(it);
    while (c == ',') {
      j_skip(it);
      if (it->err) return;
      c = j_next_token(it);
    }
    if (c != ']') {
      j_report(it);
      return;
    }
  }
  j_dec_depth(it);
}
/* Iterator.Skip (iter_skip.go) */
static void j_skip(jit* it) {
  uint8_t c = j_next_token(it);
  switch (c) {
    case '"': j_skip_string(it); break;
    case 'n': j_skip_bytes(it, "ull"); break;
    case 't': j_skip_bytes(it, "rue"); break;
    case 'f': j_skip_bytes(it, "alse"); break;
    case '0': j_number_fallback(it, it->head - 1); break; /* unreadByte(); ReadFloat32() */
    case '-': case '1': case '2': case '3': case '4': case '5': case '6': case '7': case '8': case '9':
      j_skip_number(it, it->head - 1);
      break;
    case '[': j_skip_array(it); break;
    case '{': j_skip_object(it); break;
    default: j_report(it); break;
  }
}

/* Iterator.readFieldHash (iter_object.go), caseSensitive == false for ConfigFastest */
static int64_t j_read_field_hash(jit* it) {
  uint64_t h = 0x811c9dc5ull;
  uint8_t c = j_next_token(it);
  if (c != '"') {
    j_report(it);
    return 0;
  }
  for (size_t i = it->head; i < it->tail; i++) {
    uint8_t b = it->b[i];
    if (b == '\\') {
      it->head = i;
      /* readStringSlowPath() from the backslash on; every decoded byte is lower-cased and hashed */
      ork_sink s = {NULL, 0, 0, 1, h};
      j_read_string_slow(it, &s);
      h = s.h;
      c = j_next_token(it);
      if (c != ':') {
        j_report(it);
        return 0;
      }
      return (int64_t)h;
    }
    if (b == '"') {
      it->head = i + 1;
      c = j_next_token(it);
      if (c != ':') {
        j_report(it);
        return 0;
      }
      return (int64_t)h;
    }
    if (b >= 'A' && b <= 'Z') b += 'a' - 'A';
    h ^= (uint64_t)b;
    h *= 0x1000193ull;
  }
  it->head = it->tail;
  if (!it->err) it->eof = 1;
  j_report(it); /* incomplete field name */
  return 0;
}
static int64_t field_hash_of(const char* s) {
  uint64_t h = 0x811c9dc5ull;
  for (; *s; s++) {
    h ^= (uint64_t)(uint8_t)*s;
    h *= 0x1000193ull;
  }
  return (int64_t)h;
}
/* Iterator.readObjectStart: 1 = fields follow, 0 = `{}` or null or error */
static int j_read_object_start(jit* it) {
  uint8_t c = j_next_token(it);
  if (c == '{') {
    c = j_next_token(it);
    if (c == '}') return 0;
    j_unread(it);
    return 1;
  } else if (c == 'n') {
    j_skip_bytes(it, "ull");
    return 0;
  }
  j_report(it);
  return 0;
}
/* Iterator.isObjectEnd */
static int j_is_object_end(jit* it) {
  uint8_t c = j_next_token(it);
  if (c == ',') return 0;
  if (c == '}') return 1;
  j_report(it);
  return 1;
}
/* Iterator.ReadNil */
static int j_read_nil(jit* it) {
  uint8_t c = j_next_token(it);
  if (c == 'n') {
    j_skip_bytes(it, "ull");
    return 1;
  }
  j_unread(it);
  return 0;
}
/* Iterator.ReadBool */
static int j_read_bool(jit* it) {
  uint8_t c = j_next_token(it);
  if (c == 't') {
    j_skip_bytes(it, "rue");
    return 1;
  }
  if (c == 'f') {
    j_skip_bytes(it, "alse");
    return 0;
  }
  j_report(it);
  return 0;
}
/* OptionalDecoder{boolCodec}: tri-state 0 nil, 1 false, 2 true */
static void j_decode_opt_bool(jit* it, int* v) {
  if (j_read_nil(it)) {
    *v = 0;
  } else {
    int b = j_read_bool(it);
    *v = b ? 2 : 1;
  }
}
/* frozenConfig.Unmarshal tail: only whitespace (or a NUL byte, upstream quirk) may follow */
static int j_finish(jit* it) {
  if (it->err) return 1;
  uint8_t c = j_next_token(it);
  if (c == 0) return it->err ? 1 : 0;
  return 1; /* "there are bytes left after unmarshal" */
}

/* ---- request body: struct{Model string; Stream *bool; StreamOptions *struct{IncludeUsage *bool}} ----
 * threeFieldsStructDecoder + OptionalDecoder + oneFieldStructDecoder (reflect_struct_decoder.go) */
int ork_json_request(const uint8_t* body, size_t len, ork_sink* model, int* stream, int* so_present,
                     int* include_usage, uint32_t span[2]) {
  static int64_t H_MODEL, H_STREAM, H_SO, H_IU;
  if (!H_MODEL) {
    H_MODEL = field_hash_of("model");
    H_STREAM = field_hash_of("stream");
    H_SO = field_hash_of("stream_options");
    H_IU = field_hash_of("include_usage");
  }
  jit it = {body, 0, len, 0, 0, 0, 0};
  *stream = 0;
  *so_present = 0;
  *include_usage = 0;
  if (model) model->len = 0;
  uint32_t sp[2] = {0, 0};
  if (j_read_object_start(&it) && j_inc_depth(&it)) {
    for (;;) {
      int64_t h = j_read_field_hash(&it);
      if (it.err) break;
      if (h == H_MODEL) {
        if (model) model->len = 0;
        sp[0] = sp[1] = 0;
        if (!j_read_string(&it, model) && !it.err) { /* null -> "" */
          /* raw span between the quotes (the host slices its copy of the body for the x-error-* header values) */
          size_t e = it.head - 1;
          sp[0] = (uint32_t)it.str_start;
          sp[1] = (uint32_t)(e - it.str_start);
          for (size_t k = it.str_start; k < e; k++)
            if (body[k] == '\\') sp[1] |= 0x80000000u;
          if ((sp[1] & 0x7fffffffu) == 0) sp[0] = sp[1] = 0;
        }
      } else if (h == H_STREAM) {
        j_decode_opt_bool(&it, stream);
      } else if (h == H_SO) {
        if (j_read_nil(&it)) {
          *so_present = 0;
          *include_usage = 0;
        } else {
          /* pointer reused when already allocated: fields of an earlier occurrence persist */
          *so_present = 1;
          if (j_read_object_start(&it) && j_inc_depth(&it)) {
            for (;;) {
              int64_t h2 = j_read_field_hash(&it);
              if (it.err) break;
              if (h2 == H_IU)
                j_decode_opt_bool(&it, include_usage);
              else
                j_skip(&it);
              if (it.err) break;
              if (j_is_object_end(&it)) break;
            }
            j_dec_depth(&it);
          }
        }
      } else {
        j_skip(&it);
      }
      if (it.err) break;
      if (j_is_object_end(&it)) break;
    }
    j_dec_depth(&it);
  }
  int rc = j_finish(&it);
  if (span) {
    span[0] = rc ? 0 : sp[0];
    span[1] = rc ? 0 : sp[1];
  }
  return rc;
}

/* =====================================================================================
 * gjson v1.14.4 Result.Int + apijson struct decode of openai.CompletionUsage, on a JSON value that
 * the caller has already validated (jsoniter strict skip, or encoding/json checkValid).
 * ===================================================================================== */
static size_t v_skip_ws(const uint8_t* b, size_t i, size_t n) {
  while (i < n && (b[i] == ' ' || b[i] == '\t' || b[i] == '\n' || b[i] == '\r')) i++;
  return i;
}
/* end of the string whose opening quote is at b[i] (valid JSON assumed): index after closing quote */
static size_t v_string_end(const uint8_t* b, size_t i, size_t n) {
  i++;
  while (i < n) {
    if (b[i] == '\\')
      i += 2;
    else if (b[i] == '"')
      return i + 1;
    else
      i++;
  }
  return n;
}
/* end of any value starting at b[i] */
static size_t v_value_end(const uint8_t* b, size_t i, size_t n) {
  if (i >= n) return n;
  uint8_t c = b[i];
  if (c == '"') return v_string_end(b, i, n);
  if (c == '{' || c == '[') {
    int depth = 0;
    while (i < n) {
      c = b[i];
      if (c == '"') {
        i = v_string_end(b, i, n);
        continue;
      }
      if (c == '{' || c == '[') depth++;
      if (c == '}' || c == ']') {
        depth--;
        if (depth == 0) return i + 1;
      }
      i++;
    }
    return n;
  }
  while (i < n && b[i] != ',' && b[i] != '}' && b[i] != ']' && b[i] != ' ' && b[i] != '\t' && b[i] != '\n' &&
         b[i] != '\r')
    i++;
  return i;
}
/* decoded key/string equals ASCII literal? raw = bytes between the quotes */
static int v_str_equals(const uint8_t* raw, size_t n, const char* lit) {
  size_t L = strlen(lit), k = 0, i = 0;
  while (i < n) {
    uint32_t cp;
    if (raw[i] == '\\') {
      if (i + 1 >= n) return 0;
      uint8_t e = raw[i + 1];
      i += 2;
      switch (e) {
        case '"': cp = '"'; break;
        case '\\': cp = '\\'; break;
        case '/': cp = '/'; break;
        case 'b': cp = '\b'; break;
        case 'f': cp = '\f'; break;
        case 'n': cp = '\n'; break;
        case 'r': cp = '\r'; break;
        case 't': cp = '\t'; break;
        case 'u': {
          if (i + 4 > n) return 0;
          cp = 0;
          for (int q = 0; q < 4; q++) {
            uint8_t c = raw[i + q];
            cp = cp * 16 + (c <= '9' ? c - '0' : (c | 0x20) - 'a' + 10);
          }
          i += 4;
          break;
        }
        default: return 0;
      }
      if (cp >= 0x80) return 0; /* cannot equal an ASCII literal */
    } else {
      cp = raw[i++];
    }
    if (k >= L || (uint8_t)lit[k] != cp) return 0;
    k++;
  }
  return k == L;
}
/* gjson parseInt */
static int gj_parse_int(const uint8_t* s, size_t n, int64_t* out) {
  size_t i = 0;
  int sign = 0;
  uint64_t v = 0;
  if (n > 0 && s[0] == '-') {
    sign = 1;
    i++;
  }
  if (i == n) return 0;
  for (; i < n; i++) {
    if (s[i] >= '0' && s[i] <= '9')
      v = v * 10 + (uint64_t)(s[i] - '0'); /* wraps like Go int64 */
    else
      return 0;
  }
  *out = sign ? (int64_t)(0 - v) : (int64_t)v;
  return 1;
}
/* gjson Result.Int() for the value at b[i..e) */
static int64_t gj_int(const uint8_t* b, size_t i, size_t e) {
  uint8_t c = b[i];
  int64_t out = 0;
  if (c == 't') return 1; /* True */
  if (c == '"') {         /* String: parseInt(t.Str); strings with escapes cannot be all digits */
    gj_parse_int(b + i + 1, e - i - 2, &out);
    return out;
  }
  if (c == '-' || (c >= '0' && c <= '9')) { /* Number */
    int plain = 1;
    for (size_t k = i; k < e; k++)
      if (!((b[k] >= '0' && b[k] <= '9') || (k == i && b[k] == '-'))) plain = 0;
    if (plain) {
      /* safeInt(float64) for |v| <= 2^53-1 and parseInt(raw) beyond agree with a wrapping parse */
      gj_parse_int(b + i, e - i, &out);
      return out;
    }
    /* ParseFloat reads the whole number: strtod is correctly rounded too, given all of it */
    char buf[64];
    char* tmp = e - i < sizeof buf ? buf : (char*)malloc(e - i + 1);
    if (!tmp) abort();
    memcpy(tmp, b + i, e - i);
    tmp[e - i] = 0;
    double f = strtod(tmp, NULL);
    if (tmp != buf) free(tmp);
    if (f >= -9007199254740991.0 && f <= 9007199254740991.0) return (int64_t)f;
    if (f >= -9223372036854775808.0 && f < 9223372036854775808.0) return (int64_t)f;
    return INT64_MIN; /* int64(f) on amd64, +-Inf included */
  }
  return 0; /* False, Null (never reached: nulls are skipped by apijson), JSON */
}
/* apijson newStructTypeDecoder on openai.CompletionUsage: node.Map() (last duplicate wins), null and
 * unknown keys skipped; decoding into an existing struct keeps fields that are absent. */
void ork_usage_from_value(const uint8_t* b, size_t i, size_t e, int64_t usage[3]) {
  static const char* K[3] = {"prompt_tokens", "completion_tokens", "total_tokens"};
  if (i >= e || b[i] != '{') return; /* Map() of a non-object is empty */
  size_t vi[3] = {0, 0, 0}, ve[3] = {0, 0, 0};
  int have[3] = {0, 0, 0};
  size_t p = v_skip_ws(b, i + 1, e);
  while (p < e && b[p] != '}') {
    if (b[p] != '"') break; /* tolerate jsoniter's null keys: stop scanning (unpinned corner) */
    size_t ke = v_string_end(b, p, e);
    size_t q = v_skip_ws(b, ke, e);
    if (q < e && b[q] == ':') q++;
    q = v_skip_ws(b, q, e);
    size_t qe = v_value_end(b, q, e);
    for (int f = 0; f < 3; f++)
      if (v_str_equals(b + p + 1, ke - p - 2, K[f])) {
        have[f] = 1;
        vi[f] = q;
        ve[f] = qe;
      }
    p = v_skip_ws(b, qe, e);
    if (p < e && b[p] == ',') p = v_skip_ws(b, p + 1, e);
  }
  for (int f = 0; f < 3; f++)
    if (have[f] && vi[f] < ve[f] && b[vi[f]] != 'n') usage[f] = gj_int(b, vi[f], ve[f]);
}

/* ---- non-stream response: struct{Model string; Usage openai.CompletionUsage} (twoFieldsStructDecoder);
 * Usage implements json.Unmarshaler -> unmarshalerDecoder: SkipAndReturnBytes + UnmarshalJSON ---- */
int ork_json_response(const uint8_t* body, size_t len, ork_sink* model, int64_t usage[3]) {
  static int64_t H_MODEL, H_USAGE;
  if (!H_MODEL) {
    H_MODEL = field_hash_of("model");
    H_USAGE = field_hash_of("usage");
  }
  jit it = {body, 0, len, 0, 0, 0, 0};
  usage[0] = usage[1] = usage[2] = 0;
  if (model) model->len = 0;
  if (j_read_object_start(&it) && j_inc_depth(&it)) {
    for (;;) {
      int64_t h = j_read_field_hash(&it);
      if (it.err) break;
      if (h == H_MODEL) {
        if (model) model->len = 0;
        j_read_string(&it, model);
      } else if (h == H_USAGE) {
        j_next_token(&it);
        j_unread(&it);
        size_t s = it.head;
        j_skip(&it);
        if (!it.err) ork_usage_from_value(body, s, it.head, usage);
      } else {
        j_skip(&it);
      }
      if (it.err) break;
      if (j_is_object_end(&it)) break;
    }
    j_dec_depth(&it);
  }
  return j_finish(&it);
}

/* =====================================================================================
 * encoding/json checkValid (scanner.go): strict RFC 8259, max nesting 10000
 * ===================================================================================== */
static size_t e_value(const uint8_t* b, size_t i, size_t n, int depth);
static size_t e_ws(const uint8_t* b, size_t i, size_t n) { return v_skip_ws(b, i, n); }
#define E_BAD ((size_t)-1)
static size_t e_string(const uint8_t* b, size_t i, size_t n) {
  i++;
  while (i < n) {
    uint8_t c = b[i];
    if (c == '"') return i + 1;
    if (c < 0x20) return E_BAD;
    if (c == '\\') {
      if (i + 1 >= n) return E_BAD;
      uint8_t e = b[i + 1];
      if (e == 'u') {
        if (i + 6 > n) return E_BAD;
        for (int q = 2; q < 6; q++) {
          uint8_t h = b[i + q];
          if (!((h >= '0' && h <= '9') || (h >= 'a' && h <= 'f') || (h >= 'A' && h <= 'F'))) return E_BAD;
        }
        i += 6;
      } else if (e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't') {
        i += 2;
      } else {
        return E_BAD;
      }
    } else {
      i++;
    }
  }
  return E_BAD;
}
static size_t e_lit(const uint8_t* b, size_t i, size_t n, const char* s) {
  size_t L = strlen(s);
  if (i + L > n || memcmp(b + i, s, L) != 0) return E_BAD;
  return i + L;
}
static size_t e_number(const uint8_t* b, size_t i, size_t n) {
  size_t s = i;
  if (i < n && b[i] == '-') i++;
  if (i >= n) return E_BAD;
  if (b[i] == '0')
    i++;
  else if (b[i] >= '1' && b[i] <= '9')
    while (i < n && b[i] >= '0' && b[i] <= '9') i++;
  else
    return E_BAD;
  if (i < n && b[i] == '.') {
    i++;
    if (i >= n || b[i] < '0' || b[i] > '9') return E_BAD;
    while (i < n && b[i] >= '0' && b[i] <= '9') i++;
  }
  if (i < n && (b[i] == 'e' || b[i] == 'E')) {
    i++;
    if (i < n && (b[i] == '+' || b[i] == '-')) i++;
    if (i >= n || b[i] < '0' || b[i] > '9') return E_BAD;
    while (i < n && b[i] >= '0' && b[i] <= '9') i++;
  }
  (void)s;
  return i;
}
static size_t e_value(const uint8_t* b, size_t i, size_t n, int depth) {
  i = e_ws(b, i, n);
  if (i >= n) return E_BAD;
  uint8_t c = b[i];
  if (c == '"') return e_string(b, i, n);
  if (c == 't') return e_lit(b, i, n, "true");
  if (c == 'f') return e_lit(b, i, n, "false");
  if (c == 'n') return e_lit(b, i, n, "null");
  if (c == '-' || (c >= '0' && c <= '9')) return e_number(b, i, n);
  if (c == '{') {
    if (depth + 1 > 10000) return E_BAD;
    i = e_ws(b, i + 1, n);
    if (i < n && b[i] == '}') return i + 1;
    for (;;) {
      i = e_ws(b, i, n);
      if (i >= n || b[i] != '"') return E_BAD;
      i = e_string(b, i, n);
      if (i == E_BAD) return E_BAD;
      i = e_ws(b, i, n);
      if (i >= n || b[i] != ':') return E_BAD;
      i = e_value(b, i + 1, n, depth + 1);
      if (i == E_BAD) return E_BAD;
      i = e_ws(b, i, n);
      if (i >= n) return E_BAD;
      if (b[i] == ',') {
        i++;
        continue;
      }
      if (b[i] == '}') return i + 1;
      return E_BAD;
    }
  }
  if (c == '[') {
    if (depth + 1 > 10000) return E_BAD;
    i = e_ws(b, i + 1, n);
    if (i < n && b[i] == ']') return i + 1;
    for (;;) {
      i = e_value(b, i, n, depth + 1);
      if (i == E_BAD) return E_BAD;
      i = e_ws(b, i, n);
      if (i >= n) return E_BAD;
      if (b[i] == ',') {
        i++;
        continue;
      }
      if (b[i] == ']') return i + 1;
      return E_BAD;
    }
  }
  return E_BAD;
}
/* checkValid: exactly one value surrounded by whitespace */
static int e_valid(const uint8_t* b, size_t n) {
  size_t i = e_value(b, 0, n, 0);
  if (i == E_BAD) return 0;
  i = e_ws(b, i, n);
  return i == n;
}

/* gjson.GetBytes(data, "error").Exists(): gjson is lenient; on invalid JSON either this or
 * json.Unmarshal fails and both paths end in the same 500, so existence only matters on valid JSON:
 * top-level object has a member whose (unescaped) key is "error". */
static int has_toplevel_key(const uint8_t* b, size_t n, const char* key, size_t* vi, size_t* ve) {
  size_t i = v_skip_ws(b, 0, n);
  int found = 0;
  if (i >= n || b[i] != '{') return 0;
  size_t p = v_skip_ws(b, i + 1, n);
  while (p < n && b[p] == '"') {
    size_t ke = v_string_end(b, p, n);
    size_t q = v_skip_ws(b, ke, n);
    if (q < n && b[q] == ':') q++;
    q = v_skip_ws(b, q, n);
    size_t qe = v_value_end(b, q, n);
    if (v_str_equals(b + p + 1, ke - p - 2, key)) {
      found = 1;
      if (vi) *vi = q;
      if (ve) *ve = qe; /* keep scanning: Map() semantics, last duplicate wins */
    }
    p = v_skip_ws(b, qe, n);
    if (p < n && b[p] == ',') p = v_skip_ws(b, p + 1, n);
  }
  return found;
}

/* one dispatched SSE event -> Stream.Next body (ssestream.go). returns 1 on stream error.
 * *is_chunk = 1 when an event value was produced (streaming.Current()). */
static int sse_event(const uint8_t* type, size_t type_len, const uint8_t* data, size_t data_len, int* done,
                     int64_t usage[3]) {
  if (*done) return 0;
  if (data_len >= 6 && memcmp(data, "[DONE]", 6) == 0) {
    *done = 1;
    return 0;
  }
  int valid = e_valid(data, data_len);
  /* error-key probe happens first upstream, but on invalid JSON both outcomes are the same 500 */
  if (!valid) return 1;
  if (has_toplevel_key(data, data_len, "error", NULL, NULL)) return 1;
  int wrapped = type_len >= 7 && memcmp(type, "thread.", 7) == 0;
  int64_t u[3] = {0, 0, 0};
  int n_choices = 0;
  if (!wrapped) {
    size_t vi, ve;
    if (has_toplevel_key(data, data_len, "choices", &vi, &ve)) {
      /* newArrayTypeDecoder: non-arrays fail and leave the slice nil */
      if (data[vi] == '[') {
        size_t p = v_skip_ws(data, vi + 1, ve);
        if (p < ve && data[p] != ']') n_choices = 1;
      }
    }
    if (has_toplevel_key(data, data_len, "usage", &vi, &ve)) {
      if (data[vi] != 'n') ork_usage_from_value(data, vi, ve, u);
    }
  }
  if (n_choices == 0) { /* handle_response.go:119-123: `if len(evt.Choices) == 0 { usage = evt.Usage }` */
    usage[0] = u[0];
    usage[1] = u[1];
    usage[2] = u[2];
  }
  return 0;
}

/* eventStreamDecoder.Next over bufio.Scanner(ScanLines) (ssestream.go); 64 KiB line limit.
 * on_event(ctx, type, type_len, data, data_len, n_data_lines) is called for every dispatched event, in order;
 * a non-zero return stops the scan with rc 1. */
typedef int (*sse_event_fn)(void* ctx, const uint8_t* type, size_t type_len, const uint8_t* data, size_t data_len,
                            uint32_t n_data_lines);
static int sse_scan(const uint8_t* body, size_t len, sse_event_fn on_event, void* ctx) {
  uint8_t* data = (uint8_t*)malloc(len + 16 + len / 2);
  size_t data_len = 0;
  uint32_t n_lines = 0;
  const uint8_t* ev = NULL;
  size_t ev_len = 0;
  int rc = 0;
  size_t pos = 0;
  while (pos < len) {
    size_t e = pos;
    while (e < len && body[e] != '\n') e++;
    size_t line_len = e - pos; /* before dropCR */
    if (line_len >= 65536) {   /* bufio.ErrTooLong -> decoder.Err() -> stream error */
      rc = 1;
      break;
    }
    const uint8_t* txt = body + pos;
    size_t n = line_len;
    if (n > 0 && txt[n - 1] == '\r') n--;
    pos = e < len ? e + 1 : len;
    if (n == 0) {
      if (e >= len && line_len == 0) break; /* no trailing empty token at EOF */
      /* dispatch */
      if (on_event(ctx, ev, ev_len, data, data_len, n_lines)) {
        rc = 1;
        break;
      }
      data_len = 0;
      n_lines = 0;
      ev = NULL;
      ev_len = 0;
      continue;
    }
    size_t colon = 0;
    while (colon < n && txt[colon] != ':') colon++;
    const uint8_t* val = colon < n ? txt + colon + 1 : txt + n;
    size_t vlen = colon < n ? n - colon - 1 : 0;
    if (vlen > 0 && val[0] == ' ') {
      val++;
      vlen--;
    }
    if (colon == 0) continue; /* comment (or line starting with ':') */
    if (colon == 5 && memcmp(txt, "event", 5) == 0) {
      ev = val;
      ev_len = vlen;
    } else if (colon == 4 && memcmp(txt, "data", 4) == 0) {
      memcpy(data + data_len, val, vlen);
      data_len += vlen;
      data[data_len++] = '\n';
      n_lines++;
    }
  }
  free(data);
  return rc;
}

struct sse_usage_ctx {
  int done;
  int64_t* usage;
};
static int sse_usage_event(void* ctx, const uint8_t* type, size_t type_len, const uint8_t* data, size_t data_len,
                           uint32_t n_lines) {
  struct sse_usage_ctx* c = (struct sse_usage_ctx*)ctx;
  (void)n_lines;
  return sse_event(type, type_len, data, data_len, &c->done, c->usage);
}
int ork_sse_chunk(const uint8_t* body, size_t len, int64_t usage[3]) {
  usage[0] = usage[1] = usage[2] = 0;
  struct sse_usage_ctx c = {0, usage};
  return sse_scan(body, len, sse_usage_event, &c);
}

/* test hook (tests/test_decoder_pins.py): the events the decoder dispatches for a chunk, serialised into `out` as
 * records {u32 type_len, u32 data_len, u32 n_data_lines, type bytes, data bytes}. Returns the number of events, or
 * -1 on a scanner error (line too long), -2 when `out` is too small. */
struct sse_dump_ctx {
  uint8_t* out;
  size_t cap, used;
  int n, overflow;
};
static int sse_dump_event(void* ctx, const uint8_t* type, size_t type_len, const uint8_t* data, size_t data_len,
                          uint32_t n_lines) {
  struct sse_dump_ctx* c = (struct sse_dump_ctx*)ctx;
  if (c->used + 12 + type_len + data_len > c->cap) {
    c->overflow = 1;
    return 1;
  }
  uint32_t h[3] = {(uint32_t)type_len, (uint32_t)data_len, n_lines};
  memcpy(c->out + c->used, h, 12);
  if (type_len) memcpy(c->out + c->used + 12, type, type_len);
  if (data_len) memcpy(c->out + c->used + 12 + type_len, data, data_len);
  c->used += 12 + type_len + data_len;
  c->n++;
  return 0;
}
int ork_sse_events(const uint8_t* body, size_t len, uint8_t* out, size_t cap, size_t* used) {
  struct sse_dump_ctx c = {out, cap, 0, 0, 0};
  int rc = sse_scan(body, len, sse_dump_event, &c);
  if (used) *used = c.used;
  if (c.overflow) return -2;
  return rc ? -1 : c.n;
}
