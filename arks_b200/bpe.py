"""Host side of the on-device BPE token counter (north star; SURVEY.md §0 F1: the reference counts no tokens itself — it reads
`usage` from the upstream's response — so this is a side output with an external oracle, HF `tokenizers`).

  load_tokenizer(path or dict)   HF tokenizer.json (or vocab.json + merges.txt) -> BpeTables, the flat arrays arks_load_bpe
                                 takes: the id of every single-byte token, the merge list (rank = index) as id triples, the
                                 Unicode class table of the Qwen2 split pattern (arks_b200/data/bpe_unicode.bin.z) and
                                 the flags: NFC normalisation, the Llama 3 number split, `ignore_merges` (then also the
                                 vocabulary's token strings, which arks_load_bpe_vocab takes). Only the Qwen2 and Llama 3
                                 families are accepted; anything else raises ValueError instead of being miscounted
  content_strings(body)          what is counted: every string that is the value of a key named `content` (the messages of
                                 a chat request, the message / delta of a completion), JSON escapes decoded; with
                                 keys=METERED_KEYS the wider set metered streams count (N5, arks_set_stream_metering)
  standin_tokenizer(n, seed)     a seeded byte-level BPE trained offline with `tokenizers` on synthetic text, used where
                                 the real Qwen2.5 vocabulary would be (it is not on disk and there is no network): same
                                 pre-tokenizer pattern, same algorithm, ~151 k merges at full scale. TEST / BENCH helper.

What the device computes for one text: the Qwen2 pre-tokenizer split (transformers/models/qwen2/tokenization_qwen2.py:33),
then byte-level BPE of every piece (merge the adjacent pair of lowest rank, leftmost first, until none is left) — the number of
symbols that remain is the number of tokens `tokenizers.Tokenizer.encode(text, add_special_tokens=False)` returns.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import zlib
from dataclasses import dataclass

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
UNICODE_TABLE = os.path.join(HERE, "data", "bpe_unicode.bin.z")
QWEN2_PATTERN = (r"""(?i:'s|'t|'re|'ve|'m|'ll|'d)|[^\r\n\p{L}\p{N}]?\p{L}+|\p{N}| ?[^\s\p{L}\p{N}]+[\r\n]*|\s*[\r\n]+"""
                 r"""|\s+(?!\S)|\s+""")
# Llama 3: the same alternatives, but numbers in runs of up to three
LLAMA3_PATTERN = QWEN2_PATTERN.replace(r"|\p{N}|", r"|\p{N}{1,3}|")
BPE_NFC = 1            # arks_bpe_tables.flags
BPE_DIGITS3 = 2        # the pre-tokenizer splits numbers as \p{N}{1,3} (LLAMA3_PATTERN)
BPE_IGNORE_MERGES = 4  # a pre-token that is a vocabulary entry is one token (the BPE model's "ignore_merges": true)
MAX_VOCABS = 8         # ARKS_BPE_MAX_VOCABS
MAX_PIECE = 128        # bytes of one pre-token the device counts (kBpeMaxPiece)
UNCOUNTED = 0xFFFFFFFF  # ARKS_BPE_UNCOUNTED
CONTENT_KEYS = ("content",)
# metered rows (N5): also content parts ({"type":"text","text":..}), reasoning streams and tool-call arguments
METERED_KEYS = ("content", "text", "reasoning_content", "arguments")


def bytes_to_unicode():
    """GPT-2's byte <-> printable character table (the alphabet of byte-level BPE vocabularies)"""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, map(chr, cs)))


class ArksBpeTables(C.Structure):
    _fields_ = [("byte_id", C.POINTER(C.c_uint32)), ("n_merges", C.c_uint32), ("left", C.POINTER(C.c_uint32)),
                ("right", C.POINTER(C.c_uint32)), ("merged", C.POINTER(C.c_uint32)), ("cp_class", C.POINTER(C.c_uint8)),
                ("flags", C.c_uint32)]


@dataclass
class BpeTables:
    byte_id: np.ndarray   # [256] uint32
    left: np.ndarray      # [n_merges] uint32, rank = index
    right: np.ndarray
    merged: np.ndarray
    cp_class: np.ndarray  # [0x110000 / 2] uint8, a nibble per code point (tools/gen_bpe_unicode.py)
    flags: int
    # BPE_IGNORE_MERGES only: the token strings of 2..MAX_PIECE bytes, token k = tok_bytes[tok_off[k]:tok_off[k + 1]]
    tok_bytes: np.ndarray | None = None  # uint8
    tok_off: np.ndarray | None = None    # [n + 1] uint32

    def c_struct(self) -> ArksBpeTables:
        p32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        return ArksBpeTables(p32(self.byte_id), len(self.left), p32(self.left), p32(self.right), p32(self.merged),
                             self.cp_class.ctypes.data_as(C.POINTER(C.c_uint8)), self.flags)


def unicode_classes() -> np.ndarray:
    return np.frombuffer(zlib.decompress(open(UNICODE_TABLE, "rb").read()), np.uint8).copy()


def _check_tokenizer_json(tj) -> int:
    """the flags of a tokenizer.json this counter reproduces exactly, or ValueError naming what it does not"""
    model = tj.get("model") or {}
    if model.get("type") != "BPE":
        raise ValueError(f"unsupported model type {model.get('type')!r}: only byte-level BPE")
    if model.get("dropout") not in (None, 0, 0.0):
        raise ValueError("unsupported BPE dropout")
    if model.get("byte_fallback"):
        raise ValueError("unsupported byte_fallback (SentencePiece-style BPE)")
    for k in ("continuing_subword_prefix", "end_of_word_suffix"):
        if model.get(k):
            raise ValueError(f"unsupported {k} {model[k]!r}")
    norm = tj.get("normalizer")
    if norm is not None and norm.get("type") != "NFC":
        raise ValueError(f"unsupported normalizer {norm.get('type')!r}: only none or NFC")
    pre = tj.get("pre_tokenizer") or {}
    seq = pre.get("pretokenizers") if pre.get("type") == "Sequence" else None
    if not seq or len(seq) != 2 or seq[0].get("type") != "Split" or seq[1].get("type") != "ByteLevel":
        raise ValueError(f"unsupported pre-tokenizer {json.dumps(pre)[:200]}: only Sequence[Split(regex), ByteLevel(use_regex=false)]")
    split, bl = seq
    regex = (split.get("pattern") or {}).get("Regex")
    if regex not in (QWEN2_PATTERN, LLAMA3_PATTERN):
        raise ValueError(f"unsupported split pattern {json.dumps(split.get('pattern'))[:200]}: only the Qwen2 and Llama 3 patterns")
    if split.get("behavior") != "Isolated" or split.get("invert"):
        raise ValueError(f"unsupported split behaviour {split.get('behavior')!r} invert={split.get('invert')!r}")
    if bl.get("use_regex", True):
        raise ValueError("unsupported ByteLevel(use_regex=true): the GPT-2 pre-tokenizer")
    if bl.get("add_prefix_space"):
        raise ValueError("unsupported ByteLevel(add_prefix_space=true)")
    return ((BPE_NFC if norm is not None else 0) | (BPE_DIGITS3 if regex == LLAMA3_PATTERN else 0)
            | (BPE_IGNORE_MERGES if model.get("ignore_merges") else 0))


def load_tokenizer(src, merges_txt: str | None = None) -> BpeTables:
    """src: path of a tokenizer.json / its parsed dict / its JSON text, or the path of a vocab.json when merges_txt is given
    (a Qwen2 vocabulary). A tokenizer.json must be a Qwen2 or Llama 3 style byte-level BPE (_check_tokenizer_json)."""
    if merges_txt is not None:
        vocab = json.load(open(src))
        merges = [tuple(l.split(" ")) for l in open(merges_txt).read().split("\n") if l and not l.startswith("#version")]
        flags = 0
    else:
        if isinstance(src, dict):
            tj = src
        elif isinstance(src, str) and src.lstrip().startswith("{"):
            tj = json.loads(src)
        else:
            tj = json.load(open(src))
        flags = _check_tokenizer_json(tj)
        vocab = tj["model"]["vocab"]
        merges = [tuple(m) if isinstance(m, list) else tuple(m.split(" ")) for m in tj["model"]["merges"]]
    b2u = bytes_to_unicode()
    byte_id = np.zeros(256, np.uint32)
    for b in range(256):
        if b2u[b] not in vocab:
            raise ValueError(f"byte {b} has no token: not a byte-level vocabulary")
        byte_id[b] = vocab[b2u[b]]
    left = np.fromiter((vocab[a] for a, _ in merges), np.uint32, len(merges))
    right = np.fromiter((vocab[b] for _, b in merges), np.uint32, len(merges))
    merged = np.fromiter((vocab[a + b] for a, b in merges), np.uint32, len(merges))
    t = BpeTables(byte_id, left, right, merged, unicode_classes(), flags)
    if flags & BPE_IGNORE_MERGES:
        # a pre-token is looked up as its byte-level string; entries with a character outside that alphabet never match
        u2b = {u: b for b, u in bytes_to_unicode().items()}
        strs = []
        for s in vocab:
            if 2 <= len(s) <= MAX_PIECE and all(c in u2b for c in s):
                strs.append(bytes(u2b[c] for c in s))
        t.tok_off = np.zeros(len(strs) + 1, np.uint32)
        t.tok_off[1:] = np.cumsum([len(x) for x in strs], dtype=np.uint64).astype(np.uint32)
        t.tok_bytes = np.frombuffer(b"".join(strs), np.uint8).copy()
    return t


def content_strings(body: bytes, keys=CONTENT_KEYS) -> list[str]:
    """every string value of a key named `content` (or any of `keys`), in document order (duplicated keys included)"""
    out = []

    def pairs(ps):
        for k, v in ps:
            if k in keys and isinstance(v, str):
                out.append(v)
        return None

    json.loads(body.decode("utf-8"), object_pairs_hook=pairs)
    return out


def sse_content_strings(chunk: bytes, keys=CONTENT_KEYS) -> list[str]:
    """the same over the `data:` lines of an SSE chunk (events that are not JSON carry no text)"""
    out = []
    for line in chunk.replace(b"\r\n", b"\n").split(b"\n"):
        if line.startswith(b"data:"):
            try:
                out += content_strings(line[5:].strip(), keys)
            except ValueError:
                pass
    return out


# ---- test / bench helper: a stand-in vocabulary (the real one is not on disk, there is no network) -------------------------
def _corpus(n_lines: int, seed: int):
    import random
    from .traffic import WORDS
    r = random.Random(seed)
    syll = ["ka", "lo", "mi", "ter", "an", "ex", "qu", "zen", "dor", "pha", "li", "sto", "ur", "ben", "vi", "cra", "ple", "ost",
            "ing", "tion", "ly", "er", "re", "un", "con", "pro", "ment", "able", "ful", "ness"]
    pseudo = ["".join(r.choice(syll) for _ in range(r.randint(2, 4))) for _ in range(60000)]
    cjk = [chr(r.randint(0x4E00, 0x9FA5)) for _ in range(3000)]
    extra = ["—", "é", "🙂", "...", "!?", "(", ")", "\n", "\t", "'s", "'re", "你好", "\n\n", "  ", "\\", "\"", "/", "{", "}"]
    for _ in range(n_lines):
        toks = []
        for _ in range(r.randint(5, 30)):
            x = r.random()
            if x < 0.55:
                toks.append(r.choice(WORDS))
            elif x < 0.85:
                toks.append(pseudo[int(r.paretovariate(1.1)) % len(pseudo)])
            elif x < 0.9:
                toks.append(str(r.randint(0, 99999)))
            elif x < 0.95:
                toks.append("".join(r.choice(cjk) for _ in range(r.randint(1, 4))))
            else:
                toks.append(r.choice(extra))
        yield " ".join(toks)


def standin_tokenizer(vocab_size: int = 151_643, seed: int = 0xB9E, cache_dir: str | None = None, pattern: str = QWEN2_PATTERN,
                      ignore_merges: bool = False):
    """-> (tokenizers.Tokenizer, tokenizer.json text). Deterministic; cached under cache_dir when given. pattern=LLAMA3_PATTERN,
    ignore_merges=True: a Llama 3 style stand-in (with the defaults, the Qwen2 one, unchanged)."""
    from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, trainers
    if pattern not in (QWEN2_PATTERN, LLAMA3_PATTERN):
        raise ValueError("pattern: QWEN2_PATTERN or LLAMA3_PATTERN")
    variant = ("_llama3" if pattern == LLAMA3_PATTERN else "") + ("_im" if ignore_merges else "")
    path = os.path.join(cache_dir, f"standin_bpe_{vocab_size}_{seed:x}{variant}.json") if cache_dir else None
    if path and os.path.exists(path):
        text = open(path).read()
        return Tokenizer.from_str(text), text
    tok = Tokenizer(models.BPE(ignore_merges=True) if ignore_merges else models.BPE())
    tok.pre_tokenizer = pre_tokenizers.Sequence([
        pre_tokenizers.Split(Regex(pattern), behavior="isolated", invert=False),
        pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=vocab_size, special_tokens=[], show_progress=False,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(_corpus(60_000 if vocab_size < 50_000 else 300_000, seed), trainer)
    text = tok.to_str()
    if path:
        # the cache only saves the training time: a directory that cannot be written (a read-only checkout) is not an error
        tmp = f"{path}.{os.getpid()}.tmp"
        try:
            os.makedirs(cache_dir, exist_ok=True)
            with open(tmp, "w") as f:
                f.write(text)
            os.replace(tmp, path)  # readers never see a half-written file
        except OSError:
            if os.path.exists(tmp):
                os.unlink(tmp)
    return tok, text
