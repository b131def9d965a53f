"""Host side of the on-device BPE token counter (north star; SURVEY.md §0 F1: the reference counts no tokens itself — it reads
`usage` from the upstream's response — so this is a side output with an external oracle, HF `tokenizers`).

  load_tokenizer(path or dict)   HF tokenizer.json (or vocab.json + merges.txt) -> BpeTables, the flat arrays arks_load_bpe
                                 takes: the id of every single-byte token, the merge list (rank = index) as id triples, the
                                 Unicode class table of the Qwen2 split pattern (arks_b200/data/bpe_unicode.bin.z) and
                                 whether the tokenizer normalises to NFC
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
BPE_NFC = 1            # arks_bpe_tables.flags
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

    def c_struct(self) -> ArksBpeTables:
        p32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_uint32))
        return ArksBpeTables(p32(self.byte_id), len(self.left), p32(self.left), p32(self.right), p32(self.merged),
                             self.cp_class.ctypes.data_as(C.POINTER(C.c_uint8)), self.flags)


def unicode_classes() -> np.ndarray:
    return np.frombuffer(zlib.decompress(open(UNICODE_TABLE, "rb").read()), np.uint8).copy()


def load_tokenizer(src, merges_txt: str | None = None) -> BpeTables:
    """src: path of a tokenizer.json / its parsed dict / its JSON text, or the path of a vocab.json when merges_txt is given"""
    if merges_txt is not None:
        vocab = json.load(open(src))
        merges = [tuple(l.split(" ")) for l in open(merges_txt).read().split("\n") if l and not l.startswith("#version")]
        normalizer = None
    else:
        if isinstance(src, dict):
            tj = src
        elif isinstance(src, str) and src.lstrip().startswith("{"):
            tj = json.loads(src)
        else:
            tj = json.load(open(src))
        if tj["model"]["type"] != "BPE":
            raise ValueError("only byte-level BPE tokenizers are supported")
        vocab = tj["model"]["vocab"]
        merges = [tuple(m) if isinstance(m, list) else tuple(m.split(" ")) for m in tj["model"]["merges"]]
        normalizer = tj.get("normalizer")
    b2u = bytes_to_unicode()
    byte_id = np.zeros(256, np.uint32)
    for b in range(256):
        if b2u[b] not in vocab:
            raise ValueError(f"byte {b} has no token: not a byte-level vocabulary")
        byte_id[b] = vocab[b2u[b]]
    left = np.fromiter((vocab[a] for a, _ in merges), np.uint32, len(merges))
    right = np.fromiter((vocab[b] for _, b in merges), np.uint32, len(merges))
    merged = np.fromiter((vocab[a + b] for a, b in merges), np.uint32, len(merges))
    flags = BPE_NFC if normalizer and (normalizer.get("type") == "NFC" or any(
        n.get("type") == "NFC" for n in normalizer.get("normalizers", []))) else 0
    return BpeTables(byte_id, left, right, merged, unicode_classes(), flags)


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


def standin_tokenizer(vocab_size: int = 151_643, seed: int = 0xB9E, cache_dir: str | None = None):
    """-> (tokenizers.Tokenizer, tokenizer.json text). Deterministic; cached under cache_dir when given."""
    from tokenizers import Regex, Tokenizer, decoders, models, pre_tokenizers, trainers
    path = os.path.join(cache_dir, f"standin_bpe_{vocab_size}_{seed:x}.json") if cache_dir else None
    if path and os.path.exists(path):
        text = open(path).read()
        return Tokenizer.from_str(text), text
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.Sequence([
        pre_tokenizers.Split(Regex(QWEN2_PATTERN), behavior="isolated", invert=False),
        pre_tokenizers.ByteLevel(add_prefix_space=False, use_regex=False)])
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=vocab_size, special_tokens=[], show_progress=False,
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(_corpus(60_000 if vocab_size < 50_000 else 300_000, seed), trainer)
    text = tok.to_str()
    if path:
        os.makedirs(cache_dir, exist_ok=True)
        open(path, "w").write(text)
    return tok, text
