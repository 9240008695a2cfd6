"""Tekken encoding in plain Python: the oracle of vox_tokenizer_encode and of the bias-text expansion (include/voxtral.h).

- `encode(vocab_json, text)`: the pattern of `config.pattern` through the `regex` module, then tiktoken's
  `byte_pair_merge` inside each piece (a piece that is a token is that token); id = vocab position + 1000.  The rank
  table holds the text entries below default_vocab_size - 1000 (no is_control entries, no entries without bytes), the
  lowest position winning for a repeated byte string: mistral_common's cut of the vocabulary.
- `expand(vocab_json, phrases, boosts)`: vox_session_set_bias_text's expansion rule, as (id phrases, boosts).
- `synthetic_bpe_tekken_json(corpus, n_merges)`: a deterministic byte-level BPE trainer over the Tekken pattern's
  pieces, giving multi-byte and leading-space tokens like a real vocabulary's.
"""
from __future__ import annotations

import base64
import json
from collections import Counter

TEXT_TOKEN_OFFSET = 1000
TEKKEN_PATTERN = (r"[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]*[\p{Ll}\p{Lm}\p{Lo}\p{M}]+|"
                  r"[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]+[\p{Ll}\p{Lm}\p{Lo}\p{M}]*|"
                  r"\p{N}| ?[^\s\p{L}\p{N}]+[\r\n/]*|\s*[\r\n]+|\s+(?!\S)|\s+")
# PropList.txt White_Space (\s of the pattern)
WHITE_SPACE = frozenset(map(chr, [0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028,
                                  0x2029, 0x202F, 0x205F, 0x3000]))
MAX_BIAS_LEN = 16
MAX_BIAS_PHRASES = 256


def _entry_bytes(e):
    """The bytes decode() uses for a vocab entry (base64 token_bytes, else UTF-8 token_str), None for none."""
    if e.get("is_control", False):
        return None
    tb = e.get("token_bytes")
    if tb is not None:
        try:
            return base64.b64decode(tb, validate=True)
        except Exception:
            pass
    ts = e.get("token_str")
    return ts.encode("utf-8") if ts is not None else None


def mergeable_ranks(doc: dict) -> dict:
    """bytes -> vocab position, cut at default_vocab_size - 1000, the lowest position of a repeated string winning."""
    cut = max(0, int(doc["config"]["default_vocab_size"]) - TEXT_TOKEN_OFFSET)
    ranks = {}
    for pos, e in enumerate(doc["vocab"][:cut]):
        b = _entry_bytes(e)
        if b:
            ranks.setdefault(b, pos)
    return ranks


def byte_pair_merge(ranks: dict, piece: bytes) -> list:
    """tiktoken's byte_pair_merge: the piece's tokens (bytes), merging the lowest-rank adjacent pair, leftmost first."""
    if piece in ranks:
        return [piece]
    parts = [piece[i:i + 1] for i in range(len(piece))]
    while len(parts) > 1:
        best, at = None, -1
        for i in range(len(parts) - 1):
            r = ranks.get(parts[i] + parts[i + 1])
            if r is not None and (best is None or r < best):
                best, at = r, i
        if best is None:
            break
        parts[at:at + 2] = [parts[at] + parts[at + 1]]
    return parts


class Encoder:
    def __init__(self, doc):
        import regex
        self.doc = json.loads(doc) if isinstance(doc, str) else doc
        if self.doc["config"].get("pattern") != TEKKEN_PATTERN:
            raise ValueError("not the Tekken pattern")
        self.ranks = mergeable_ranks(self.doc)
        missing = [b for b in range(256) if bytes([b]) not in self.ranks]
        if missing:
            raise ValueError(f"no token for byte {missing[0]:#04x}")
        self.pat = regex.compile(TEKKEN_PATTERN)

    def pieces(self, text: str) -> list:
        return self.pat.findall(text)

    def encode(self, text: str) -> list:
        out = []
        for p in self.pieces(text):
            out += [self.ranks[t] + TEXT_TOKEN_OFFSET for t in byte_pair_merge(self.ranks, p.encode("utf-8"))]
        return out

    def expand(self, phrases, boosts):
        """vox_session_set_bias_text's expansion: (id phrases, boosts); ValueError where the call returns VOX_EINVAL
        before reaching vox_session_set_bias."""
        boosts = [float(b) for b in boosts] if hasattr(boosts, "__len__") else [float(boosts)] * len(phrases)
        ids, out_b = [], []
        for p, (w, b) in enumerate(zip(phrases, boosts)):
            if not w:
                raise ValueError(f"phrase {p} is empty")
            forms = [self.encode(w)]
            if w[0] not in WHITE_SPACE:
                spaced = self.encode(" " + w)
                if spaced != forms[0]:
                    forms.append(spaced)
            for f in forms:
                if len(f) > MAX_BIAS_LEN:
                    raise ValueError(f"phrase {p} encodes to {len(f)} ids")
                if len(ids) == MAX_BIAS_PHRASES:
                    raise ValueError(f"phrase {p}: more than {MAX_BIAS_PHRASES} id phrases")
                ids.append(f)
                out_b.append(b)
        return ids, out_b


def tiktoken_encoding(doc: dict):
    """A tiktoken.Encoding over the same ranks (ids without the 1000 offset); None when tiktoken is missing."""
    try:
        import tiktoken
    except ImportError:
        return None
    return tiktoken.Encoding(name="synthetic", pat_str=doc["config"]["pattern"], mergeable_ranks=mergeable_ranks(doc),
                             special_tokens={})


def synthetic_bpe_tekken_json(corpus, n_merges: int, pattern: str = TEKKEN_PATTERN) -> str:
    """A tekken.json-shaped BPE vocabulary trained on `corpus` (strings): the 256 bytes, then up to n_merges merges, each
    the most frequent adjacent pair over the corpus's pre-tokenized pieces (the smaller pair on a tie), so the result
    depends on the corpus alone.  Text entries only (rank = position); default_vocab_size = 1000 + their count."""
    import regex
    pat = regex.compile(TEKKEN_PATTERN)
    words = Counter()
    for s in corpus:
        for p in pat.findall(s):
            words[tuple(bytes([b]) for b in p.encode("utf-8"))] += 1
    vocab = [bytes([b]) for b in range(256)]
    known = set(vocab)
    words = dict(words)
    for _ in range(n_merges):
        pairs = Counter()
        for w, c in words.items():
            for a, b in zip(w, w[1:]):
                pairs[(a, b)] += c
        if not pairs:
            break
        top = max(pairs.values())
        a, b = min(p for p, c in pairs.items() if c == top)
        ab = a + b
        if ab not in known:
            known.add(ab)
            vocab.append(ab)
        merged = {}
        for w, c in words.items():
            out, i = [], 0
            while i < len(w):
                if i + 1 < len(w) and w[i] == a and w[i + 1] == b:
                    out.append(ab)
                    i += 2
                else:
                    out.append(w[i])
                    i += 1
            merged[tuple(out)] = merged.get(tuple(out), 0) + c
        words = merged
    entries = []
    for r, t in enumerate(vocab):
        try:
            s = t.decode("utf-8")
        except UnicodeDecodeError:
            s = None
        entries.append({"rank": r, "token_bytes": base64.b64encode(t).decode(), "token_str": s})
    doc = {"config": {"pattern": pattern, "num_vocab_tokens": len(vocab), "default_vocab_size": TEXT_TOKEN_OFFSET + len(vocab),
                      "default_num_special_tokens": TEXT_TOKEN_OFFSET, "version": "v3"},
           "vocab": entries}
    return json.dumps(doc)


# a small multilingual corpus for synthetic vocabularies: leading-space words, digits, punctuation, non-ASCII letters
BPE_CORPUS = [
    "The quick brown fox jumps over the lazy dog near the river bank.",
    "I spoke in the original phonograph, and the recording was played back at the station.",
    "Zürich, Genève and Köln are cities; São Paulo and Bogotá are too.",
    "Please transcribe the meeting about the quarterly budget and the new hiring plan.",
    "Voxtral streams audio in real time: every token arrives as soon as its audio is final.",
    "Custom vocabulary boosts rare words such as Kubernetes, PyTorch, Hopper and wgmma.",
    "Der schnelle braune Fuchs springt über den faulen Hund.",
    "Le café est très chaud, mais la crème brûlée est froide.",
    "Η γρήγορη καφέ αλεπού πηδάει πάνω από τον τεμπέλη σκύλο.",
    "Быстрая коричневая лиса прыгает через ленивую собаку.",
    "Call me at 555-0199 or write to support@example.com before 10:30 on 2024/05/17.",
    "  indented line\twith tabs\r\nand CRLF line endings\n\nand blank lines  ",
    "Dr. Smith's patients -- all 42 of them -- were seen on time (mostly).",
    "Mistral, Voxtral, Tekken, transcription, transcribe, transcribed, transcribing.",
    "the the the and and of of to to in in is is that that it it for for on on with with as as",
]
