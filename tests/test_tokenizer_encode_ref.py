"""Tekken encoding (vox_tokenizer_encode) on the CPU, against mistral_common's Tekkenizer and the Python oracle.

1. The real vocabulary (tekken_240911.json, shipped with mistral_common; skipped without it): the reference tokenizer's
   golden both ways, and a fixed corpus of a few thousand strings compared id for id with Tekkenizer.encode(s, bos=False,
   eos=False).  The oracle (tests/tekken_reference.py: `regex` + byte_pair_merge) equals Tekkenizer on the same corpus,
   and decode(encode(s)) == s for every string.
2. Synthetic BPE vocabularies: the library, the oracle and a tiktoken.Encoding over the same ranks agree, including a
   repeated byte string (the lowest position wins); a vocabulary cut below its 256 byte tokens and an unknown pattern
   fail with VOX_EFORMAT while decoding keeps working.
3. Errors and buffers: invalid UTF-8 -> VOX_EINVAL, a short id buffer -> VOX_ECAPACITY with the count set, empty text ->
   no ids; two threads encoding through one fresh handle build the rank table once and agree.
4. scripts/gen_unicode_tables.py reproduces the committed csrc/unicode_tables.h.
"""
import base64
import ctypes
import json
import os
import random
import subprocess
import sys
import threading
import unicodedata

import numpy as np
import pytest

import tekken_reference as tr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOX_EINVAL, VOX_EFORMAT, VOX_ECAPACITY = 1, 6, 7   # include/voxtral.h
GOLDEN_IDS = [1362, 19135, 1294, 1278, 4618, 40307, 3910, 1046]   # reference src/tokenizer/mod.rs:255-268
GOLDEN_TEXT = " I spoke in the original phonograph."

pytest.importorskip("regex")


def _code(vx, fn):
    with pytest.raises(vx.VoxtralError) as e:
        fn()
    return e.value.code


def build_corpus(n_random=2400, seed=1234):
    """The fixed comparison corpus: hand-written families, then seeded random strings over every general category."""
    base = list(tr.BPE_CORPUS) + [
        GOLDEN_TEXT, "Hello, world!", "It's 3:45pm -- isn't it?", "e.g. U.S.A. and Ph.D.s", "you'll we'd they're I'm",
        "CamelCaseWords and snake_case_words and SHOUTING", "McDonald's iPhone eBay OpenAI", "naïve coöperate façade",
    ]
    out = list(base)
    out += ["1234567890", "3.14159", "1,000,000", "v2.0.1", "x1y2z3", "٣٤٥ ४५६ 一二三", "Ⅻ ½ ²³"]   # digits one by one
    out += ["!!!", "?!?!", "...\r\n", "--//\r\n//", "a // b", " ///\n\n", "(*&^%$#@!)", "“quotes” ‘and’ «guillemets»",
            "foo/bar/baz", "C:\\path\\to", "http://x.org/a?b=c&d=e", "<tag attr='1'/>", "#hashtag @mention"]
    out += ["line one\r\nline two\r\n\r\nline four", "para\n\n\npara", "\n", "\r\n", "\r", "\n\n\n", " \n \n ", "\t\r\n\t",
            "a\rb", "x\n", "  \r\n  y"]
    for w in ("word", "Word", "WORD", "123", "...", "ǅ"):
        for pre in ("", " ", "  ", "   ", "\t", " \t", "\t ", "\t\t"):
            for post in ("", " ", "  ", "\t", " \t "):
                out.append(pre + w + post)
                out.append(pre + w + post + w)
    special = ["\u00a0", "\u3000", "\x1c", "\x1d", "\x1e", "\x1f", "\x85", "\x0b", "\x0c", "\u2028", "\u202f", "\u180e",
               "\u200b", "\ufeff"]
    for c in special:
        out += [f"a{c}b", f"a{c}{c}b", f"{c}word", f"word{c}", f" {c} x", f"{c}\n", f"1{c}2", f"{c}"]
    out += ["ǅemal ǅǅ ǈ ǋa", "ʰello ˈstress ʼapostrophe", "ᵃᵇᶜ", "ǄǅǆDž", "ﬁnal ﬂow", "ß ẞ"]
    for s in ("café résumé naïve", "Ångström Zürich", "Việt Nam", "ñandú", "e\u0301\u0302\u0303", "\u0301a", " \u0301",
              "a\u0301\u0301b"):
        out += [s, unicodedata.normalize("NFD", s), unicodedata.normalize("NFC", s)]
    out += ["Καλημέρα κόσμε, ΑΘΗΝΑ", "Привет, мир! ПРИВЕТ", "مرحبا بالعالم ١٢٣", "नमस्ते दुनिया १२३", "こんにちは世界、カタカナ",
            "你好，世界。中文测试", "안녕하세요 세계", "שלום עולם", "ไทย ภาษา", "👍🏽 👨‍👩‍👧‍👦 🏳️‍🌈 😀😀", "\ue000\ue001 \U000f0000",
            "[INST] hello [/INST]", "<s></s>[TOOL_CALLS]", "[STREAMING_PAD]"]
    # seeded random strings drawn from every general category among code points assigned in Unicode 15.0
    by_cat = {}
    for cp in range(0x110000):
        cat = unicodedata.category(chr(cp))
        if cat not in ("Cn", "Cs"):
            by_cat.setdefault(cat, []).append(cp)
    cats = sorted(by_cat)
    rng = random.Random(seed)
    for i in range(n_random):
        n = rng.randint(1, 12)
        chars = []
        for _ in range(n):
            r = rng.random()
            if r < 0.15:
                chars.append(" ")
            elif r < 0.2:
                chars.append(rng.choice("\r\n\t/"))
            else:
                chars.append(chr(rng.choice(by_cat[cats[rng.randrange(len(cats))]])))
        out.append("".join(chars))
    return out


@pytest.fixture(scope="module")
def corpus():
    return build_corpus()


@pytest.fixture(scope="module")
def real(vx):
    mc = pytest.importorskip("mistral_common")
    path = os.path.join(os.path.dirname(mc.__file__), "data", "tekken_240911.json")
    if not os.path.exists(path):
        pytest.skip("mistral_common without tekken_240911.json")
    from mistral_common.tokens.tokenizers.tekken import Tekkenizer
    with open(path, encoding="utf-8") as f:
        doc = json.load(f)
    return vx.VoxtralTokenizer.from_file(path), Tekkenizer.from_file(path), tr.Encoder(doc)


def test_real_vocabulary_golden(real):
    t, tk, _ = real
    assert t.encode(GOLDEN_TEXT).tolist() == GOLDEN_IDS
    assert t.decode(GOLDEN_IDS) == GOLDEN_TEXT
    assert tk.encode(GOLDEN_TEXT, bos=False, eos=False) == GOLDEN_IDS


def test_real_vocabulary_corpus(real, corpus):
    t, tk, oracle = real
    assert len(corpus) > 3000
    bad_vx, bad_or, bad_rt = [], [], []
    for s in corpus:
        want = tk.encode(s, bos=False, eos=False)
        got = t.encode(s).tolist()
        if got != want:
            bad_vx.append((s, got, want))
        if oracle.encode(s) != want:
            bad_or.append(s)
        if t.decode(got) != s:
            bad_rt.append(s)
        assert all(i >= tr.TEXT_TOKEN_OFFSET for i in got)
    assert not bad_vx, bad_vx[:5]
    assert not bad_or, bad_or[:5]
    assert not bad_rt, bad_rt[:5]


def test_real_vocabulary_no_normalisation_and_no_special_ids(real):
    t, tk, _ = real
    nfc, nfd = "café", unicodedata.normalize("NFD", "café")
    assert nfc != nfd and t.encode(nfc).tolist() != t.encode(nfd).tolist()
    assert t.decode(t.encode(nfd)) == nfd
    ids = t.encode("[INST] hi [/INST]</s>").tolist()
    assert min(ids) >= 1000 and ids == tk.encode("[INST] hi [/INST]</s>", bos=False, eos=False)


@pytest.fixture(scope="module")
def synth_doc():
    return json.loads(tr.synthetic_bpe_tekken_json(tr.BPE_CORPUS, 700))


def _vx_tok(vx, doc):
    return vx.VoxtralTokenizer.from_json(json.dumps(doc))


def _check_three_way(vx, doc, strings):
    t = _vx_tok(vx, doc)
    oracle = tr.Encoder(doc)
    enc = tr.tiktoken_encoding(doc)
    for s in strings:
        got = t.encode(s).tolist()
        assert got == oracle.encode(s), s
        if enc is not None:
            assert got == [i + tr.TEXT_TOKEN_OFFSET for i in enc.encode(s, disallowed_special=())], s
        assert t.decode(got) == s
    return t, enc


def test_synthetic_bpe_vocabulary(vx, synth_doc, corpus):
    v = synth_doc["vocab"]
    toks = [base64.b64decode(e["token_bytes"]) for e in v]
    assert len(v) > 600
    assert sum(1 for b in toks if b.startswith(b" ") and len(b) > 2) > 50     # leading-space tokens
    assert any(len(b.decode("utf-8", "ignore")) < len(b) and len(b) > 2 for b in toks)   # multi-byte letters merged
    t, enc = _check_three_way(vx, synth_doc, corpus[:1500])
    if enc is None:
        print("\n[tekken] tiktoken not installed: compared with the oracle only")
    ids = t.encode(" the transcription").tolist()
    assert len(ids) < len(" the transcription") // 2      # merges apply


def test_duplicated_byte_string_lowest_position_wins(vx, synth_doc):
    doc = json.loads(json.dumps(synth_doc))
    v = doc["vocab"]
    toks = [base64.b64decode(e["token_bytes"]) for e in v]
    q = max(i for i, b in enumerate(toks) if b.startswith(b" ") and b[1:].isalpha() and len(b) > 4)
    word = toks[q].decode()
    # a copy at the end never wins; a copy at a lower position (overwriting another token) does: the piece is a token
    v.append({"rank": len(v), "token_bytes": v[q]["token_bytes"], "token_str": word})
    low = 300
    v[low] = {"rank": low, "token_bytes": v[q]["token_bytes"], "token_str": word}
    doc["config"]["default_vocab_size"] = 1000 + len(v)
    t, _ = _check_three_way(vx, doc, [word, word * 3, "x" + word + " ", "the transcription of" + word])
    assert t.encode(word).tolist() == [low + 1000]
    assert t.decode([q + 1000]) == t.decode([len(v) - 1 + 1000]) == word


def test_cut_below_byte_tokens_and_unknown_pattern(vx, synth_doc):
    doc = json.loads(json.dumps(synth_doc))
    doc["config"]["default_vocab_size"] = 1000 + 200       # bytes 200..255 are cut away
    t = _vx_tok(vx, doc)
    assert _code(vx, lambda: t.encode("abc")) == VOX_EFORMAT
    assert _code(vx, lambda: t.encode("")) == VOX_EFORMAT   # the vocabulary, not the text, is refused
    assert t.decode([1000 + ord("a"), 1000 + 300]) == "a" + base64.b64decode(doc["vocab"][300]["token_bytes"]).decode()
    with pytest.raises(ValueError):
        tr.Encoder(doc)
    for pattern in ("", r"\s+|\S+", tr.TEKKEN_PATTERN + "|x"):
        d2 = json.loads(json.dumps(synth_doc))
        d2["config"]["pattern"] = pattern
        t2 = _vx_tok(vx, d2)
        assert _code(vx, lambda: t2.encode("hello")) == VOX_EFORMAT
        assert t2.decode([1000 + ord("h"), 1000 + ord("i")]) == "hi"
    # a vocabulary without the pattern field (the older synthetic decode-only fixture) only decodes
    from oracle import tokenizer as otok
    t3 = vx.VoxtralTokenizer.from_json(otok.synthetic_tekken_json())
    assert _code(vx, lambda: t3.encode("a")) == VOX_EFORMAT


INVALID_UTF8 = [b"\xff", b"\xfe", b"\x80", b"a\xbfb", b"\xc0\xaf", b"\xc1\x81", b"\xe0\x80\xaf", b"\xf0\x80\x80\xaf",
                b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xc3", b"abc\xe2\x82",
                b"\xf0\x9f\x98", b"\xe2\x28\xa1", b"ok \xc3\x28"]


def test_errors_and_buffers(vx, synth_doc):
    t = _vx_tok(vx, synth_doc)
    for raw in INVALID_UTF8:
        assert _code(vx, lambda: t.encode(raw)) == VOX_EINVAL, raw
    for raw in (b"\xef\xbf\xbf", b"\xf4\x8f\xbf\xbf", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\x00", b"a\x00b"):
        ids = t.encode(raw)   # the valid edges of the encoding, NUL included
        assert t.decode(ids).encode("utf-8") == raw, raw
    assert t.encode("").size == 0 and t.encode(b"").dtype == np.int32
    lib = vx.lib()
    text = "the quick brown fox".encode()
    n = ctypes.c_size_t(0)
    assert lib.vox_tokenizer_encode(t._h, text, len(text), None, 0, ctypes.byref(n)) == 0
    need = n.value
    assert need == t.encode(text).size > 2
    buf = np.zeros(need, np.int32)
    n.value = 0
    assert lib.vox_tokenizer_encode(t._h, text, len(text), buf.ctypes.data_as(ctypes.c_void_p), need - 1,
                                    ctypes.byref(n)) == VOX_ECAPACITY
    assert n.value == need
    assert lib.vox_tokenizer_encode(t._h, text, len(text), buf.ctypes.data_as(ctypes.c_void_p), need, ctypes.byref(n)) == 0
    assert buf.tolist() == t.encode(text).tolist()
    assert lib.vox_tokenizer_encode(t._h, None, 0, None, 0, ctypes.byref(n)) == 0 and n.value == 0
    assert lib.vox_tokenizer_encode(None, text, len(text), None, 0, ctypes.byref(n)) == VOX_EINVAL
    assert lib.vox_tokenizer_encode(t._h, text, len(text), None, 0, None) == VOX_EINVAL


def test_two_threads_share_one_fresh_handle(vx, synth_doc, corpus):
    want = [tr.Encoder(synth_doc).encode(s) for s in corpus[:400]]
    t = _vx_tok(vx, synth_doc)   # no encode yet: the rank table is built by whichever thread gets there first
    results, errors = [None, None], []

    def work(k):
        try:
            results[k] = [t.encode(s).tolist() for s in corpus[:400]]
        except Exception as e:   # pragma: no cover - reported below
            errors.append(e)

    th = [threading.Thread(target=work, args=(k,)) for k in range(2)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors and results[0] == results[1] == want


def test_unicode_tables_are_generated():
    if unicodedata.unidata_version != "15.0.0":
        pytest.skip(f"Python's unicodedata is {unicodedata.unidata_version}; the header is generated from 15.0.0")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "gen_unicode_tables.py"), "--check"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
