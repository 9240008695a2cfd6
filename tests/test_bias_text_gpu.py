"""Phrase boosting from words on the device (vox_session_set_bias_text, vox_stream_set_bias_text).

Model: the decoder-geometry model (vocab 32768, decoder window 40) of test_bias_gpu.py, 11 streams at the mixed delays of
test_delay_rows_gpu.  Tokenizer: a synthetic BPE vocabulary (tests/tekken_reference.py) whose text ids, 1000 + about 950
positions, fit the model's vocabulary.  Every list given as words must behave exactly like the oracle's expansion of the
same words given as ids to vox_session_set_bias:

1. Incremental prefill and decode at B = 1, 3, 8, 11: bit-identical ids, every emitted id the rule's choice on the step's
   own logits, and the same single extra launch per prefill and decode step as an id list.
2. transcribe_streaming with a graph replay, and transcribe_pcm_ragged with per-stream lists.
3. Bounded and unbounded streaming pools, with the list set before the first tick and mid-stream.
4. A one-token word with a large boost changes emitted ids; every refusal leaves the previous list in force.
"""
import ctypes
import json

import numpy as np
import pytest

import bias_reference as br
import tekken_reference as tr
from oracle import mel as omel
from test_decode_geometry_ref import geometry_model_bytes
from test_delay_rows_gpu import MEL_FRAMES, N, PREFIX, VOX_EINVAL
from test_delay_rows_ref import DELAYS, delay_mel

pytestmark = pytest.mark.gpu

VOX_EFORMAT = 6   # include/voxtral.h
WORDS = ["the", "transcription", "Zürich", "Kubernetes", "café", "quick brown", "\tindented", "Voxtral", "of", "and",
         "São Paulo", "42", "PyTorch", "over the", "budget", "Genève", " and", "streams", "lazy dog", "Fuchs"]


def make_lists(rng):
    """Per stream: 3..7 words with boosts log-uniform in [1e-3, 3), from below the top-2 margins of this model's logits to
    well above them, so that some positions flip and others do not; streams with i % 3 == 2 get none."""
    lists = []
    for i in range(N):
        if i % 3 == 2:
            lists.append(([], []))
            continue
        k = 3 + i % 5
        words = [WORDS[(i * 7 + j * 3) % len(WORDS)] for j in range(k)]
        lists.append((words, [float(np.float32(10.0 ** rng.uniform(-3.0, 0.5))) for _ in words]))
    return lists


class TextBias:
    def __init__(self, vx):
        self.vx = vx
        self.data = geometry_model_bytes(40)
        self.model = m = vx.Q4ModelLoader.from_bytes(self.data).load(0, max_batch=N, max_mel_frames=MEL_FRAMES)
        self.vocab = m.info["vocab"]
        self.doc = json.loads(tr.synthetic_bpe_tekken_json(tr.BPE_CORPUS, 700))
        self.tok = vx.VoxtralTokenizer.from_json(json.dumps(self.doc))
        self.enc = tr.Encoder(self.doc)
        assert len(self.doc["vocab"]) + 1000 < self.vocab
        self.mels = np.concatenate([delay_mel(i) for i in range(N)])
        m.set_delays(DELAYS)
        self.n_out = np.asarray(m.transcribe_streaming(self.mels)).shape[1]
        self.lists = make_lists(np.random.default_rng(11))
        # stream 0 also boosts a one-token word hard: it must win positions
        self.strong = "the"
        assert len(self.enc.encode(self.strong)) == 1
        self.lists[0] = (self.lists[0][0] + [self.strong], self.lists[0][1] + [40.0])

    def expand(self, lst):
        return self.enc.expand(*lst) if lst[0] else ([], [])

    def apply(self, B, text, lists=None):
        """Stream i < B gets lists[i] as words (text) or as the oracle's id phrases; every other stream none."""
        lists = self.lists if lists is None else lists
        self.model.set_bias([], 1.0)
        for i in range(B):
            if not lists[i][0]:
                continue
            if text:
                self.model.set_bias_text(lists[i][0], lists[i][1], self.tok, stream=i)
            else:
                self.model.set_bias(*self.expand(lists[i]), stream=i)

    def incremental(self, B, lists=None, check=True):
        """Prefill + free-running decode steps over streams [0, B); with check, every row's id against the rule on the
        step's own logits.  Returns ids [B][n] and the launches of each call."""
        lists = self.lists if lists is None else lists
        m = self.model
        ref = [br.Stream(*self.expand(lists[i])) for i in range(B)]
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        n0 = m.launch_count()
        toks = [m.prefill(np.tile(PREFIX, (B, 1)).astype(np.int32))]
        launches = [m.launch_count() - n0]
        steps = self.n_out - 1
        for step in range(steps + 1):
            if check:
                logits = m.debug("logits").reshape(B, self.vocab)
                assert toks[-1].tolist() == [ref[i].emit(logits[i]) for i in range(B)], (B, step)
            if step == steps:
                break
            n0 = m.launch_count()
            toks.append(m.decode_step(batch=B))
            launches.append(m.launch_count() - n0)
        return np.stack(toks, 1), np.array(launches)


@pytest.fixture(scope="module")
def tb(vx):
    g = TextBias(vx)
    yield g
    g.model.close()


def test_expansion_forms(tb):
    """The oracle's expansion of the test's words: both forms, one form for words that start with White_Space."""
    ids, boosts = tb.expand((["the", "\tindented", " and"], [1.0, 2.0, 3.0]))
    assert ids[0] == tb.enc.encode("the") and ids[1] == tb.enc.encode(" the") and ids[0] != ids[1]
    assert ids[2] == tb.enc.encode("\tindented") and ids[3] == tb.enc.encode(" and") and len(ids) == 4
    assert boosts == [1.0, 1.0, 2.0, 3.0]


@pytest.mark.parametrize("B", [1, 3, 8, 11])
def test_incremental_text_equals_ids(tb, B):
    tb.apply(B, text=True)
    text, l_text = tb.incremental(B)
    tb.apply(B, text=False)
    ids, l_ids = tb.incremental(B, check=False)
    tb.model.set_bias([], 1.0)
    plain, l_plain = tb.incremental(B, check=False)
    assert np.array_equal(text, ids), B
    assert np.array_equal(l_text, l_ids) and np.all(l_text - l_plain == 1), (l_text, l_plain)
    flipped = int(np.sum(text[0] != plain[0]))
    strong = set(tb.enc.encode(tb.strong) + tb.enc.encode(" " + tb.strong))
    print(f"\n[bias_text] B={B}: stream 0 flipped at {flipped} of {text.shape[1]} positions; streams 1.. at "
          f"{int(np.sum(text[1:] != plain[1:]))} of {text[1:].size}")
    assert flipped > 0 and any(int(t) in strong for t in text[0])
    for i in range(B):   # rows without a list: the ids of the call without lists
        if not tb.lists[i][0]:
            assert np.array_equal(text[i], plain[i]), i


def test_streaming_graph_replay(tb):
    m, B = tb.model, 8
    tb.apply(B, text=False)
    want = np.asarray(m.transcribe_streaming(tb.mels[:B]))
    tb.apply(B, text=True)
    first = np.asarray(m.transcribe_streaming(tb.mels[:B]))
    again = np.asarray(m.transcribe_streaming(tb.mels[:B]))   # the captured step graph replays
    assert np.array_equal(first, want) and np.array_equal(again, want)
    # other lists as words, same graph
    other = [tb.lists[(i + 1) % N] for i in range(N)]
    tb.apply(B, text=True, lists=other)
    got = np.asarray(m.transcribe_streaming(tb.mels[:B]))
    tb.apply(B, text=False, lists=other)
    assert np.array_equal(got, np.asarray(m.transcribe_streaming(tb.mels[:B])))
    m.set_bias_text([], 1.0, None)   # an empty list clears; the tokenizer is not needed
    plain = np.asarray(m.transcribe_streaming(tb.mels[:B]))
    assert int(np.sum(plain != want)) > 0


def test_ragged_per_stream_lists(tb):
    m = tb.model
    audios = [omel.peak_normalize(omel.speechlike(s, 870 + i)) for i, s in enumerate((6.0, 4.5, 7.5, 5.0, 6.5))]
    lists = [tb.lists[j] for j in (0, 2, 1, 4, 3)]   # stream 1 without a list
    m.set_delay(6.0)
    try:
        got = {}
        for text in (True, False):
            m.set_bias([], 1.0)
            for i, lst in enumerate(lists):
                if lst[0]:
                    if text:
                        m.set_bias_text(*lst, tb.tok, stream=i)
                    else:
                        m.set_bias(*tb.expand(lst), stream=i)
            got[text] = m.transcribe_pcm_ragged(audios, peak_normalize=False)
        for a, b in zip(got[True], got[False]):
            assert np.array_equal(a, b)
        m.set_bias([], 1.0)
        plain = m.transcribe_pcm_ragged(audios, peak_normalize=False)
        assert sum(int(np.sum(a != b)) for a, b in zip(got[True], plain)) > 0
    finally:
        m.set_bias([], 1.0)
        m.set_delays(DELAYS)


def _pool_run(vx, tb, audios, lists, text, unbounded, mid=None):
    """Sessions opened at tick 0, lists[i] set before their first tick (as words or ids); mid = (session index, ids
    polled, list): set once that session has polled that many ids.  Returns per session the ids."""
    pool = vx.StreamingPool(tb.model, max_sessions=len(audios), max_seconds=None if unbounded else 12.0)

    def put(sid, lst):
        if text:
            pool.set_bias_text(sid, lst[0], lst[1], tb.tok)
        else:
            pool.set_bias(sid, *tb.expand(lst))

    try:
        n = len(audios)
        sids = [pool.open() for _ in range(n)]
        for s, lst in zip(sids, lists):
            if lst[0]:
                put(s, lst)
                if text:   # a refused list leaves this one in force
                    with pytest.raises(vx.VoxtralError) as e:
                        pool.set_bias_text(s, lst[0] + [b"\xc3"], 1.0, tb.tok)
                    assert e.value.code == VOX_EINVAL
        fed, ids, done_mid = [0] * n, [[] for _ in range(n)], False
        for _ in range(2000):
            if mid is not None and not done_mid and len(ids[mid[0]]) >= mid[1]:
                put(sids[mid[0]], mid[2])
                done_mid = True
            for i in range(n):
                if fed[i] < audios[i].size:
                    pool.push(sids[i], audios[i][fed[i]:fed[i] + 1280])
                    fed[i] += 1280
                    if fed[i] >= audios[i].size:
                        pool.finish(sids[i])
            pool.tick()
            done_all = True
            for i in range(n):
                got, done = pool.poll(sids[i])
                ids[i] += got
                done_all = done_all and done
            if done_all:
                break
        return ids
    finally:
        pool.close()


@pytest.mark.parametrize("unbounded", [False, True], ids=["bounded", "unbounded"])
def test_streaming_pool(vx, tb, unbounded):
    m = tb.model
    audios = [omel.peak_normalize(omel.speechlike(s, 810 + i)) for i, s in enumerate((5.0, 6.5, 4.0, 5.5))]
    lists = [tb.lists[0], ([], []), tb.lists[1], tb.lists[3]]
    m.set_delay(6.0)
    try:
        text = _pool_run(vx, tb, audios, lists, True, unbounded)
        assert text == _pool_run(vx, tb, audios, lists, False, unbounded)
        plain = _pool_run(vx, tb, audios, [([], [])] * 4, False, unbounded)
        assert text[1] == plain[1] and text[0] != plain[0]
        # mid-stream: the ids polled before the list are the unboosted ones, and text equals ids after it
        mid_text = _pool_run(vx, tb, audios[:1], [([], [])], True, unbounded, mid=(0, 10, tb.lists[0]))
        mid_ids = _pool_run(vx, tb, audios[:1], [([], [])], False, unbounded, mid=(0, 10, tb.lists[0]))
        assert mid_text == mid_ids
        assert mid_text[0][:10] == plain[0][:10] and mid_text[0] != plain[0]
        pool = vx.StreamingPool(m, max_sessions=2, max_seconds=None if unbounded else 12.0)
        try:
            with pytest.raises(vx.VoxtralError) as e:   # a session that is not open
                pool.set_bias_text(1, ["the"], 1.0, tb.tok)
            assert e.value.code == VOX_EINVAL
        finally:
            pool.close()
    finally:
        m.set_bias([], 1.0)
        m.set_delays(DELAYS)


def test_refusals_keep_the_previous_list(vx, tb):
    m, B = tb.model, 3
    tb.apply(B, text=True)
    want = np.asarray(m.transcribe_streaming(tb.mels[:B]))
    words = lambda k: [f"w{j}x" for j in range(k)]   # noqa: E731
    assert len(tb.expand((words(128), [1.0] * 128))[0]) == 256
    long_word = "".join(chr(c) for c in range(14, 31))   # 17 control characters (not White_Space) that never merge
    assert len(tb.enc.encode(long_word)) == 17
    bad = [
        dict(phrases=[""], boost=1.0),                                   # empty phrase
        dict(phrases=["the", b"\xffbad"], boost=1.0),                    # invalid UTF-8
        dict(phrases=["ok", b"\xed\xa0\x80"], boost=1.0),                # a surrogate
        dict(phrases=["the", long_word], boost=1.0),                     # a form longer than 16 ids
        dict(phrases=words(129), boost=1.0),                             # 258 forms
        dict(phrases=["the"], boost=0.0),                                # what set_bias refuses
        dict(phrases=["the"], boost=float("nan")),
        dict(phrases=["the"], boost=1.0, stream=N),
    ]
    for kw in bad:
        with pytest.raises(vx.VoxtralError) as e:
            m.set_bias_text(tokenizer=tb.tok, **kw)
        assert e.value.code == VOX_EINVAL, kw
    with pytest.raises(vx.VoxtralError) as e:
        m.set_bias_text(["ok"] * 3 + [long_word], 1.0, tb.tok)
    assert "phrase 3" in e.value.msg
    # an id outside the model's vocabulary: a tokenizer whose word sits past position 31768
    big = json.loads(json.dumps(tb.doc))
    v = big["vocab"]
    while len(v) < 32000:
        v.append({"rank": len(v), "token_bytes": None, "token_str": f"\x01fill{len(v)}"})
    v.append({"rank": len(v), "token_bytes": None, "token_str": "Quetzalcoatl"})
    big["config"]["default_vocab_size"] = 1000 + len(v)
    big_tok = vx.VoxtralTokenizer.from_json(json.dumps(big))
    assert big_tok.encode("Quetzalcoatl").tolist() == [len(v) - 1 + 1000]
    with pytest.raises(vx.VoxtralError) as e:
        m.set_bias_text(["Quetzalcoatl"], 1.0, big_tok)
    assert e.value.code == VOX_EINVAL
    # a tokenizer that cannot encode
    other = json.loads(json.dumps(tb.doc))
    other["config"]["pattern"] = r"\S+"
    with pytest.raises(vx.VoxtralError) as e:
        m.set_bias_text(["the"], 1.0, vx.VoxtralTokenizer.from_json(json.dumps(other)))
    assert e.value.code == VOX_EFORMAT
    lib = vx.lib()
    one = (ctypes.c_char_p * 1)(b"the")
    b1 = np.ones(1, np.float32)
    assert lib.vox_session_set_bias_text(m._s, 0, None, ctypes.cast(one, ctypes.c_void_p),
                                         b1.ctypes.data_as(ctypes.c_void_p), 1) == VOX_EINVAL   # NULL tokenizer
    assert lib.vox_session_set_bias_text(m._s, 0, tb.tok._h, None, b1.ctypes.data_as(ctypes.c_void_p), 1) == VOX_EINVAL
    assert lib.vox_session_set_bias_text(m._s, 0, tb.tok._h, ctypes.cast(one, ctypes.c_void_p), None, 1) == VOX_EINVAL
    assert lib.vox_session_set_bias_text(m._s, 0, tb.tok._h, None, None, -1) == VOX_EINVAL
    with pytest.raises(ValueError):
        m.set_bias_text(["a\0b"], 1.0, tb.tok)
    # a beam transcription while a text list is set is refused like one with an id list
    m.set_beam(2)
    try:
        with pytest.raises(vx.VoxtralError) as e:
            m.transcribe_streaming(tb.mels[:2])
        assert e.value.code == VOX_EINVAL
    finally:
        m.set_beam(1)
    assert np.array_equal(np.asarray(m.transcribe_streaming(tb.mels[:B])), want)
    m.set_bias([], 1.0)
