"""Phrase boosting on the device (vox_session_set_bias, vox_stream_set_bias; rule in tests/bias_reference.py).

Model: the decoder-geometry model (vocab 32768) at decoder windows 40 and 8192, 11 streams at the mixed delays of
test_delay_rows_gpu.  The phrases are built from an unboosted run's runner-up ids (token scores), with boosts near the
top-2 margins, so that they flip decisions; every run asserts that they do.

1. The decision rule, bit for bit, on the device's own logits: an incremental prefill, then free-running decode steps
   at B = 1, 3, 8, 11 with different lists on different streams (some empty), on the persistent kernel and both per-op
   paths.  After every call each row's emitted id must be bias_reference's choice from debug("logits") and the history
   tracked here.  The token scores of every step are the top-k of those same unboosted logits.
2. Rows without a list emit exactly the ids of the same call with no list at all; setting and clearing gives them back.
3. transcribe_streaming (graph-replayed) gives test 1's ids; another call with other lists replays the same graph and
   equals a fresh session.
4. transcribe_pcm_ragged with per-stream lists equals each stream's own transcribe_pcm.
5. Streaming pools (bounded, unbounded, per-op): a list set before the first tick gives transcribe_pcm's boosted ids;
   a list set mid-stream leaves every id polled before unchanged; a reused slot starts without a list.
6. One extra launch per prefill and decode step while a list is set, none without.
7. Every VOX_EINVAL case leaves the session usable with its previous list.
"""
import ctypes

import numpy as np
import pytest

import bias_reference as br
from oracle import mel as omel
from test_decode_geometry_ref import geometry_model_bytes
from test_delay_rows_gpu import MEL_FRAMES, N, PREFIX, VOX_EINVAL
from test_delay_rows_ref import DELAYS, delay_mel
from test_token_scores_gpu import check_own_logits

pytestmark = pytest.mark.gpu

K = 4   # token scores kept while testing: the runner-ups and check_own_logits


def make_lists(top_ids, top_lp, rng):
    """Per stream, phrases of 1..4 runner-up ids of consecutive positions (text ids only) with boosts around the margin
    at their first position; streams 2, 5, 8 (i % 3 == 2) get no list."""
    lists = []
    for i in range(top_ids.shape[0]):
        if i % 3 == 2:
            lists.append(([], []))
            continue
        phrases, betas = [], []
        n = top_ids.shape[1]
        for p in range(i % 4, n - 4, 3 + i % 3):
            L = 1 + (p + i) % 4
            ph = [int(t) for t in top_ids[i, p:p + L, 1] if t >= br.FIRST_TEXT_ID]
            if not ph:
                continue
            margin = float(top_lp[i, p, 0] - top_lp[i, p, 1])
            phrases.append(ph)
            betas.append(np.float32(max(1e-3, margin * rng.uniform(0.6, 1.8))))
        lists.append((phrases[:br.MAX_PHRASES], betas[:br.MAX_PHRASES]))
    return lists


class Biased:
    def __init__(self, vx, window):
        self.vx = vx
        self.window = window
        self.data = geometry_model_bytes(window)
        self.model = m = vx.Q4ModelLoader.from_bytes(self.data).load(0, max_batch=N, max_mel_frames=MEL_FRAMES)
        self.vocab = m.info["vocab"]
        self.mels = np.concatenate([delay_mel(i) for i in range(N)])
        m.set_delays(DELAYS)
        m.set_top_k(K)
        self.free = np.asarray(m.transcribe_streaming(self.mels))
        top_ids, top_lp = m.token_scores()
        self.lists = make_lists(top_ids, top_lp, np.random.default_rng(window))
        assert sum(len(p) for p, _ in self.lists) > 20

    def apply(self, B, lists=None):
        """Stream i < B gets lists[i] (every other stream none)."""
        lists = self.lists if lists is None else lists
        self.model.set_bias([], 1.0)
        for i in range(B):
            if lists[i][0]:
                self.model.set_bias(lists[i][0], lists[i][1], stream=i)

    def incremental(self, B, lists=None, check=True):
        """Prefill + free-running decode steps over streams [0, B); with check, every row's id against the rule on the
        step's own logits, and the token scores against those logits.  Returns ids [B][n] and launches per call."""
        lists = self.lists if lists is None else lists
        m = self.model
        ref = [br.Stream(*lists[i]) for i in range(B)]
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        n0 = m.launch_count()
        toks = [m.prefill(np.tile(PREFIX, (B, 1)).astype(np.int32))]
        launches = [m.launch_count() - n0]
        out_steps = self.free.shape[1] - 1
        for step in range(out_steps + 1):
            if check:
                logits = m.debug("logits").reshape(B, self.vocab)
                want = [ref[i].emit(logits[i]) for i in range(B)]
                assert toks[-1].tolist() == want, (self.window, B, step)
                ids, lp = m.token_scores()
                check_own_logits(logits[:, None], ids, lp, (self.window, B, step))
            if step == out_steps:
                break
            n0 = m.launch_count()
            toks.append(m.decode_step(batch=B))
            launches.append(m.launch_count() - n0)
        return np.stack(toks, 1), np.array(launches)


@pytest.fixture(scope="module", params=(40, 8192), ids=lambda w: f"window{w}")
def biased(request, vx):
    g = Biased(vx, request.param)
    yield g
    g.model.close()


def flips(ids, free, lists):
    return sum(int(np.sum(ids[i] != free[i])) for i in range(ids.shape[0]) if lists[i][0])


@pytest.mark.parametrize("B", [1, 3, 8, 11])
@pytest.mark.parametrize("path", ["mega_auto", "mega_off", "tc_off"])
def test_rule_on_own_logits(biased, path, B):
    m = biased.model
    m.debug(path)
    try:
        biased.apply(B)
        ids, _ = biased.incremental(B)
        m.set_bias([], 1.0)
        plain, _ = biased.incremental(B, lists=[([], [])] * N, check=False)
    finally:
        m.debug("tc_on" if path == "tc_off" else "mega_auto")
    n_flip = flips(ids, plain, biased.lists)
    print(f"\n[bias] window {biased.window} {path} B={B}: {n_flip} of {ids.size} positions flipped")
    assert n_flip >= (3 if B < 3 else 10), (path, B)
    for i in range(B):   # rows without a list: the ids of the call without lists
        if not biased.lists[i][0]:
            assert np.array_equal(ids[i], plain[i]), (path, B, i)


def test_offline_equals_incremental_and_graph_replay(biased, vx):
    m, B = biased.model, 8
    m.set_bias([], 1.0)
    plain = np.asarray(m.transcribe_streaming(biased.mels[:B]))
    biased.apply(B)
    inc, _ = biased.incremental(B, check=False)
    off = np.asarray(m.transcribe_streaming(biased.mels[:B]))   # graph captured with the kernel in it
    assert np.array_equal(off, inc)
    # other lists, same StepKey: the captured graph replays and reads the new lists in place
    other = [biased.lists[(i + 1) % N] for i in range(N)]
    biased.apply(B, other)
    again = np.asarray(m.transcribe_streaming(biased.mels[:B]))
    fresh = vx.Q4ModelLoader.from_bytes(biased.data).load(0, max_batch=N, max_mel_frames=MEL_FRAMES)
    try:
        fresh.set_delays(DELAYS)
        fresh.set_top_k(K)
        for i in range(B):
            if other[i][0]:
                fresh.set_bias(other[i][0], other[i][1], stream=i)
        assert np.array_equal(again, np.asarray(fresh.transcribe_streaming(biased.mels[:B])))
    finally:
        fresh.close()
    # setting and then clearing every list gives the unboosted ids back
    m.set_bias([], 1.0)
    assert np.array_equal(np.asarray(m.transcribe_streaming(biased.mels[:B])), plain)
    assert flips(off, plain, biased.lists) >= 10


def test_launches(biased):
    m, B = biased.model, 3
    biased.apply(B)
    _, on = biased.incremental(B, check=False)
    m.set_bias([], 1.0)
    _, off = biased.incremental(B, check=False)
    assert np.all(on - off == 1), (on - off)


def test_ragged_per_stream_lists(biased):
    if biased.window != 40:
        pytest.skip("one window is enough for the row-to-stream map")
    m = biased.model
    audios = [omel.peak_normalize(omel.speechlike(s, 870 + i)) for i, s in enumerate((6.0, 4.5, 7.5, 5.0, 6.5))]
    lists = [biased.lists[j] for j in (0, 2, 1, 4, 3)]   # stream 1 without a list
    m.set_delay(6.0)
    try:
        m.set_bias([], 1.0)
        for i, (ph, be) in enumerate(lists):
            if ph:
                m.set_bias(ph, be, stream=i)
        got = m.transcribe_pcm_ragged(audios, peak_normalize=False)
        total = 0
        for i, a in enumerate(audios):
            m.set_bias([], 1.0)
            if lists[i][0]:
                m.set_bias(*lists[i], stream=0)
            one = m.transcribe_pcm(a, peak_normalize=False)[0]
            assert np.array_equal(got[i], one), i
            m.set_bias([], 1.0)
            total += int(np.sum(one != m.transcribe_pcm(a, peak_normalize=False)[0]))
        assert total >= 5
    finally:
        m.set_bias([], 1.0)
        m.set_delays(DELAYS)


def _pool_run(vx, model, audios, lists, unbounded, mid=None):
    """Sessions opened at tick 0 with lists[i] set before their first tick; mid = (session index, ids polled, list): set
    once that session has polled that many ids.  Returns per session the ids and, for mid, how many ids it had polled
    before the list changed."""
    pool = vx.StreamingPool(model, max_sessions=len(audios), max_seconds=None if unbounded else 12.0)
    n = len(audios)
    sids = [pool.open() for _ in range(n)]
    for s, (ph, be) in zip(sids, lists):
        if ph:
            pool.set_bias(s, ph, be)
    fed, ids, before = [0] * n, [[] for _ in range(n)], None
    try:
        for tick in range(2000):
            if mid is not None and before is None and len(ids[mid[0]]) >= mid[1]:
                before = len(ids[mid[0]])
                pool.set_bias(sids[mid[0]], *mid[2])
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
        return pool, sids, ids, before
    except Exception:
        pool.close()
        raise


@pytest.mark.parametrize("unbounded", [False, True], ids=["bounded", "unbounded"])
@pytest.mark.parametrize("mega", [True, False], ids=["mega", "mega_off"])
def test_streaming_pool(vx, biased, monkeypatch, unbounded, mega):
    if biased.window != 40:
        pytest.skip("one window is enough for the pool's bookkeeping")
    if not mega:
        monkeypatch.setenv("VOX_MEGA", "0")   # the pool's session reads it when it is created
    m = biased.model
    audios = [omel.peak_normalize(omel.speechlike(s, 810 + i)) for i, s in enumerate((5.0, 6.5, 4.0, 5.5))]
    lists = [biased.lists[0], ([], []), biased.lists[1], biased.lists[3]]
    m.set_delay(6.0)

    def offline(a, lst):
        m.set_bias([], 1.0)
        if lst[0]:
            m.set_bias(*lst, stream=0)
        out = m.transcribe_pcm(a, peak_normalize=False)[0].tolist()
        m.set_bias([], 1.0)
        return out

    try:
        want = [offline(a, l) for a, l in zip(audios, lists)]
        plain = [offline(a, ([], [])) for a in audios]
        assert sum(w != p for w, p in zip(want, plain)) >= 2
        pool, sids, ids, _ = _pool_run(vx, m, audios, lists, unbounded)
        try:
            assert ids == want
            # a reused slot starts without a list
            pool.close_session(sids[0])
            reuse = pool.open()
            assert reuse == sids[0]
            pool.push(reuse, audios[0])
            pool.finish(reuse)
            got = []
            for _ in range(50):
                pool.tick()
                part, done = pool.poll(reuse)
                got += part
                if done:
                    break
            assert got == plain[0]
            with pytest.raises(vx.VoxtralError) as e:   # a session that is not open
                pool.set_bias(len(audios) + 3, *lists[0])
            assert e.value.code == VOX_EINVAL
        finally:
            pool.close()
        # a list set in mid-stream on an unboosted session: the ids polled before it are the unboosted ones
        pool, sids, ids, before = _pool_run(vx, m, audios[1:2], [([], [])], unbounded, mid=(0, 10, lists[0]))
        pool.close()
        assert 0 < before < len(plain[1])
        assert ids[0][:before] == plain[1][:before]
        assert len(ids[0]) == len(plain[1])
    finally:
        m.set_bias([], 1.0)
        m.set_delays(DELAYS)


def test_invalid_arguments_keep_the_previous_list(biased, vx):
    m, B = biased.model, 3
    biased.apply(B)
    want = np.asarray(m.transcribe_streaming(biased.mels[:B]))
    V = biased.vocab
    bad = [
        dict(phrases=[[1001]], boost=1.0, stream=N),          # unknown stream
        dict(phrases=[[1001]], boost=1.0, stream=-2),
        dict(phrases=[[1001]] * 257, boost=1.0),               # too many phrases
        dict(phrases=[[]], boost=1.0),                         # length 0
        dict(phrases=[[1001] * 17], boost=1.0),                # length 17
        dict(phrases=[[999]], boost=1.0),                      # a special id
        dict(phrases=[[V]], boost=1.0),                        # past the vocabulary
        dict(phrases=[[1001]], boost=0.0),                     # boosts must be > 0 and finite
        dict(phrases=[[1001]], boost=-1.0),
        dict(phrases=[[1001]], boost=float("nan")),
        dict(phrases=[[1001]], boost=float("inf")),
    ]
    for kw in bad:
        with pytest.raises(vx.VoxtralError) as e:
            m.set_bias(**kw)
        assert e.value.code == VOX_EINVAL, kw
    lib = vx.lib()
    assert lib.vox_session_set_bias(m._s, 0, None, None, None, 1) == VOX_EINVAL   # NULL buffers with a phrase
    one = np.array([1], np.int32)
    assert lib.vox_session_set_bias(m._s, 0, None, one.ctypes.data_as(ctypes.c_void_p), None, 1) == VOX_EINVAL
    # a beam transcription while a list is set is refused before any device work
    m.set_beam(2)
    try:
        with pytest.raises(vx.VoxtralError) as e:
            m.transcribe_streaming(biased.mels[:2])
        assert e.value.code == VOX_EINVAL
        with pytest.raises(vx.VoxtralError) as e:
            m.transcribe_pcm_ragged([omel.speechlike(4.0, 1), omel.speechlike(5.0, 2)])
        assert e.value.code == VOX_EINVAL
    finally:
        m.set_beam(1)
    assert np.array_equal(np.asarray(m.transcribe_streaming(biased.mels[:B])), want)
    m.set_bias([], 1.0)
