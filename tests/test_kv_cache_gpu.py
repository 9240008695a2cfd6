"""Decoder KV pages of a stream pool handed out again (csrc/kv_cache.cu DecoderKv::reserve / release / bind): a pool of
two slots runs more sessions, one after the other with overlapping lifetimes, than its pages could hold without reuse.
A session decodes into pages that earlier sessions wrote and released, and its ids must still be those of
transcribe_pcm of the same audio.  The bounded pool and the unbounded pool (each session's pages a ring) are both
covered.  The model is the tiny model with a decoder window of 48 positions, so the ring is 8 pages."""
import math

import numpy as np
import pytest

from oracle import mel as omel

pytestmark = pytest.mark.gpu

DEC_WINDOW, KV_PAGE, M_MAX = 48, 16, 64
PIECE = 5120                 # samples pushed per tick per session (0.32 s)


@pytest.fixture(scope="module")
def model(vx, tmp_path_factory):
    from voxtral_mini_realtime_rs_b200 import synth
    p = str(tmp_path_factory.mktemp("kv_reuse") / "tiny_w48.gguf")
    synth.write_synthetic_gguf(p, synth.tiny_window_config(DEC_WINDOW), seed=3)
    m = vx.Q4ModelLoader.from_file(p).load(0, max_batch=1, max_mel_frames=2048)
    yield m
    m.close()


def _pages_per_session(vx, max_seconds):
    """Decoder KV pages each session of a pool owns at most (Session::create sizing, DecoderKv::create)."""
    if max_seconds is None:
        return (DEC_WINDOW + M_MAX) // KV_PAGE + 1
    lib = vx.lib()
    t = lib.vox_mel_num_frames(lib.vox_pad_audio_len(math.ceil(max_seconds * 16000), None))
    for _ in range(2):
        t = (t + 2 - 3) // 2 + 1
    return -(-(max(t // 4, M_MAX) + M_MAX) // KV_PAGE)


@pytest.mark.parametrize("max_seconds,lengths", [
    (2.0, [1.9, 1.4, 2.0, 1.6, 1.2, 1.8]),
    (None, [11.0, 5.0, 8.5, 12.0, 4.0]),
], ids=["bounded", "unbounded"])
def test_released_pages_are_reused(vx, model, max_seconds, lengths):
    rng = np.random.default_rng(len(lengths))
    audios = [omel.peak_normalize(omel.speechlike(s, 500 + i)) for i, s in enumerate(lengths)]
    per_session = _pages_per_session(vx, max_seconds)
    pool = vx.StreamingPool(model, max_sessions=2, max_seconds=max_seconds)
    n = len(audios)
    sid, fed, ids, pages = [None] * n, [0] * n, [[] for _ in range(n)], [0] * n
    closed, nxt, opened_at, most_open = [False] * n, 0, 0, 0
    try:
        for tick in range(5000):
            live = [i for i in range(n) if sid[i] is not None and not closed[i]]
            # the next session opens a few ticks after the last one, while that one still runs
            if nxt < n and len(live) < 2 and (nxt == 0 or tick >= opened_at + 3):
                sid[nxt] = pool.open()
                opened_at = tick
                live.append(nxt)
                nxt += 1
            most_open = max(most_open, len(live))
            for i in live:
                if fed[i] < audios[i].size:
                    k = int(rng.integers(PIECE // 2, PIECE * 2))
                    pool.push(sid[i], audios[i][fed[i]:fed[i] + k])
                    fed[i] += k
                    if fed[i] >= audios[i].size:
                        pool.finish(sid[i])
            pool.tick()
            for i in live:
                got, done = pool.poll(sid[i])
                ids[i] += got
                pages[i] = max(pages[i], pool.session_info(sid[i])["kv_pages"])
                if done:
                    pool.close_session(sid[i])
                    closed[i] = True
            if all(closed):
                break
    finally:
        pool.close()
    assert all(closed)
    assert most_open == 2                                   # lifetimes overlapped
    assert sum(pages) > 2 * per_session                     # more pages than the pool has: released pages were reused
    assert all(0 < p <= per_session for p in pages), (pages, per_session)
    if max_seconds is None:
        assert max(pages) == per_session                    # a full ring
    for i, a in enumerate(audios):
        want = model.transcribe_pcm(a, peak_normalize=False)[0].tolist()
        assert ids[i] == want, (i, len(ids[i]), len(want), next((k for k, (x, y) in enumerate(zip(ids[i], want)) if x != y), None))
