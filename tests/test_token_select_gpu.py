"""Token selection across call sequences: the record of a call's results and the lazy allocation of its device state.

The other GPU tests check token scores, beam search and phrase boosting one call at a time.  Here:
  * a beam transcribe's scores and n-best lists, then an incremental prefill and decode steps at width 1: the scores
    follow the last step, the n-best lists stay those of the transcribe;
  * vox_transcribe_pcm_ragged reports counts over all its streams at equal and at mixed lengths; a later greedy call
    leaves no n-best list, a call at top_k 0 no scores;
  * the score, beam and bias buffers are allocated once, with the same sizes in any order of the setters, and
    set_beam(2) on a fresh session includes the score buffers;
  * a transcribe refused for capacity leaves the previous call's record in place.
"""
import ctypes

import numpy as np
import pytest

from oracle import mel as omel
from oracle.model import PREFIX_LEN
from test_decode_geometry_ref import geometry_model_bytes
from test_token_scores_gpu import check_own_logits

pytestmark = pytest.mark.gpu

PREFIX = [1] + [32] * (PREFIX_LEN - 1)
VOX_EINVAL, VOX_ECAPACITY = 1, 7   # include/voxtral.h
K, W = 4, 2


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def counts(vx, m):
    """(b, n, k) of vox_session_token_scores and (b, w, n) of vox_session_nbest, without reading the arrays."""
    lib = vx.lib()
    s = [ctypes.c_int32() for _ in range(6)]
    assert lib.vox_session_token_scores(m._s, None, None, 0, *map(ctypes.byref, s[:3])) == 0
    assert lib.vox_session_nbest(m._s, None, None, 0, *map(ctypes.byref, s[3:])) == 0
    return tuple(v.value for v in s[:3]), tuple(v.value for v in s[3:])


@pytest.fixture(scope="module")
def tiny(vx, tiny_gguf):
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=4, max_mel_frames=2000)
    audio = np.stack([omel.speechlike(4.0, seed=1234), omel.speechlike(4.0, seed=77)]).astype(np.float32)
    yield m, audio
    m.close()


def test_incremental_calls_replace_scores_and_keep_nbest(tiny):
    m, audio = tiny
    m.set_top_k(K)
    m.set_beam(W)
    out = m.transcribe_pcm(audio)
    n = out.shape[1]
    ids, lp = m.token_scores()
    assert ids.shape == lp.shape == (2, n, K)
    nb_ids, nb_scores = m.nbest()
    assert nb_ids.shape == (2, W, n) and nb_scores.shape == (2, W)
    assert np.array_equal(nb_ids[:, 0], out)

    m.set_beam(1)
    m.encode_audio(np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(a)) for a in audio]))
    m.reset_cache()
    tok = m.prefill(np.tile(PREFIX, (2, 1)).astype(np.int32))
    for _ in range(2):
        tok = m.decode_step(batch=2)
    ids, lp = m.token_scores()
    assert ids.shape == lp.shape == (2, 1, K)
    assert np.array_equal(ids[:, 0, 0], tok)
    check_own_logits(m.debug("logits").reshape(2, 1, -1), ids, lp, "last decode step")
    again_ids, again_scores = m.nbest()
    assert np.array_equal(again_ids, nb_ids) and np.array_equal(again_scores, nb_scores)
    m.set_top_k(0)


def test_ragged_counts_and_later_calls(vx, tiny):
    m, audio = tiny
    m.set_top_k(K)
    m.set_beam(W)
    for lens in ((64000, 64000), (48000, 64000)):
        streams = [audio[i][:lens[i]] for i in range(2)]
        got = m.transcribe_pcm_ragged(streams)
        total = sum(len(g) for g in got)
        assert counts(vx, m) == ((2, total, K), (2, W, total)), lens
    m.set_beam(1)
    m.transcribe_pcm(audio)
    with pytest.raises(vx.VoxtralError) as e:   # the last transcribe ran greedy
        m.nbest()
    assert e.value.code == VOX_EINVAL
    m.set_top_k(0)
    m.transcribe_pcm(audio)
    with pytest.raises(vx.VoxtralError) as e:   # ... and without scores
        m.token_scores()
    assert e.value.code == VOX_EINVAL


def test_refused_transcribe_keeps_the_record(vx, tiny):
    m, audio = tiny
    m.set_top_k(K)
    m.set_beam(W)
    out = m.transcribe_pcm(audio)
    scores, nbest = m.token_scores(), m.nbest()
    lib = vx.lib()
    ids = np.zeros(out.size, np.int32)
    n_out = ctypes.c_int32()
    rc = lib.vox_transcribe_pcm(m._s, ptr(audio), 2, audio.shape[1], 1, ptr(ids), out.size - 1, ctypes.byref(n_out), None)
    assert rc == VOX_ECAPACITY
    for want, got in zip(scores + nbest, m.token_scores() + m.nbest()):
        assert np.array_equal(want, got)
    m.set_beam(1)
    m.set_top_k(0)


def test_device_bytes_in_any_order(vx):
    """Bias ids lie in [1000, vocab): the decoder-geometry model's vocabulary of 32768 holds them."""
    data = geometry_model_bytes(8192)
    loader = vx.Q4ModelLoader.from_bytes(data)
    setters = {
        "top_k": lambda m: m.set_top_k(K),
        "beam": lambda m: m.set_beam(W),
        "bias": lambda m: m.set_bias([[1001, 1002], [1003]], 1.5),
    }
    sessions = [loader.load(0, max_batch=4, max_mel_frames=400) for _ in range(4)]
    try:
        a, b, fresh, scores_only = sessions
        base = a.device_bytes()
        assert all(s.device_bytes() == base for s in sessions)
        for m, order in ((a, ("top_k", "beam", "bias")), (b, ("bias", "beam", "top_k"))):
            for name in order:
                setters[name](m)
                once = m.device_bytes()
                setters[name](m)
                assert m.device_bytes() == once, name   # a repeated call allocates nothing
        assert a.device_bytes() == b.device_bytes() > base
        fresh.set_beam(W)
        scores_only.set_top_k(K)
        score_bytes = scores_only.device_bytes() - base
        scores_only.set_beam(W)
        assert score_bytes > 0
        assert fresh.device_bytes() == scores_only.device_bytes()   # set_beam allocated the score buffers too
    finally:
        for s in sessions:
            s.close()
