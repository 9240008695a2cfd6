"""Beam search on the GPU (vox_session_set_beam, vox_session_nbest).

  * against the reference beam search (tests/beam_reference.py, OracleModel in float64) on the tiny model, three streams
    at mixed delays, b x W = 2, 8, 12 and 24 rows (more than one group of 8, and a ragged last group), with the
    persistent kernel, the per-op path and eager steps: the n-best ids equal the reference wherever every selection
    margin and the final rank margins exceed twice the accumulated score bound; elsewhere the rank-0 score is at least
    the reference's best minus that bound;
  * fork correctness without a reference, on the decoder-geometry model at windows 40 and 8192: every returned
    hypothesis, teacher-forced through vox_prefill / vox_decode_step at width 1, sums to its reported score.  A wrongly
    shared or partly copied KV page changes those logits;
  * width 1 is the greedy path bitwise, and a beam call leaves the session as a fresh one would be.
"""
import ctypes

import numpy as np
import pytest
import torch

from beam_reference import log_softmax64, oracle_beam
from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import geometry_model_bytes
from test_delay_rows_ref import DELAYS, delay_mel
from test_token_scores_ref import score_bound

pytestmark = pytest.mark.gpu

PREFIX = [1] + [32] * (PREFIX_LEN - 1)
VOX_EINVAL, VOX_ECAPACITY = 1, 7   # include/voxtral.h
STREAMS = 3
MAX_ROWS = 24
SHAPES = [(1, 2), (1, 8), (3, 4), (3, 8)]   # (b, W): 2, 8, 12 and 24 rows


def tiny_mels(seconds=4.0):
    return np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(seconds, 60 + i)))
                           for i in range(STREAMS)])


def teacher_forced_scores(m, hyps, k=0):
    """hyps [b][n] fed through prefill / decode_step at width 1 over the embeddings resident in the session: per row the
    sum of log_softmax over the GPU's own logits of its ids, and (k > 0) the token scores [b][n][k]."""
    b, n = hyps.shape
    m.set_top_k(k)
    m.reset_cache()
    m.prefill(np.tile(PREFIX, (b, 1)).astype(np.int32))
    total = np.zeros(b)
    ids, lps = [], []
    for j in range(n):
        lg = m.debug("logits").reshape(b, -1)
        total += log_softmax64(lg)[np.arange(b), hyps[:, j]]
        if k:
            t = m.token_scores()
            ids.append(t[0])
            lps.append(t[1])
        if j + 1 < n:
            m.decode_step(tok=hyps[:, j])
    m.set_top_k(0)
    return total, (np.concatenate(ids, 1), np.concatenate(lps, 1)) if k else None


def check_consistent(m, mels, ids, scores, what):
    """Every hypothesis sums to its reported score over the GPU's own teacher-forced logits."""
    b, W, n = ids.shape
    m.set_beam(1)
    m.encode_audio(mels[:b])
    for w in range(W):
        total, _ = teacher_forced_scores(m, ids[:, w])
        err = np.abs(total - scores[:, w]).max()
        assert err <= 1e-4 * n, (what, w, err)
    assert np.all(np.diff(scores, axis=1) <= 0), what
    for s in range(b):
        assert len({tuple(r) for r in ids[s]}) == W, (what, s)


class Tiny:
    def __init__(self, vx, tiny_gguf):
        self.m = m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=MAX_ROWS, max_mel_frames=2000)
        m.set_delays(DELAYS[:STREAMS])
        self.mels = tiny_mels()
        emb = m.encode_audio(self.mels)
        self.S4 = emb.shape[1]
        o = OracleModel(tiny_gguf, dtype=torch.float64)
        self.ref = {}
        for W in sorted({w for _, w in SHAPES}):
            for s in range(STREAMS):
                rec = {}
                ids, sc = oracle_beam(o, emb[s], omel.time_embedding(DELAYS[s], o.cfg.dec_dim), W, rec)
                bounds = np.array([score_bound(r).max() for r in rec["logits"]])
                self.ref[W, s] = (ids, sc, rec["margins"], np.cumsum(bounds))


@pytest.fixture(scope="module")
def tiny(vx, tiny_gguf):
    t = Tiny(vx, tiny_gguf)
    yield t
    t.m.close()


@pytest.mark.parametrize("path", ["mega_auto", "mega_off", "graph_off"])
@pytest.mark.parametrize("b,W", SHAPES)
def test_against_reference(tiny, path, b, W):
    m = tiny.m
    assert tiny.S4 > PREFIX_LEN + 12   # positions 47, 48 and 49: forks at pos % 16 = 15, 0 and 1
    m.debug(path)
    try:
        m.set_beam(W)
        out = np.asarray(m.transcribe_streaming(tiny.mels[:b])).reshape(b, -1)
        ids, scores = m.nbest()
    finally:
        m.set_beam(1)
        m.debug("graph_on" if path == "graph_off" else "mega_auto")
    n = out.shape[1]
    assert ids.shape == (b, W, n) and scores.shape == (b, W)
    assert np.array_equal(ids[:, 0], out)
    exact = 0
    for s in range(b):
        r_ids, r_sc, margins, acc = tiny.ref[W, s]
        sure = all(mg[W - 1] > 2 * a for mg, a in zip(margins, acc) if len(mg) >= W) and \
            np.all(margins[-1] > 2 * acc[-1])
        if sure:
            exact += 1
            assert np.array_equal(ids[s], r_ids), (path, b, W, s)
            assert np.abs(scores[s] - r_sc).max() <= acc[-1], (path, b, W, s)
        else:
            assert scores[s, 0] >= r_sc[0] - acc[-1], (path, b, W, s, scores[s, 0], r_sc[0])
    print(f"\n[beam] tiny {path:>9s} b={b} W={W}: {exact}/{b} streams decided beyond the bound, n-best equal to the f64 "
          f"reference")
    check_consistent(m, tiny.mels, ids, scores, f"{path} b={b} W={W}")


def test_width_one_is_greedy_bitwise(vx, tiny_gguf, tiny):
    fresh = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=MAX_ROWS, max_mel_frames=2000)
    try:
        fresh.set_delays(DELAYS[:STREAMS])

        def run(mm):
            out = []
            for _ in range(2):
                n0 = mm.launch_count()
                ids = mm.transcribe_streaming(tiny.mels)
                out.append((ids, mm.debug("logits").copy(), mm.launch_count() - n0))
            return out

        base = run(fresh)
        m = tiny.m
        m.set_beam(4)
        m.transcribe_streaming(tiny.mels[:2])
        m.set_beam(1)
        got = run(m)
        for (i0, l0, n0), (i1, l1, n1) in zip(base, got):
            assert np.array_equal(i0, i1) and np.array_equal(l0, l1)
        assert base[1][2] == got[1][2]   # a replayed step: the same launches
        # the incremental API after a beam call and a reset: the fresh session's ids
        m.set_beam(4)
        m.transcribe_streaming(tiny.mels[:2])
        assert m.cache_len() == 0
        m.set_beam(1)
        for mm in (fresh, m):
            mm.encode_audio(tiny.mels)
            mm.reset_cache()
        seq = [(fresh.prefill(np.tile(PREFIX, (STREAMS, 1)).astype(np.int32)),
                m.prefill(np.tile(PREFIX, (STREAMS, 1)).astype(np.int32)))]
        for _ in range(tiny.S4 - PREFIX_LEN - 1):
            seq.append((fresh.decode_step(batch=STREAMS), m.decode_step(batch=STREAMS)))
        for a, c in seq:
            assert np.array_equal(a, c)
        assert np.array_equal(np.stack([a for a, _ in seq], 1), base[0][0])
    finally:
        fresh.close()


def test_gathered_token_scores(tiny):
    m = tiny.m
    m.set_beam(4)
    m.set_top_k(8)
    try:
        out = np.asarray(m.transcribe_streaming(tiny.mels)).reshape(STREAMS, -1)
        top_ids, top_lp = m.token_scores()
    finally:
        m.set_beam(1)
        m.set_top_k(0)
    assert top_ids.shape == (STREAMS, out.shape[1], 8)
    m.encode_audio(tiny.mels)
    _, (r_ids, r_lp) = teacher_forced_scores(m, out, k=8)
    assert np.abs(top_lp - r_lp).max() <= 1e-4
    gap = -np.diff(r_lp, axis=-1) > 1e-4   # ids agree where neighbouring ranks are apart
    sure = np.concatenate([gap[..., :1], gap[..., 1:] & gap[..., :-1]], -1)
    assert np.array_equal(top_ids[..., :7][sure], r_ids[..., :7][sure])


def test_errors(vx, tiny):
    m = tiny.m
    for w in (0, -1, 9):
        with pytest.raises(vx.VoxtralError) as e:
            m.set_beam(w)
        assert e.value.code == VOX_EINVAL, w
    m.set_beam(1)
    m.transcribe_streaming(tiny.mels[:1])
    with pytest.raises(vx.VoxtralError) as e:     # the last transcribe ran greedy
        m.nbest()
    assert e.value.code == VOX_EINVAL
    m.set_beam(8)
    with pytest.raises(vx.VoxtralError) as e:     # b x W = 32 > max_batch
        m.transcribe_streaming(np.concatenate([tiny.mels, tiny.mels[:1]]))
    assert e.value.code == VOX_EINVAL
    m.set_beam(2)
    try:
        out = np.asarray(m.transcribe_streaming(tiny.mels[:2])).reshape(2, -1)
        lib = vx.lib()
        need = out.size * 2
        ids, sc = np.empty(need, np.int32), np.empty(4, np.float64)
        b, w, n = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        assert lib.vox_session_nbest(m._s, ptr(ids), ptr(sc), need - 1, ctypes.byref(b), ctypes.byref(w),
                                     ctypes.byref(n)) == VOX_ECAPACITY
        assert lib.vox_session_nbest(m._s, ptr(ids), ptr(sc), need, ctypes.byref(b), ctypes.byref(w), ctypes.byref(n)) == 0
        assert (b.value, w.value, n.value) == (2, 2, out.shape[1])
        m.encode_audio(tiny.mels[:2])
        with pytest.raises(vx.VoxtralError) as e:
            m.prefill(np.tile(PREFIX, (2, 1)).astype(np.int32))
        assert e.value.code == VOX_EINVAL
        with pytest.raises(vx.VoxtralError) as e:
            m.decode_step(tok=np.zeros(2, np.int32))
        assert e.value.code == VOX_EINVAL
    finally:
        m.set_beam(1)


@pytest.fixture(scope="module", params=(40, 8192), ids=lambda w: f"window{w}")
def geometry(request, vx):
    m = vx.Q4ModelLoader.from_bytes(geometry_model_bytes(request.param)).load(0, max_batch=MAX_ROWS, max_mel_frames=2000)
    m.set_delays(DELAYS[:STREAMS])
    yield m
    m.close()


@pytest.mark.parametrize("b,W", [(3, 4), (1, 8), (3, 8)])
def test_fork_consistency_decoder_geometry(geometry, b, W):
    mels = np.concatenate([delay_mel(i, 5.0) for i in range(b)])
    m = geometry
    m.set_beam(W)
    try:
        out = np.asarray(m.transcribe_streaming(mels)).reshape(b, -1)
        ids, scores = m.nbest()
    finally:
        m.set_beam(1)
    assert out.shape[1] > 12
    assert np.array_equal(ids[:, 0], out)
    check_consistent(m, mels, ids, scores, f"geometry b={b} W={W}")


@pytest.mark.slow
def test_full_size_goldens_width_four(vx, full_gguf):
    import os
    from voxtral_mini_realtime_rs_b200 import synth
    here = os.path.dirname(os.path.abspath(__file__))
    m = vx.Q4ModelLoader.from_file(full_gguf).load(0, max_batch=8, max_mel_frames=2400)
    try:
        for name in ("full_s42_16s.npz", "full_s42_16s_b.npz"):
            gold = np.load(os.path.join(here, "golden", name))
            audio = synth.speechlike(float(gold["seconds"]), seed=int(gold["audio_seed"]) if "audio_seed" in gold else 1234)
            greedy = m.transcribe_pcm(audio)
            m.set_beam(4)
            try:
                out = m.transcribe_pcm(audio)
                ids, scores = m.nbest()
            finally:
                m.set_beam(1)
            gold_ids = np.asarray(gold["tokens"], np.int32)[None]
            m.transcribe_pcm(audio)   # leaves this utterance's embeddings resident
            g_score, _ = teacher_forced_scores(m, gold_ids)
            n = out.shape[1]
            print(f"\n[beam] full size {name}: W=4 rank-0 {scores[0, 0]:.3f} vs golden greedy {g_score[0]:.3f}; "
                  f"{int((out[0] != gold_ids[0]).sum())}/{n} positions differ from greedy "
                  f"({int((greedy[0] != gold_ids[0]).sum())} for this run's greedy)")
            assert scores[0, 0] >= g_score[0] - 1e-4 * n
            total, _ = teacher_forced_scores(m, ids[:, 0])
            assert abs(total[0] - scores[0, 0]) <= 1e-4 * n
    finally:
        m.close()
