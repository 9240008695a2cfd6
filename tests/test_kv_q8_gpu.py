"""The 8-bit decoder KV cache (vox_session_create_ex / vox_stream_pool_create_ex with VOX_DTYPE_KV_Q8) on the GPU.

  * API: VOX_DTYPE_KV_Q8 creates sessions and pools, and kv_dtype="q8" works; device_bytes(f32) - device_bytes(q8) is
    exactly 23/32 of the f32 KV bytes the shapes give (1.125 bytes per value instead of 4), for a session and for an
    unbounded pool.
  * Storage, bitwise: identical ids teacher-forced through an f32 and a q8 session of the tiny model.  Up to layer 0's
    K/V store the two sessions compute the same thing, so the q8 session's kv_k0 / kv_v0 must be the rule
    (tests/test_kv_q8_ref.py) applied to the f32 session's values, at prefill and decode positions, on the persistent
    kernel at B = 1, 3, 8, on mega_off and on tc_off -- and with layer 0's K/V scaled past 65504 * 127, where scales
    saturate at 65504 and values clamp at +-127.
  * Read path against f64: streams on the decoder-geometry model at windows 8192 and 383, teacher-forced along the q8
    session's own greedy ids; every step's logits within KV8_LOGIT_REL_BOUND of KvQ8Oracle(float64), and the device
    argmax equal to the argmax of the logits.  The q8 tilings the persistent kernel reports ("mega_attn") are pinned in
    TILING8.
  * Ring pool: an unbounded q8 pool wraps its KV ring; its scores match the q8-KV f64 reference past the wrap.
  * Beams: every n-best hypothesis of a q8 session, teacher-forced on the same session, sums to its reported score
    (a fork that forgets the scales breaks it).
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mel as omel
from test_beam_gpu import check_consistent
from test_decode_attn_tiles_ref import RING_POSITIONS, TILING, chunk_tiles
from test_decode_geometry_ref import geometry_model_bytes
from test_delay_rows_ref import delay_mel
from test_kv_half_gpu import (GEOM_FRAMES, PREFIX, PREFIX_LEN, SECONDS, TINY_FRAMES, _conv_out, _f64_logits,
                              _kv_bytes_f32, _scaled_gamma_gguf, _teacher_forced_kv)
from test_kv_q8_ref import KV8_LOGIT_REL_BOUND, KvQ8Oracle, kv8_decode, kv8_quant
from test_token_scores_ref import MAX_TOP_K, log_softmax64

pytestmark = pytest.mark.gpu

VOX_DTYPE_KV_Q8 = 100
# the persistent kernel's attention tiling with a q8 cache, {rows: (keys per tile, key chunks)}: a q8 key and its scales
# take fewer scratch bytes than an f16 one, so the tiles are longer still; the chunks are test_decode_attn_tiles_ref's
TILING8 = {1: (96, 4), 2: (224, 4), 3: (288, 4), 5: (288, 3), 8: (288, 2)}


@pytest.fixture(scope="module")
def tiny_audio():
    return np.stack([omel.speechlike(4.0, seed=1234 + i) for i in range(8)])


def _score_bound(ref):
    """Per row: the largest accepted |log-probability error| of a q8 session, twice its logit bound (the log-softmax's
    normaliser moves by at most the largest logit error)."""
    return 2 * KV8_LOGIT_REL_BOUND * np.maximum(1.0, np.abs(ref).max(-1))


def _rule(a32, hd):
    """The q8 rule applied to f32 values [..., hd]: the decoded f32 values a q8 cache holds."""
    a = np.asarray(a32, np.float32).reshape(-1, hd)
    return kv8_decode(*kv8_quant(a)).reshape(np.shape(a32))


def test_q8_creates_sessions_and_pools(vx, tiny_gguf, tiny_audio):
    lib = vx.lib()
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=1, max_mel_frames=TINY_FRAMES)
    try:
        h = ctypes.c_void_p()
        assert lib.vox_session_create_ex(m._m, 1, TINY_FRAMES, VOX_DTYPE_KV_Q8, ctypes.byref(h)) == 0 and h.value
        lib.vox_session_free(h)
        h = ctypes.c_void_p()
        assert lib.vox_stream_pool_create_ex(m._m, 1, 0.0, VOX_DTYPE_KV_Q8, ctypes.byref(h)) == 0 and h.value
        lib.vox_stream_pool_free(h)
        with pytest.raises(ValueError):
            vx.StreamingPool(m, max_sessions=1, kv_dtype="bf16")
    finally:
        m.close()
    m8 = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=2, max_mel_frames=TINY_FRAMES, kv_dtype="q8")
    try:
        assert m8.transcribe_pcm(tiny_audio[:2]).shape[0] == 2
    finally:
        m8.close()


def test_device_bytes_saving_is_23_32_of_the_f32_kv_bytes(vx, tiny_gguf):
    loader = vx.Q4ModelLoader.from_file(tiny_gguf)
    B = 3
    m32 = loader.load(0, max_batch=B, max_mel_frames=TINY_FRAMES)
    m8 = loader.load(0, max_batch=B, max_mel_frames=TINY_FRAMES, kv_dtype="q8")
    try:
        info = m32.info
        m_max = max(info["prefix_len"], 64)
        s4 = _conv_out(_conv_out(TINY_FRAMES)) // info["reshape_factor"]
        pages = -(-(max(s4, m_max) + m_max) // 16)
        kv = _kv_bytes_f32(info, B, pages)
        assert kv * 23 % 32 == 0 and m32.device_bytes() - m8.device_bytes() == kv * 23 // 32
        p32 = vx.StreamingPool(m32, max_sessions=4, max_seconds=None)
        p8 = vx.StreamingPool(m32, max_sessions=4, max_seconds=None, kv_dtype="q8")
        try:
            ring_pages = (info["dec_window"] + m_max) // 16 + 1
            assert p32.device_bytes() - p8.device_bytes() == _kv_bytes_f32(info, 4, ring_pages) * 23 // 32
            print(f"\n[kv8] tiny model: session {m32.device_bytes()} -> {m8.device_bytes()} B, unbounded pool of 4 "
                  f"{p32.device_bytes()} -> {p8.device_bytes()} B")
        finally:
            p32.close()
            p8.close()
    finally:
        m32.close()
        m8.close()


def _check_storage(m32, m8, mels, seqs, path, B):
    hd = m32.info["dec_head_dim"]
    for m in (m32, m8):
        m.debug(path)
    r32, r8 = _teacher_forced_kv(m32, mels, seqs, B), _teacher_forced_kv(m8, mels, seqs, B)
    for (k32, v32), (k8, v8) in zip(r32, r8):
        assert k8.size == k32.size > 0
        for a32, a8 in ((k32, k8), (v32, v8)):
            want = _rule(a32, hd)
            got = np.asarray(a8, np.float32)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
                (path, B, int(np.sum(got.view(np.uint32) != want.view(np.uint32))))
    return r32, r8


@pytest.mark.parametrize("path,B", [("mega_auto", 1), ("mega_auto", 3), ("mega_auto", 8), ("mega_off", 3),
                                    ("tc_off", 1)])
def test_layer0_storage_is_the_q8_rule_of_f32_bitwise(vx, tiny_gguf, tiny_audio, path, B):
    loader = vx.Q4ModelLoader.from_file(tiny_gguf)
    m32 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES)
    m8 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES, kv_dtype="q8")
    try:
        mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(a)) for a in tiny_audio])
        free = np.asarray(m32.transcribe_streaming(mels)).reshape(8, -1)
        seqs = np.concatenate([np.tile(PREFIX, (8, 1)), free[:, :-1]], 1).astype(np.int32)
        _, r8 = _check_storage(m32, m8, mels, seqs, path, B)
        print(f"\n[kv8] {path} B={B}: layer 0 K/V of {r8[-1][0].size // B} values per row bitwise the q8 rule")
    finally:
        m32.close()
        m8.close()


@pytest.mark.parametrize("path,B", [("mega_auto", 3), ("mega_off", 3), ("tc_off", 1)])
def test_layer0_storage_saturates_scale_and_clamps_bitwise(vx, tiny_gguf, tiny_audio, path, B):
    """Layer 0's attention-norm weight scaled so that layer 0's largest K and V values pass 1.5 x 65504 x 127: their
    blocks store d = 65504 and clamp values past 127.5 x 65504 to +-127, bit for bit the rule of the f32 session's."""
    mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(a)) for a in tiny_audio])
    plain = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=8, max_mel_frames=TINY_FRAMES)
    try:
        free = np.asarray(plain.transcribe_streaming(mels)).reshape(8, -1)
        seqs = np.concatenate([np.tile(PREFIX, (8, 1)), free[:, :-1]], 1).astype(np.int32)
        k, v = _teacher_forced_kv(plain, mels, seqs, B)[-1]
        top = max(np.abs(k).max(), np.abs(v).max())
    finally:
        plain.close()
    loader = vx.Q4ModelLoader.from_bytes(_scaled_gamma_gguf(tiny_gguf, 1.5 * 65504.0 * 127.0 / top))
    m32 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES)
    m8 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES, kv_dtype="q8")
    try:
        r32, r8 = _check_storage(m32, m8, mels, seqs, path, B)
        hd = m32.info["dec_head_dim"]
        saturated = clamped = 0
        for (k32, v32), _ in zip(r32, r8):
            for a32 in (k32, v32):
                assert np.all(np.isfinite(a32))
                q, d = kv8_quant(np.asarray(a32, np.float32).reshape(-1, hd))
                saturated += int(np.sum(d == np.float16(65504.0)))
                clamped += int(np.sum(np.abs(np.asarray(a32, np.float32)) > 127.5 * 65504.0))
        assert saturated > 0 and clamped > 0, (path, B, saturated, clamped)
        print(f"\n[kv8] scaled layer-0 norm, {path} B={B}: {saturated} blocks at d = 65504, {clamped} values clamped")
    finally:
        m32.close()
        m8.close()


class Q8Streams:
    """One window: a q8 session of the decoder-geometry model, the streams' mels, the q8 session's own greedy ids and
    the q8-KV f64 reference logits."""

    def __init__(self, vx, window):
        self.window = window
        self.n = n = 8
        data = geometry_model_bytes(window)
        self.data = data
        self.model = vx.Q4ModelLoader.from_bytes(data).load(0, max_batch=n, max_mel_frames=GEOM_FRAMES, kv_dtype="q8")
        self.vocab = self.model.info["vocab"]
        self.o64 = o64 = KvQ8Oracle(data, dtype=torch.float64)
        if window == 400:   # the ring pool test's model: it runs its own sessions
            return
        self.mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(SECONDS, 900 + i)))
                                    for i in range(n)])
        emb = self.model.encode_audio(self.mels)
        self.S4 = emb.shape[1]
        free = self.model.transcribe_streaming(self.mels)
        self.seqs = np.concatenate([np.tile(PREFIX, (n, 1)), free], 1).astype(np.int32)
        self.ref = np.stack([_f64_logits(o64, emb[i], self.seqs[i]) for i in range(n)])
        self.ref_max = np.abs(self.ref).max(-1)

    def check(self, B):
        m = self.model
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        toks = m.prefill(self.seqs[:B, :PREFIX_LEN])
        worst = self._row(0, B, toks)
        for p in range(PREFIX_LEN, self.S4):
            toks = m.decode_step(tok=self.seqs[:B, p])
            worst = max(worst, self._row(p - PREFIX_LEN + 1, B, toks))
        return worst, m.debug("mega_attn")

    def _row(self, r, B, toks):
        logits = self.model.debug("logits").reshape(B, self.vocab).astype(np.float64)
        err = np.abs(logits - self.ref[:B, r]).max(-1) / np.maximum(1.0, self.ref_max[:B, r])
        assert err.max() <= KV8_LOGIT_REL_BOUND, (self.window, B, PREFIX_LEN - 1 + r, err.max())
        assert np.array_equal(np.asarray(toks).reshape(-1)[:B], logits.argmax(-1)), (self.window, B, r)
        return float(err.max())


@pytest.fixture(scope="module", params=(8192, 383, 400), ids=lambda w: f"window{w}")
def q8_streams(request, vx):
    g = Q8Streams(vx, request.param)
    yield g
    g.model.close()


@pytest.mark.parametrize("path,B", [("mega_auto", 1), ("mega_auto", 2), ("mega_auto", 3), ("mega_auto", 5),
                                    ("mega_auto", 8), ("mega_off", 3)])
def test_q8_read_path_vs_f64_reference(q8_streams, path, B):
    g = q8_streams
    if g.window == 400:
        pytest.skip("the window-400 model serves the ring pool test")
    g.model.debug(path)
    try:
        worst, tiling = g.check(B)
    finally:
        g.model.debug("mega_auto")
    desc = ""
    if path == "mega_auto":
        groups = tiling.reshape(-1, 4).astype(int)
        assert groups[:, 0].tolist() == [min(8, B - b0) for b0 in range(0, B, 8)], groups
        for rows, MT, KT, NC in groups.tolist():
            assert (KT, NC) == TILING8[rows], ("q8 attention tiling changed: update TILING8", rows, KT, NC)
            assert NC == TILING[rows][1], (rows, KT, NC)
            tiles = [t for t in chunk_tiles(g.S4 - 1, g.window, NC, KT) if t]
            desc += f"; {rows} rows: q8 KT {KT} NC {NC}, tiles per chunk {[len(t) for t in tiles]}"
    else:
        assert tiling is None
    print(f"\n[kv8] window {g.window} {path} B={B}: max |dlogit| / max(1, max|ref|) = {worst:.2e} over "
          f"{g.S4 - PREFIX_LEN + 1} steps (bound {KV8_LOGIT_REL_BOUND:.1e}){desc}")


def test_beam_forks_on_a_q8_session(vx):
    m = vx.Q4ModelLoader.from_bytes(geometry_model_bytes(40)).load(0, max_batch=24, max_mel_frames=2000,
                                                                    kv_dtype="q8")
    try:
        b, W = 3, 4
        mels = np.concatenate([delay_mel(i, 5.0) for i in range(b)])
        m.set_beam(W)
        try:
            out = np.asarray(m.transcribe_streaming(mels)).reshape(b, -1)
            ids, scores = m.nbest()
        finally:
            m.set_beam(1)
        assert out.shape[1] > 12 and np.array_equal(ids[:, 0], out)
        check_consistent(m, mels, ids, scores, f"q8 b={b} W={W}")
    finally:
        m.close()


def test_q8_ring_pool_wraps_scores_vs_f64_reference(vx, q8_streams):
    """An unbounded q8 pool on the window-400 model: 3 sessions of 150 s wrap their 480-position KV ring (the RING = true,
    KV = int8_t instantiations); each emitted token's top-k log-probabilities against log_softmax of KvQ8Oracle(float64)
    run on that session's own embeddings and ids, within twice KV8_LOGIT_REL_BOUND."""
    g = q8_streams
    if g.window != 400:
        pytest.skip("the ring instantiation runs on the window-400 model")
    n = 3
    audios = [omel.peak_normalize(omel.speechlike(SECONDS, 900 + i)) for i in range(n)]
    pool = vx.StreamingPool(g.model, max_sessions=n, max_seconds=None, kv_dtype="q8")
    try:
        pool.set_top_k(MAX_TOP_K)
        sids = [pool.open() for _ in range(n)]
        fed, finished = [0] * n, [False] * n
        ids, tops, lps, embs = ([[] for _ in range(n)] for _ in range(4))
        for _ in range(10000):
            for i in range(n):
                if fed[i] < audios[i].size:
                    pool.push(sids[i], audios[i][fed[i]:fed[i] + 32000])
                    fed[i] += 32000
                elif not finished[i]:
                    pool.finish(sids[i])
                    finished[i] = True
            pool.tick()
            done_all = True
            for i in range(n):
                got, done, t, l = pool.poll(sids[i], scores=True)
                ids[i] += got
                tops[i].append(t)
                lps[i].append(l)
                have = sum(e.shape[0] for e in embs[i])
                info = pool.session_info(sids[i])
                if info["audio_embeds"] > have:
                    embs[i].append(pool.audio_embeds(sids[i], first=have, n=info["audio_embeds"] - have))
                done_all = done_all and done
            if done_all:
                break
        infos = [pool.session_info(s) for s in sids]
    finally:
        pool.close()
    worst = 0.0
    for i in range(n):
        top, lp, emb = np.concatenate(tops[i]), np.concatenate(lps[i]), np.concatenate(embs[i])
        assert len(ids[i]) > 900 and infos[i]["decoder_positions"] > RING_POSITIONS   # the KV ring wrapped
        assert top[:, 0].tolist() == ids[i]
        seq = PREFIX + ids[i][:-1]
        ref = _f64_logits(g.o64, np.ascontiguousarray(emb[:len(seq)]), seq).astype(np.float64)
        err = np.abs(lp - np.take_along_axis(log_softmax64(ref), top, -1)).max(-1) / _score_bound(ref)
        worst = max(worst, float(err.max()))
        assert err.max() <= 1.0, (i, int(np.argmax(err)) + PREFIX_LEN - 1, err.max())
    print(f"\n[kv8] q8 ring pool, window 400, {n} sessions x {infos[0]['decoder_positions']} positions: "
          f"max |dlogprob| = {worst:.2f} x the q8 score bound")
