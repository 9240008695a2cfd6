"""The f16 decoder KV cache (vox_session_create_ex / vox_stream_pool_create_ex with VOX_DTYPE_F16) on the GPU.

  * API: the _ex form at VOX_DTYPE_F32 is the plain create, bit for bit (ids and logits, tiny model); a bad kv_dtype is
    VOX_EINVAL and leaves no handle; device_bytes(f32) - device_bytes(f16) is exactly half the KV bytes the shapes give,
    for a session and for an unbounded pool.
  * Storage, bitwise: identical ids teacher-forced through an f32 and an f16 session of the tiny model.  Up to layer
    0's K/V store the two sessions compute the same thing, so the f16 session's kv_k0 / kv_v0 must be the clamp + RNE
    of the f32 session's, at prefill and decode positions, on the persistent kernel at B = 1, 3, 8, on mega_off and on
    tc_off.
  * Read path against f64: streams on the decoder-geometry model at windows 8192 and 383, teacher-forced along the f16
    session's own greedy ids; every step's logits within KV16_LOGIT_REL_BOUND (tests/test_kv_half_ref.py) of
    KvHalfOracle(float64), and the device argmax equal to the argmax of the logits.  The f16 tilings the persistent
    kernel reports ("mega_attn") are pinned in TILING16.
  * Beams: every n-best hypothesis of an f16 session, teacher-forced on the same session, sums to its reported score
    (tests/test_beam_gpu.py's fork check: a wrong page copy breaks it).
"""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN
from test_beam_gpu import check_consistent
from test_decode_attn_tiles_ref import RING_POSITIONS, TILING, chunk_tiles
from test_decode_geometry_ref import geometry_model_bytes
from test_delay_rows_ref import delay_mel
from test_kv_half_ref import KV16_LOGIT_REL_BOUND, KvHalfOracle, kv16_from_f32
from test_token_scores_ref import MAX_TOP_K, log_softmax64, score_bound

pytestmark = pytest.mark.gpu

VOX_EINVAL = 1
PREFIX = [1] + [32] * (PREFIX_LEN - 1)
TINY_FRAMES = 2000
# the persistent kernel's attention tiling with an f16 cache, {rows: (keys per tile, key chunks)}: the f16 key takes
# fewer scratch bytes than the f32 one, so the tiles are longer than test_decode_attn_tiles_ref.TILING's
TILING16 = {1: (64, 4), 2: (128, 4), 3: (160, 4), 5: (160, 3), 8: (160, 2)}


def _conv_out(t):
    return (t + 2 - 3) // 2 + 1


def _kv_bytes_f32(info, max_batch, max_pages):
    """Bytes of an f32 KV cache (K and V) of max_batch rows of max_pages pages of 16 positions."""
    return 2 * 4 * info["dec_layers"] * max_batch * max_pages * info["dec_kv_heads"] * 16 * info["dec_head_dim"]


@pytest.fixture(scope="module")
def tiny_audio():
    return np.stack([omel.speechlike(4.0, seed=1234 + i) for i in range(8)])


def test_ex_f32_is_the_plain_create_bitwise(vx, tiny_gguf, tiny_audio):
    lib = vx.lib()
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=2, max_mel_frames=TINY_FRAMES, kv_dtype="f32")
    try:
        got_ex = m.transcribe_pcm(tiny_audio[:2])
        logits_ex = m.debug("logits")
        lib.vox_session_free(m._s)
        m._s = ctypes.c_void_p()
        assert lib.vox_session_create(m._m, 2, TINY_FRAMES, ctypes.byref(m._s)) == 0
        got = m.transcribe_pcm(tiny_audio[:2])
        assert np.array_equal(got, got_ex)
        assert np.array_equal(m.debug("logits").view(np.uint32), logits_ex.view(np.uint32))
    finally:
        m.close()


def test_ex_f32_pool_is_the_plain_pool_bitwise(vx, tiny_gguf, tiny_audio):
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=1, max_mel_frames=TINY_FRAMES)
    lib = vx.lib()
    try:
        out = []
        for ex in (False, True):
            pool = vx.StreamingPool(m, max_sessions=2, max_seconds=None, kv_dtype="f32")
            if not ex:   # swap in a pool made by the plain create
                lib.vox_stream_pool_free(pool._p)
                pool._p = ctypes.c_void_p()
                assert lib.vox_stream_pool_create(m._m, 2, 0.0, ctypes.byref(pool._p)) == 0
            try:
                pool.set_top_k(4)
                sids = [pool.open() for _ in range(2)]
                for s, a in zip(sids, tiny_audio[:2]):
                    pool.push(s, a)
                    pool.finish(s)
                res = [[] for _ in sids]
                for _ in range(1000):
                    pool.tick()
                    done = True
                    for i, s in enumerate(sids):
                        got, d, t, l = pool.poll(s, scores=True)
                        res[i].append((list(got), t.copy(), l.copy()))
                        done = done and d
                    if done:
                        break
                out.append(res)
            finally:
                pool.close()
        for a, b in zip(*out):
            assert [x[0] for x in a] == [x[0] for x in b]
            assert all(np.array_equal(x[1], y[1]) and np.array_equal(x[2].view(np.uint32), y[2].view(np.uint32))
                       for x, y in zip(a, b))
    finally:
        m.close()


def test_bad_kv_dtype_is_einval_and_leaves_no_handle(vx, tiny_gguf):
    lib = vx.lib()
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=1, max_mel_frames=TINY_FRAMES)
    try:
        for bad in (2, -1, 7):
            h = ctypes.c_void_p()
            assert lib.vox_session_create_ex(m._m, 1, TINY_FRAMES, bad, ctypes.byref(h)) == VOX_EINVAL
            assert h.value is None
            assert lib.vox_stream_pool_create_ex(m._m, 1, 0.0, bad, ctypes.byref(h)) == VOX_EINVAL
            assert h.value is None
        with pytest.raises(ValueError):
            vx.StreamingPool(m, max_sessions=1, kv_dtype="bf16")
    finally:
        m.close()


def test_device_bytes_saving_is_half_the_kv_bytes(vx, tiny_gguf):
    loader = vx.Q4ModelLoader.from_file(tiny_gguf)
    B = 3
    m32 = loader.load(0, max_batch=B, max_mel_frames=TINY_FRAMES)
    m16 = loader.load(0, max_batch=B, max_mel_frames=TINY_FRAMES, kv_dtype="f16")
    try:
        info = m32.info
        m_max = max(info["prefix_len"], 64)
        s4 = _conv_out(_conv_out(TINY_FRAMES)) // info["reshape_factor"]
        pages = -(-(max(s4, m_max) + m_max) // 16)
        kv = _kv_bytes_f32(info, B, pages)
        assert m32.device_bytes() - m16.device_bytes() == kv // 2
        p32 = vx.StreamingPool(m32, max_sessions=4, max_seconds=None)
        p16 = vx.StreamingPool(m32, max_sessions=4, max_seconds=None, kv_dtype="f16")
        try:
            ring_pages = (info["dec_window"] + m_max) // 16 + 1
            assert p32.device_bytes() - p16.device_bytes() == _kv_bytes_f32(info, 4, ring_pages) // 2
            print(f"\n[kv16] tiny model: session {m32.device_bytes()} -> {m16.device_bytes()} B, unbounded pool of 4 "
                  f"{p32.device_bytes()} -> {p16.device_bytes()} B")
        finally:
            p32.close()
            p16.close()
    finally:
        m32.close()
        m16.close()


def _teacher_forced_kv(m, mels, seqs, B):
    """Encode streams [0, B), prefill the prefix, decode along seqs; kv_k0 / kv_v0 after the prefill and at the end."""
    m.encode_audio(mels[:B])
    m.reset_cache()
    m.prefill(seqs[:B, :PREFIX_LEN])
    out = [(m.debug("kv_k0"), m.debug("kv_v0"))]
    for p in range(PREFIX_LEN, seqs.shape[1]):
        m.decode_step(tok=seqs[:B, p])
    out.append((m.debug("kv_k0"), m.debug("kv_v0")))
    return out


@pytest.mark.parametrize("path,B", [("mega_auto", 1), ("mega_auto", 3), ("mega_auto", 8), ("mega_off", 3),
                                    ("tc_off", 1)])
def test_layer0_storage_is_clamp_rne_of_f32_bitwise(vx, tiny_gguf, tiny_audio, path, B):
    loader = vx.Q4ModelLoader.from_file(tiny_gguf)
    m32 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES)
    m16 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES, kv_dtype="f16")
    try:
        mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(a)) for a in tiny_audio])
        free = np.asarray(m32.transcribe_streaming(mels)).reshape(8, -1)
        seqs = np.concatenate([np.tile(PREFIX, (8, 1)), free[:, :-1]], 1).astype(np.int32)
        for m in (m32, m16):
            m.debug(path)
        r32, r16 = _teacher_forced_kv(m32, mels, seqs, B), _teacher_forced_kv(m16, mels, seqs, B)
        for (k32, v32), (k16, v16) in zip(r32, r16):
            assert k16.size == k32.size > 0
            for a32, a16 in ((k32, k16), (v32, v16)):
                want = kv16_from_f32(a32)
                assert np.array_equal(a16.astype(np.float16).view(np.uint16), want.view(np.uint16)), \
                    (path, B, int(np.sum(a16.astype(np.float16) != want)))
        print(f"\n[kv16] {path} B={B}: layer 0 K/V of {r16[-1][0].size // B} values per row bitwise clamp + RNE")
    finally:
        m32.close()
        m16.close()


SECONDS = 150.0            # 984 positions: at window 8192 every chunk holds 2 f16 tiles or more at every batch size
GEOM_FRAMES = 15800


class HalfStreams:
    """One window: an f16 session of the decoder-geometry model, the streams' mels, the f16 session's own greedy ids and
    the f16-KV f64 reference logits."""

    def __init__(self, vx, window):
        self.window = window
        self.n = n = 11 if window == 8192 else 8
        data = geometry_model_bytes(window)
        self.data = data
        self.model = vx.Q4ModelLoader.from_bytes(data).load(0, max_batch=n, max_mel_frames=GEOM_FRAMES, kv_dtype="f16")
        self.vocab = self.model.info["vocab"]
        self.mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(SECONDS, 900 + i)))
                                    for i in range(n)])
        emb = self.model.encode_audio(self.mels)
        self.S4 = emb.shape[1]
        free = self.model.transcribe_streaming(self.mels)
        self.seqs = np.concatenate([np.tile(PREFIX, (n, 1)), free], 1).astype(np.int32)
        self.o64 = o64 = KvHalfOracle(data, dtype=torch.float64)
        refs = [_f64_logits(o64, emb[i], self.seqs[i]) for i in range(n)]
        self.ref = np.stack(refs)
        self.ref_max = np.abs(self.ref).max(-1)

    def check(self, B):
        """Streams 0..B-1 teacher-forced; every step checked.  Returns (largest error, "mega_attn" of the last step)."""
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
        assert err.max() <= KV16_LOGIT_REL_BOUND, (self.window, B, PREFIX_LEN - 1 + r, err.max())
        assert np.array_equal(np.asarray(toks).reshape(-1)[:B], logits.argmax(-1)), (self.window, B, r)
        return float(err.max())


def _f64_logits(o64, emb, seq):
    """f16-KV f64 reference logits of positions 37 .. len(seq) - 1 of one stream."""
    t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
    return o64.forward_streaming(None, list(seq), t_embed, audio_embeds=torch.from_numpy(emb)).numpy()[PREFIX_LEN - 1:]


@pytest.fixture(scope="module", params=(8192, 383, 400), ids=lambda w: f"window{w}")
def half_streams(request, vx):
    g = HalfStreams(vx, request.param)
    yield g
    g.model.close()


@pytest.mark.parametrize("path,B", [("mega_auto", 1), ("mega_auto", 2), ("mega_auto", 3), ("mega_auto", 5),
                                    ("mega_auto", 8), ("mega_auto", 11), ("mega_off", 3)])
def test_f16_read_path_vs_f64_reference(half_streams, path, B):
    g = half_streams
    if B > g.n:
        pytest.skip("11 streams only at window 8192")
    g.model.debug(path)
    try:
        worst, tiling = g.check(B)
    finally:
        g.model.debug("mega_auto")
    desc = ""
    if path == "mega_auto":
        groups = tiling.reshape(-1, 4).astype(int)
        assert groups[:, 0].tolist() == [min(8, B - b0) for b0 in range(0, B, 8)], groups   # 11 rows: 8 + 3
        for rows, MT, KT, NC in groups.tolist():
            assert (KT, NC) == TILING16[rows], ("f16 attention tiling changed: update TILING16", rows, KT, NC)
            assert NC == TILING[rows][1] and KT > TILING[rows][0], (rows, KT, NC)
            tiles = [t for t in chunk_tiles(g.S4 - 1, g.window, NC, KT) if t]
            if g.window == 8192:    # the online softmax runs across f16 tiles at every batch size
                assert min(map(len, tiles)) >= 2, (rows, tiles)
            desc += f"; {rows} rows: f16 KT {KT} NC {NC}, tiles per chunk {[len(t) for t in tiles]}"
    else:
        assert tiling is None
    print(f"\n[kv16] window {g.window} {path} B={B}: max |dlogit| / max(1, max|ref|) = {worst:.2e} over "
          f"{g.S4 - PREFIX_LEN + 1} steps (bound {KV16_LOGIT_REL_BOUND:.1e}){desc}")


def test_beam_forks_on_an_f16_session(vx):
    m = vx.Q4ModelLoader.from_bytes(geometry_model_bytes(40)).load(0, max_batch=24, max_mel_frames=2000,
                                                                    kv_dtype="f16")
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
        check_consistent(m, mels, ids, scores, f"f16 b={b} W={W}")
    finally:
        m.close()


def test_f16_ring_pool_wraps_scores_vs_f64_reference(vx, half_streams):
    """An unbounded f16 pool on the window-400 model: 3 sessions of 150 s wrap their 480-position KV ring (the RING = true,
    KV = __half instantiations); each emitted token's top-k log-probabilities against log_softmax of KvHalfOracle(float64)
    run on that session's own embeddings and ids, within score_bound (tests/test_token_scores_ref.py)."""
    g = half_streams
    if g.window != 400:
        pytest.skip("the ring instantiation runs on the window-400 model")
    n = 3
    audios = [omel.peak_normalize(omel.speechlike(SECONDS, 900 + i)) for i in range(n)]
    pool = vx.StreamingPool(g.model, max_sessions=n, max_seconds=None, kv_dtype="f16")
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
        err = np.abs(lp - np.take_along_axis(log_softmax64(ref), top, -1)).max(-1) / score_bound(ref)
        worst = max(worst, float(err.max()))
        assert err.max() <= 1.0, (i, int(np.argmax(err)) + PREFIX_LEN - 1, err.max())
    print(f"\n[kv16] f16 ring pool, window 400, {n} sessions x {infos[0]['decoder_positions']} positions: "
          f"max |dlogprob| = {worst:.2f} x score_bound")


def _scaled_gamma_gguf(path, scale):
    """The tiny model's GGUF with decoder layer 0's attention-norm weight multiplied by `scale` (q, k and v of layer 0
    scale with it)."""
    from oracle.gguf_synth import GgufFile
    data = bytearray(open(path, "rb").read())
    g = GgufFile(bytes(data))
    dt, shape, off = g.tensors["layers.0.attention_norm.weight"]
    assert dt == 0, dt                                           # f32
    a = g.data_off + off
    n = int(np.prod(shape))
    data[a:a + 4 * n] = (np.frombuffer(data[a:a + 4 * n], np.float32) * np.float32(scale)).tobytes()
    return bytes(data)


@pytest.mark.parametrize("path,B", [("mega_auto", 3), ("mega_off", 3), ("tc_off", 1)])
def test_layer0_storage_saturates_to_f16_max_bitwise(vx, tiny_gguf, tiny_audio, path, B):
    """Layer 0's attention-norm weight scaled so that about a third of layer 0's largest K and V values pass 65504: the
    f16 session stores them as +-65504 (never +-inf), bit for bit the clamp + RNE of the f32 session's values, at the
    prefill's positions and the decode steps'."""
    mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(a)) for a in tiny_audio])
    plain = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=8, max_mel_frames=TINY_FRAMES)
    try:
        free = np.asarray(plain.transcribe_streaming(mels)).reshape(8, -1)
        seqs = np.concatenate([np.tile(PREFIX, (8, 1)), free[:, :-1]], 1).astype(np.int32)
        k, v = _teacher_forced_kv(plain, mels, seqs, B)[-1]
        top = max(np.abs(k).max(), np.abs(v).max())
    finally:
        plain.close()
    loader = vx.Q4ModelLoader.from_bytes(_scaled_gamma_gguf(tiny_gguf, 1.5 * 65504.0 / top))
    m32 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES)
    m16 = loader.load(0, max_batch=8, max_mel_frames=TINY_FRAMES, kv_dtype="f16")
    try:
        for m in (m32, m16):
            m.debug(path)
        r32, r16 = _teacher_forced_kv(m32, mels, seqs, B), _teacher_forced_kv(m16, mels, seqs, B)
        saturated = 0
        for (k32, v32), (k16, v16) in zip(r32, r16):
            for a32, a16 in ((k32, k16), (v32, v16)):
                assert np.all(np.isfinite(a32)) and np.all(np.isfinite(a16))
                want = kv16_from_f32(a32)
                assert np.array_equal(a16.astype(np.float16).view(np.uint16), want.view(np.uint16)), (path, B)
                saturated += int(np.sum(np.abs(a32) > 65504.0))
                assert np.all(np.abs(a16[np.abs(a32) > 65504.0]) == 65504.0)
        assert saturated > 0, (path, B)
        print(f"\n[kv16] scaled layer-0 norm, {path} B={B}: {saturated} K/V values past 65504 stored as +-65504")
    finally:
        m32.close()
        m16.close()
