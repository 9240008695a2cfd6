"""The audio encoder, adapter and streaming encoder at the production encoder geometry against a float64 reference, with
the encoder's sliding window biting.

Model: synth.encoder_geometry_config -- the production encoder layer (1280, 32 x 64 heads, FFN 5120) at 2 layers, the
production adapter (5120 -> 3072 -> 3072) and the decoder-geometry decoder -- at encoder windows
  750 (production; 750 mod 64 = 46: the mask edge falls inside a 64-key tile of both attention kernels; K/V ring of
      750 + 256 = 1006 slots),
   64 (the mask edge on a key-tile boundary; ring of 320 slots),
    1 (the window bites at every position, 2 keys per query; ring of 257 = max_new + 1 slots, the tightest possible).

Every comparison is max |GPU - f64| / max(1, max |f64|) over the compared tensor, printed; the bounds and their
justification (sensitivity to a one-key window error, to a lost low f16 piece) are in test_encoder_geometry_ref.py.

  * Offline encode_audio, layer by layer (debug capture): each stage is compared with the f64 reference of that stage
    fed the GPU's own input to it -- conv stem of the mel, each layer of the GPU's previous layer, final norm of the
    GPU's last layer, adapter of the GPU's encoder output -- and the embeddings with the f64 encode_audio of the mel.
    Inputs: 60 s of mel (T = 6000, S = 1500), a ragged length (S = 995: not a multiple of 64 or 128, > 751) and a
    single query tile (S = 50); paths: tensor-core attention + wgmma GEMM at B = 1 and 3, SIMT attention at B = 1 and
    3, SIMT GEMM at B = 1; and S = 250 at B = 1, which reaches the wgmma GEMM's split-K (below).
  * Streaming pools (vox_stream_*): 45-60 s sessions fed 80 ms (2 encoder rows) per tick (tensor-core matvec with bias + RESIDUAL /
    SILU_MUL / NONE epilogues at K = 1280, 2048, 5120 and the adapter's GELU matvec), two sessions opened at different
    ticks, five sessions (wgmma GEMM with split-K at encoder N), one session fed 12 s at once (passes of 256 rows: the
    ring at capacity), and the SIMT matvec / GEMM.  Embeddings against the f64 encode_audio of the GPU's own mel.
  * encode_audio_with_cache (vox_stream_encode_chunk): chunks of 400, 1100 and 3000 mel frames into one session.
  * An unbounded session of 180 s at window 750: past encoder frame 4096 (the model's RoPE table), through the
    per-session encoder RoPE ring and several slides of the 30 s buffers, against the f64 suffix reference.
  * Slow: the full-size model (32 layers), one 60 s utterance layer by layer.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import OracleModel
from suffix_reference import enc_warmup_positions, suffix_reference
from test_encoder_geometry_ref import (ADAPTER_REL_BOUND, EMBED_REL_BOUND, ENC_LAYER_REL_BOUND, WGMMA_LAYER_REL_BOUND,
                                       WINDOWS, encoder_geometry_bytes, geometry_mel, rel_err)

pytestmark = pytest.mark.gpu

MEL_FRAMES = 6000
MAX_BATCH = 3
# mel frames -> encoder frames S = conv_out(conv_out(T)), conv_out(t) = (t - 1) // 2 + 1
INPUTS = {"S1500": 6000, "S995": 3979, "S50": 200}
PATHS = [("tc", 1), ("tc", 3), ("enc_attn_simt", 1), ("enc_attn_simt", 3), ("gemm_simt", 1)]
# S = 250, B = 1: the wgmma GEMM's output tiles for N = 1280 are (1280 / 128) x ceil(250 / 128) = 20 < 132 * 2 / 3, so
# launch_q4_gemm_tc5 splits K: SK = min(8, 132 / 20) = 6, lowered while K / 64 / SK < 4 -> 5 slices of 4 k-steps for
# K = 1280 (wqkv, wo); for K = 5120 (w2) 5 slices of 16 k-steps; w13 (N = 10240, 160 tiles) is not split.
SPLIT_K_FRAMES = 1000


def _report(what, err, bound):
    print(f"\n[encoder geometry] {what}: max |d| / max(1, max|ref|) = {err:.2e} (bound {bound:.0e})")
    assert err <= bound, (what, err)
    return err


class Geometry:
    def __init__(self, vx, window, data=None):
        self.window = window
        self.data = encoder_geometry_bytes(window) if data is None else data
        self.model = vx.Q4ModelLoader.from_bytes(self.data).load(0, max_batch=MAX_BATCH, max_mel_frames=MEL_FRAMES)
        self.o64 = OracleModel(self.data, dtype=torch.float64)
        assert self.model.info["enc_window"] == window and self.model.info["enc_head_dim"] == 64
        # three different 55 s utterances: 62.5 s of padded mel each, cropped per input
        self.mels = np.concatenate([geometry_mel(55.0, 40 + i)[:, :, :MEL_FRAMES] for i in range(MAX_BATCH)])


@pytest.fixture(scope="module", params=WINDOWS, ids=lambda w: f"window{w}")
def geom(request, vx):
    g = Geometry(vx, request.param)
    yield g
    g.model.close()


def _f64(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.float64)


def _offline(g, T, path, B, tag):
    """encode_audio of B streams of T mel frames with the debug capture on; every stage of every stream against the f64
    reference of that stage fed the GPU's own input.  Returns the largest error per stage."""
    m, o = g.model, g.o64
    mels = np.ascontiguousarray(g.mels[:B, :, :T])
    m.debug("capture_on")
    if path != "tc":
        m.debug(path)
    try:
        emb = m.encode_audio(mels)
    finally:
        m.debug("enc_attn_tc")
        m.debug("gemm_tc")
    d = o.cfg.enc_dim
    S = (((T - 1) // 2 + 1) - 1) // 2 + 1
    cap = {k: m.debug(k).reshape(B, S, d) for k in ["conv"] + [f"enc{i}" for i in range(o.cfg.enc_layers)] + ["enc_out"]}
    worst = {}
    for b in range(B):
        errs = {"conv": rel_err(cap["conv"][b], o.conv_stem(mels[b:b + 1]))}
        prev = cap["conv"][b]
        for i in range(o.cfg.enc_layers):
            errs[f"enc{i}"] = rel_err(cap[f"enc{i}"][b], o.encoder_layer(_f64(prev), i))
            prev = cap[f"enc{i}"][b]
        errs["enc_out"] = rel_err(cap["enc_out"][b], o.encoder_norm(_f64(prev)))
        errs["adapter"] = rel_err(emb[b], o.adapter(_f64(cap["enc_out"][b])))
        errs["embeds"] = rel_err(emb[b], o.encode_audio(mels[b:b + 1]))
        for k, v in errs.items():
            worst[k] = max(worst.get(k, 0.0), v)
    what = f"window {g.window:3d} {tag:6s} S={S:4d} {path:13s} B={B}"
    layer_bound = ENC_LAYER_REL_BOUND if path == "gemm_simt" else WGMMA_LAYER_REL_BOUND
    for k, v in worst.items():
        bound = {"embeds": EMBED_REL_BOUND, "adapter": ADAPTER_REL_BOUND, "conv": ENC_LAYER_REL_BOUND,
                 "enc_out": ENC_LAYER_REL_BOUND}.get(k, layer_bound)
        _report(f"{what} {k:8s}", v, bound)
    return worst


@pytest.mark.parametrize("inp", list(INPUTS))
def test_offline_encoder_layer_by_layer(geom, inp):
    for path, B in PATHS:
        _offline(geom, INPUTS[inp], path, B, inp)


def test_offline_encoder_split_k_single_stream(geom):
    _offline(geom, SPLIT_K_FRAMES, "tc", 1, "splitK")


# ---------------------------------------------------------------------------------------------------------------------
# Streaming pools
def _gpu_mel(vx, audio):
    """The GPU's own log-mel of the padded signal, [1, 128, T]."""
    return vx.MelSpectrogram.voxtral(0).compute_log(vx.pad_audio(audio)).T[None]


def _run_pool(vx, model, audios, opens, piece):
    """Feeds every session `piece` samples per tick from its opening tick on, then finishes it; returns each session's
    audio embeddings and the encoder row count of every tick."""
    pool = vx.StreamingPool(model, max_sessions=len(audios), max_seconds=60.0)
    n = len(audios)
    sids, fed, done = [None] * n, [0] * n, [False] * n
    rows = []
    try:
        for tick in range(100000):
            for i in range(n):
                if tick == opens[i]:
                    sids[i] = pool.open()
                if sids[i] is None or done[i]:
                    continue
                if fed[i] < audios[i].size:
                    pool.push(sids[i], audios[i][fed[i]:fed[i] + piece])
                    fed[i] += piece
                else:
                    pool.finish(sids[i])
                    done[i] = True
            rows.append(pool.tick()["encoder_rows"])
            if all(done):
                pool.tick()
                break
        return [pool.audio_embeds(s) for s in sids], np.array(rows)
    finally:
        pool.close()


STREAM_PATTERNS = {
    # name: (session lengths in s, opening ticks, samples per push)
    "one_80ms": ((52.0,), (0,), 1280),
    "two_staggered": ((47.0, 58.0), (0, 10), 1280),
    "five": ((45.0, 60.0, 50.0, 55.0, 48.0), (0, 2, 4, 6, 8), 1280),
    "one_12s_pieces": ((59.0,), (0,), 12 * 16000),
}


@pytest.mark.parametrize("pattern,env", [("one_80ms", None), ("two_staggered", None), ("five", None),
                                         ("one_12s_pieces", None), ("one_80ms", ("VOX_MATVEC", "simt")),
                                         ("five", ("VOX_GEMM", "simt"))],
                         ids=["one_80ms", "two_staggered", "five", "one_12s_pieces", "one_80ms_matvec_simt",
                              "five_gemm_simt"])
def test_streaming_pool_vs_f64(vx, geom, monkeypatch, pattern, env):
    """Each session's embeddings (every position: the window bites from encoder frame 751 on and the K/V ring wraps)
    against the f64 encode_audio of the GPU's own mel of the same padded signal."""
    if env is not None:
        monkeypatch.setenv(*env)          # read when the pool's session is created
    secs, opens, piece = STREAM_PATTERNS[pattern]
    audios = [omel.peak_normalize(omel.speechlike(s, 900 + 7 * i + int(s))) for i, s in enumerate(secs)]
    embs, rows = _run_pool(vx, geom.model, audios, opens, piece)
    # the first tick carries the left padding (152 frames) and the last the right padding: the steady state is the median
    steady = int(np.median(rows[rows > 0]))
    print(f"\n[encoder geometry] window {geom.window:3d} pool {pattern} {env}: encoder rows per tick {steady} "
          f"(median), {rows.max()} (largest)")
    # 80 ms = 2 encoder frames per session and tick
    if pattern == "one_80ms":
        assert steady == 2                        # the tensor-core matvec (R <= 8)
    elif pattern == "two_staggered":
        assert steady == 4                        # both sessions' rows, at different positions, in one matvec pass
    elif pattern == "five":
        assert steady == 10                       # the wgmma GEMM (R > 8; split-K at encoder N)
    else:
        assert rows.max() > 256                   # several passes of 256 rows in one tick
    for i, a in enumerate(audios):
        ref = geom.o64.encode_audio(_gpu_mel(vx, a)).numpy()
        assert embs[i].shape == ref.shape, (i, embs[i].shape, ref.shape)
        _report(f"window {geom.window:3d} pool {pattern} {env} session {i} embeds", rel_err(embs[i], ref), EMBED_REL_BOUND)


def test_encode_audio_with_cache_vs_f64(vx, geom):
    """Chunks of 400, 1100 (275 rows: two passes) and 3000 mel frames: by the last one the window reaches back across
    chunk boundaries.  The conv stem runs on each chunk alone, as upstream."""
    mel = geometry_mel(40.0, 31)
    pool = vx.StreamingPool(geom.model, max_sessions=1, max_seconds=60.0)
    try:
        sid = pool.open()
        cache = geom.o64.new_encoder_cache()
        a = 0
        for n in (400, 1100, 3000):
            chunk = np.ascontiguousarray(mel[:, :, a:a + n])
            got = pool.encode_audio_with_cache(sid, chunk[0])
            ref = geom.o64.encode_audio_with_cache(chunk, cache).numpy()
            assert got.shape == ref.shape, (n, got.shape, ref.shape)
            _report(f"window {geom.window:3d} encode_chunk frames {a}..{a + n}", rel_err(got, ref), EMBED_REL_BOUND)
            a += n
    finally:
        pool.close()


def test_unbounded_session_past_the_encoder_rope_table(vx):
    """Window 750: one session of 180 s fed in 5.12 s pieces (4 700 encoder frames).  The last 100 resident embeddings
    against the f64 suffix reference started enc_warmup_positions earlier (~60 s): beyond that reach nothing before the
    suffix can affect them."""
    data = encoder_geometry_bytes(750)
    model = vx.Q4ModelLoader.from_bytes(data).load(0, max_batch=1, max_mel_frames=100)
    o64 = OracleModel(data, dtype=torch.float64)
    piece = 32 * 2560
    audio = omel.peak_normalize(omel.speechlike(180.0, 17))
    pool = vx.StreamingPool(model, max_sessions=1, max_seconds=None)
    try:
        sid = pool.open()
        for a in range(0, audio.size, piece):
            pool.push(sid, audio[a:a + piece])
            pool.tick()
        info = pool.session_info(sid)
        assert info["encoder_frames"] > 4096 + 400 and info["first_audio_embed"] > 0
        n_cmp = 100
        first = info["audio_embeds"] - n_cmp
        emb = pool.audio_embeds(sid, first=first, n=n_cmp)
    finally:
        pool.close()
        model.close()
    p0 = first - enc_warmup_positions(o64.cfg)
    padded = np.concatenate([np.zeros(76 * 1280, np.float32), audio])[:info["samples"]]
    _, ref, _ = suffix_reference(o64, np.zeros(o64.cfg.dec_dim, np.float32), padded, p0 * 2560, [], n_pos=0)
    assert ref.shape[0] >= first - p0 + n_cmp and ref.dtype == np.float64
    _report(f"window 750 unbounded embeds {first}..{first + n_cmp - 1}", rel_err(emb, ref[first - p0:first - p0 + n_cmp]),
            EMBED_REL_BOUND)


@pytest.mark.slow
def test_full_size_encoder_layer_by_layer(vx, full_gguf):
    """The full-size model (seed 42, 32 layers), one 60 s utterance (T = 6000, S = 1500), default paths."""
    m = vx.Q4ModelLoader.from_file(full_gguf).load(0, max_batch=1, max_mel_frames=MEL_FRAMES)
    try:
        g = Geometry.__new__(Geometry)
        g.window, g.model = 750, m
        g.o64 = OracleModel(full_gguf, dtype=torch.float64)
        g.mels = geometry_mel(55.0, 40)[:, :, :MEL_FRAMES]
        _offline(g, MEL_FRAMES, "tc", 1, "full")
    finally:
        m.close()
