"""Streaming pools with no length limit (max_seconds=None -> vox_stream_pool_create(..., 0)): every session keeps a
fixed amount of device state -- 30 s of padded audio in sliding PCM / mel / conv / encoder-output / embedding buffers,
the encoder K/V rings, the decoder KV as a ring of pages covering the decoder window, RoPE rows filled for the positions
in flight -- and still computes what the whole-utterance path computes.

The model is the decoder-geometry model (production decoder layer, tiny encoder) with a decoder window of 40
positions, so the KV ring (7 pages = 112 positions) wraps every ~18 s, and the audio is 70-110 s, so the 30 s audio
buffers slide several times.  Ids are compared with transcribe_pcm of the same audio, like the bounded pool's tests.
"""
import numpy as np
import pytest

from oracle import mel as omel

pytestmark = pytest.mark.gpu

DEC_WINDOW = 40
KV_PAGE, M_MAX = 16, 64
RING_PAGES = (DEC_WINDOW + M_MAX) // KV_PAGE + 1  # 16 L > dec_window + the rows a prefill appends before reading


@pytest.fixture(scope="module")
def geo_model(vx, tmp_path_factory):
    from voxtral_mini_realtime_rs_b200 import synth
    p = str(tmp_path_factory.mktemp("geo_unbounded") / "geo40.gguf")
    synth.write_synthetic_gguf(p, synth.decoder_geometry_config(DEC_WINDOW), seed=7)
    m = vx.Q4ModelLoader.from_file(p).load(0, max_batch=1, max_mel_frames=12000)
    yield m
    m.close()


def _run_pool(vx, model, audios, opens, piece_seed):
    """Feeds every session ragged pieces (0.1-1.2 s) per tick from its opening tick on; collects ids, the audio
    embeddings as they appear (through the range call) and the largest KV page count seen."""
    rng = np.random.default_rng(piece_seed)
    pool = vx.StreamingPool(model, max_sessions=len(audios), max_seconds=None)
    n = len(audios)
    sids, fed, finished = [None] * n, [0] * n, [False] * n
    ids = [[] for _ in range(n)]
    embs = [[] for _ in range(n)]
    max_pages, wrapped = 0, [False] * n
    for tick in range(100000):
        for i in range(n):
            if tick == opens[i]:
                sids[i] = pool.open()
            if sids[i] is None or finished[i]:
                continue
            if fed[i] < audios[i].size:
                k = int(rng.integers(1600, 19200))
                pool.push(sids[i], audios[i][fed[i]:fed[i] + k])
                fed[i] += k
            else:
                pool.finish(sids[i])
                finished[i] = True
        pool.tick()
        all_done = True
        for i in range(n):
            if sids[i] is None:
                all_done = False
                continue
            got, done = pool.poll(sids[i])
            ids[i] += got
            info = pool.session_info(sids[i])
            have = sum(e.shape[0] for e in embs[i])
            if info["audio_embeds"] > have:
                embs[i].append(pool.audio_embeds(sids[i], first=have, n=info["audio_embeds"] - have))
            wrapped[i] |= info["first_audio_embed"] > 0
            max_pages = max(max_pages, info["kv_pages"])
            all_done = all_done and done
        if all_done:
            break
    infos = [pool.session_info(s) for s in sids]
    pool.close()
    return ids, [np.concatenate(e) for e in embs], max_pages, wrapped, infos


@pytest.mark.parametrize("n_sessions,mega", [(1, True), (3, True), (8, True), (11, True), (3, False), (11, False)])
def test_unbounded_equals_offline(vx, geo_model, monkeypatch, n_sessions, mega):
    """Decoder steps run the persistent kernel's ring instantiation (groups of 8 rows at 11 sessions).  With it switched
    off (the pool's session reads VOX_MEGA when it is created) they run the fused single-token attention at 3 rows and
    the per-op RoPE-append + attention kernels at 11; every prefill runs the latter."""
    if not mega:
        monkeypatch.setenv("VOX_MEGA", "0")
    rng = np.random.default_rng(100 + n_sessions)
    secs = [float(rng.uniform(70.0, 110.0)) for _ in range(n_sessions)]
    audios = [omel.peak_normalize(omel.speechlike(s, 300 + 17 * i + n_sessions)) for i, s in enumerate(secs)]
    opens = [int(rng.integers(0, 60)) for _ in range(n_sessions)]
    opens[0] = 0
    ids, embs, max_pages, wrapped, infos = _run_pool(vx, geo_model, audios, opens, n_sessions)
    for i, a in enumerate(audios):
        want = geo_model.transcribe_pcm(a, peak_normalize=False)[0].tolist()
        assert ids[i] == want, (i, len(ids[i]), len(want), next((k for k, (x, y) in enumerate(zip(ids[i], want)) if x != y), None))
        ref = geo_model.encode_audio(omel.mel_tensor_from_audio(a))[0]
        assert embs[i].shape == ref.shape, (embs[i].shape, ref.shape)
        assert np.abs(embs[i] - ref).max() <= 1e-3
        assert wrapped[i]                                     # the embedding buffer really slid
        assert infos[i]["decoder_positions"] > 4 * RING_PAGES * KV_PAGE   # and the KV ring wrapped several times
        assert infos[i]["ids_emitted"] == len(ids[i])
    assert max_pages == RING_PAGES


def test_unbounded_limits(vx, geo_model):
    pool = vx.StreamingPool(geo_model, max_sessions=2, max_seconds=None)
    sid = pool.open()
    # more than the resident 30 s not yet consumed: refused until a tick has consumed what is there
    with pytest.raises(vx.VoxtralError, match="vox_stream_tick"):
        pool.push(sid, np.zeros(16000 * 31, np.float32))
    audio = omel.peak_normalize(omel.speechlike(60.0, 9))
    pool.push(sid, audio[:16000 * 20])
    with pytest.raises(vx.VoxtralError, match="vox_stream_tick"):
        pool.push(sid, audio[16000 * 20:16000 * 40])
    pool.tick()
    pool.push(sid, audio[16000 * 20:16000 * 40])              # the session continues after the tick
    pool.tick()
    pool.push(sid, audio[16000 * 40:])
    pool.tick()
    info = pool.session_info(sid)
    assert info["first_audio_embed"] > 0                      # 60 s of audio: the first embeddings were evicted
    with pytest.raises(vx.VoxtralError, match="vox_stream_audio_embeds_range"):
        pool.audio_embeds(sid)
    with pytest.raises(vx.VoxtralError, match="no longer resident"):
        pool.audio_embeds(sid, first=0, n=1)
    with pytest.raises(vx.VoxtralError, match="not produced"):
        pool.audio_embeds(sid, first=info["audio_embeds"], n=1)
    tail = pool.audio_embeds(sid, first=info["first_audio_embed"])
    assert tail.shape == (info["audio_embeds"] - info["first_audio_embed"], geo_model.info["dec_dim"])
    sid2 = pool.open()
    mel = omel.mel_tensor_from_audio(audio[:16000 * 2])
    with pytest.raises(vx.VoxtralError, match="max_seconds > 0"):
        pool.encode_audio_with_cache(sid2, mel[0])
    with pytest.raises(vx.VoxtralError):
        pool.session_info(5)
    pool.close()
    # bounded pools keep their limits
    with pytest.raises(vx.VoxtralError, match="out of range"):
        vx.StreamingPool(geo_model, max_sessions=1, max_seconds=0.5)


# ---------------------------------------------------------------------------------------------------------------------
# Past the model's RoPE tables: checked against the suffix reference (tests/suffix_reference.py), which follows the same
# arithmetic from part-way into the stream with empty caches and absolute positions.  Tiny model, decoder window 48.
from suffix_reference import dec_warmup_positions, enc_warmup_positions, suffix_reference  # noqa: E402

LEFT_PAD = 76 * 1280
PIECE = 32 * 2560          # 5.12 s per tick: 32 decoder positions, so stream offsets stay multiples of one position


@pytest.fixture(scope="module")
def window_pair(vx, tmp_path_factory):
    from oracle.model import OracleModel
    from voxtral_mini_realtime_rs_b200 import synth
    p = str(tmp_path_factory.mktemp("tiny_w48") / "tiny_w48.gguf")
    synth.write_synthetic_gguf(p, synth.tiny_window_config(48), seed=3)
    m = vx.Q4ModelLoader.from_file(p).load(0, max_batch=1, max_mel_frames=1500)
    yield m, OracleModel(p)
    m.close()


def _check_against_suffix(oracle, padded, ids, emb, first_emb, n_pos):
    """Resident embeddings [first_emb, ...) and the ids of the last ~200 positions against the suffix reference."""
    cfg = oracle.cfg
    t_embed = omel.time_embedding(6.0, cfg.dec_dim)
    p0 = max(0, min(first_emb, n_pos - 200) - enc_warmup_positions(cfg))
    _, ref, out = suffix_reference(oracle, t_embed, padded, p0 * 2560, ids, n_pos=n_pos)
    assert ref.shape[0] >= first_emb - p0 + emb.shape[0]
    err = np.abs(emb - ref[first_emb - p0:first_emb - p0 + emb.shape[0]]).max()
    assert err <= 1e-3, err
    checked = [p for p in out if p >= p0 + dec_warmup_positions(cfg)]
    assert len(checked) >= 50
    close = 0
    for p in checked:
        tok, margin = out[p]
        if margin < 2e-3:     # too close to call in f32: the comparison re-synchronises on the GPU's id (teacher forcing)
            close += 1
            continue
        assert tok == ids[p - 37], (p, tok, ids[p - 37], margin)
    assert close < len(checked) // 4


def test_past_the_encoder_rope_table(vx, window_pair):
    """One session of 210 s: 5 000+ encoder frames, past the 4096-row encoder RoPE table."""
    model, oracle = window_pair
    audio = omel.peak_normalize(omel.speechlike(210.0, 11))
    pool = vx.StreamingPool(model, max_sessions=1, max_seconds=None)
    sid = pool.open()
    ids = []
    for a in range(0, audio.size, PIECE):
        pool.push(sid, audio[a:a + PIECE])
        pool.tick()
        ids += pool.poll(sid)[0]
    info = pool.session_info(sid)
    assert info["encoder_frames"] > 4096 + 500
    emb = pool.audio_embeds(sid, first=info["first_audio_embed"])
    pool.close()
    padded = np.concatenate([np.zeros(LEFT_PAD, np.float32), audio])[:info["samples"]]
    _check_against_suffix(oracle, padded, ids, emb, info["first_audio_embed"], info["decoder_positions"])


@pytest.mark.slow
def test_long_haul_46_minutes(vx, window_pair):
    """Three sessions over 46 min of deterministic synthetic audio generated piecewise: past encoder frame 4096, past
    decoder position 16384 (the model's decoder RoPE table) and through many KV-ring and RoPE-ring wraps.  Session B
    gets A's audio 4096 positions later, so the two collide in the 4096-row decoder RoPE ring at every step (one of them
    waits a step): B's ids must be A's.  A is checked against the suffix reference just past encoder frame 4096, just
    past decoder position 16384, and at the end; C (other audio, opened at another time) at the end."""
    model, oracle = window_pair
    ticks = int(46 * 60 * 16000) // PIECE + 1
    def piece(seed, k):
        return omel.peak_normalize(omel.speechlike(PIECE / 16000, 1000 * seed + k))
    pool = vx.StreamingPool(model, max_sessions=3, max_seconds=None)
    opens = {"A": 0, "B": 4096 * 2560 // PIECE, "C": 37}
    seeds = {"A": 1, "B": 1, "C": 2}
    sid, ids, fed, sig = {}, {k: [] for k in opens}, {k: 0 for k in opens}, {"A": [], "C": []}
    checkpoints, pages = [], set()
    marks = [("enc", lambda i: i["encoder_frames"] > 4096 + 100), ("dec", lambda i: i["decoder_positions"] > 16384 + 100)]
    for t in range(ticks):
        for k, t0 in opens.items():
            if t == t0:
                sid[k] = pool.open()
            if k in sid:
                x = piece(seeds[k], fed[k])
                pool.push(sid[k], x)
                fed[k] += 1
                if k in sig:
                    sig[k].append(x)
        pool.tick()
        for k in sid:
            ids[k] += pool.poll(sid[k])[0]
        infoA = pool.session_info(sid["A"])
        if marks and marks[0][1](infoA):
            checkpoints.append(("A", infoA, list(ids["A"]), pool.audio_embeds(sid["A"], first=infoA["first_audio_embed"])))
            marks.pop(0)
        if infoA["decoder_positions"] > 200:
            pages.add(infoA["kv_pages"])
    for k in ("A", "C"):
        info = pool.session_info(sid[k])
        checkpoints.append((k, info, list(ids[k]), pool.audio_embeds(sid[k], first=info["first_audio_embed"])))
    infoB = pool.session_info(sid["B"])
    pool.close()
    assert not marks and checkpoints[-2][1]["decoder_positions"] > 16384 + 500
    assert len(ids["B"]) > 12000 and ids["B"] == ids["A"][:len(ids["B"])]
    assert infoB["decoder_positions"] + 4096 == checkpoints[-2][1]["decoder_positions"]
    assert pages == {(48 + 64) // 16 + 1}                        # constant once the ring is full
    for k, info, kid, emb in checkpoints:
        padded = np.concatenate([np.zeros(LEFT_PAD, np.float32)] + sig[k])[:info["samples"]]
        _check_against_suffix(oracle, padded, kid, emb, info["first_audio_embed"], info["decoder_positions"])
