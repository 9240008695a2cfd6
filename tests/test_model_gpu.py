"""GPU parity of the model path (mel -> encode_audio -> transcribe_streaming, generate_step) on a
tiny synthetic GGUF, against the CPU oracle, through the C ABI.

Tolerances (f32 path; the north_star bounds encoder hidden states at 1e-3 abs):
  mel log-spectrogram 2e-4 abs; audio embeds 1e-3 abs (asserted much tighter here, tiny model);
  logits 1e-3 abs; token ids bit-exact (the oracle's top-2 margin is asserted to dominate the error).
"""
import numpy as np
import pytest

from oracle import mel as omel

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny_model(vx, tiny_gguf):
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=4, max_mel_frames=3000)
    yield m
    m.close()


@pytest.fixture(scope="module")
def tiny_model8(vx, tiny_gguf):
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=8, max_mel_frames=1500)
    yield m
    m.close()


def _mel(seconds, seed=1234):
    a = omel.peak_normalize(omel.speechlike(seconds, seed))
    return a, omel.mel_tensor_from_audio(a)


def test_mel_gpu_vs_oracle(vx):
    ms = vx.MelSpectrogram.voxtral(0)
    o = omel.MelSpectrogram()
    assert np.abs(ms.window() - o.window).max() < 1e-7
    fb, ofb = ms.mel_basis(), o.mel_basis
    assert np.abs(fb - ofb).max() < 2e-5 * ofb.max()
    for sig in (omel.sine_16k(1.0), omel.noise_chirp(3.0), omel.pad_audio(omel.speechlike(2.0)),
                np.zeros(16000, np.float32), omel.speechlike(0.3)[:3333]):
        g = ms.compute_log(sig)
        e = o.compute_log(sig)
        assert g.shape == e.shape == (omel.num_frames(sig.size), 128)
        assert np.abs(g - e).max() < 2e-4, np.abs(g - e).max()
    # reference pins (mel.rs:409-421, 438-456): silence -> floor, 440 Hz sine in [-2, 3]
    assert np.all(ms.compute_log(np.zeros(16000, np.float32)) == np.float32((-6.5 + 4.0) / 4.0))
    s = ms.compute_log(omel.sine_16k(1.0))
    assert s.min() >= -2.0 and s.max() <= 3.0


def test_encode_audio_parity(tiny_model, tiny_oracle):
    _, mel = _mel(4.0)
    got = tiny_model.encode_audio(mel)
    cap = {}
    exp = tiny_oracle.encode_audio(mel, capture=cap).numpy()
    assert got.shape == (1,) + exp.shape
    err = np.abs(got[0] - exp).max()
    assert err < 1e-3
    assert err < 5e-5 * max(1.0, np.abs(exp).max()), err
    enc = tiny_model.debug("enc_out").reshape(cap["enc_out"].shape)
    assert np.abs(enc - cap["enc_out"].numpy()).max() < 1e-3


def test_encoder_layers_capture(tiny_model, tiny_oracle):
    _, mel = _mel(2.0, seed=9)
    tiny_model.debug("capture_on")
    tiny_model.encode_audio(mel)
    cap = {}
    tiny_oracle.encode_audio(mel, capture=cap)
    conv = tiny_model.debug("conv").reshape(cap["conv"].shape)
    assert np.abs(conv - cap["conv"].numpy()).max() < 1e-4
    for i in range(tiny_oracle.cfg.enc_layers):
        g = tiny_model.debug(f"enc{i}").reshape(cap[f"enc{i}"].shape)
        assert np.abs(g - cap[f"enc{i}"].numpy()).max() < 2e-4, i
    tiny_model.debug("capture_off")


def test_encoder_attention_tensor_core_vs_simt(tiny_model, tiny_oracle):
    """enc_attn_tc.cu (mma.sync, two-piece f16 operands; default) against the f32 SIMT kernel and the oracle:
    same encoder output to f32 rounding noise, with the sliding window biting (window 20 < S)."""
    _, mel = _mel(5.0, seed=77)
    exp = tiny_oracle.encode_audio(mel).numpy()[None]
    tiny_model.debug("enc_attn_tc")
    got_tc = tiny_model.encode_audio(mel).copy()
    tiny_model.debug("enc_attn_simt")
    try:
        got_simt = tiny_model.encode_audio(mel).copy()
    finally:
        tiny_model.debug("enc_attn_tc")
    assert np.abs(got_tc - exp).max() < 1e-3            # the north-star bound
    assert np.abs(got_tc - got_simt).max() < 2e-5 * max(1.0, np.abs(got_simt).max())
    assert np.abs(got_tc - exp).max() < 3 * np.abs(got_simt - exp).max() + 1e-6


def test_sliding_window_bites(tiny_model, tiny_oracle):
    """tiny enc_window=20 < S: the window mask changes the result, and we match the oracle."""
    _, mel = _mel(3.0, seed=4)
    got = tiny_model.encode_audio(mel)[0]
    exp = tiny_oracle.encode_audio(mel).numpy()
    assert np.abs(got - exp).max() < 1e-3
    saved = tiny_oracle.cfg.enc_window
    tiny_oracle.cfg.enc_window = 100000
    try:
        nowin = tiny_oracle.encode_audio(mel).numpy()
    finally:
        tiny_oracle.cfg.enc_window = saved
    assert np.abs(nowin - exp).max() > 10 * np.abs(got - exp).max()


def test_transcribe_streaming_token_parity(vx, tiny_model, tiny_oracle):
    _, mel = _mel(4.0)
    t_embed = omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim)
    info = {}
    exp = tiny_oracle.transcribe_streaming(mel, t_embed, info=info)
    tm = vx.Timings()
    got = tiny_model.transcribe_streaming(mel, timings=tm)
    assert len(exp) == mel.shape[2] // 16 - 38 == tm.decode_tokens
    assert got == exp, (got, exp, min(info["margins"]))
    assert len(set(exp)) > 2          # not a degenerate constant sequence
    assert tm.decode_ms > 0 and tm.encode_ms > 0
    # eager (no CUDA graph) path gives the same ids
    tiny_model.debug("graph_off")
    assert tiny_model.transcribe_streaming(mel) == exp
    tiny_model.debug("graph_on")
    # the SIMT matvec (tensor-core-assisted matvec disabled) gives the same ids
    tiny_model.debug("tc_off")
    assert tiny_model.transcribe_streaming(mel) == exp
    tiny_model.debug("tc_on")


@pytest.mark.parametrize("batch", [1, 2, 3, 5, 8])
def test_persistent_decode_kernel_matches_per_op_launches(vx, tiny_model8, tiny_oracle, batch):
    """decode_mega.cu (one persistent kernel per decode step; default) against the per-op launch path
    and the oracle: same ids for every batch size / token-capacity instantiation (1, 2, 4, 8), and the
    last step's logits agree to f32 summation-order noise."""
    sigs = np.stack([omel.speechlike(3.5, seed=40 + i) for i in range(batch)])
    t_embed = omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim)
    exp = [tiny_oracle.transcribe_streaming(omel.mel_tensor_from_audio(omel.peak_normalize(s)), t_embed) for s in sigs]
    tiny_model8.debug("mega_on")
    n0 = tiny_model8.launch_count()
    got = tiny_model8.transcribe_pcm(sigs)
    n_mega = tiny_model8.launch_count() - n0
    lg_mega = tiny_model8.debug("logits").copy()
    tiny_model8.debug("mega_off")
    try:
        n0 = tiny_model8.launch_count()
        ref = tiny_model8.transcribe_pcm(sigs)
        n_ops = tiny_model8.launch_count() - n0
        lg_ops = tiny_model8.debug("logits").copy()
    finally:
        tiny_model8.debug("mega_auto")
    for i in range(batch):
        assert got[i].tolist() == exp[i], i
    assert np.array_equal(got, ref)
    assert n_mega < n_ops  # the persistent kernel really replaced the per-op launches
    v = tiny_oracle.cfg.vocab
    assert np.abs(lg_mega[:batch * v] - lg_ops[:batch * v]).max() < 1e-4 * max(1.0, np.abs(lg_ops[:batch * v]).max())


def test_transcribe_short_audio_returns_empty(tiny_model):
    mel = np.zeros((1, 128, 37 * 16), np.float32)  # seq_len 37 < 38 (model.rs:887-889)
    assert tiny_model.transcribe_streaming(mel) == []


def test_transcribe_pcm_pipeline_and_batch(vx, tiny_model, tiny_oracle):
    """PCM entry point (device peak-normalise + pad + GPU mel) == oracle pipeline; batched streams
    give exactly the per-stream results."""
    sigs = [omel.speechlike(3.0, seed=s) for s in (11, 12, 13)]
    t_embed = omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim)
    exp = []
    for s in sigs:
        mel = omel.mel_tensor_from_audio(omel.peak_normalize(s))
        exp.append(tiny_oracle.transcribe_streaming(mel, t_embed))
    got_b = tiny_model.transcribe_pcm(np.stack(sigs))
    assert got_b.shape == (3, len(exp[0]))
    for i in range(3):
        assert got_b[i].tolist() == exp[i], i
        assert tiny_model.transcribe_pcm(sigs[i])[0].tolist() == exp[i]


def test_batches_above_eight_streams(vx, tiny_gguf, tiny_oracle):
    """More than 8 streams per GPU: each decode step runs the persistent decode kernel (token capacity 8) over
    consecutive groups of up to 8 rows, and the prefill's linears (B x 38 rows) are the wgmma GEMM -- same ids as the
    oracle, graph replay == eager."""
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=20, max_mel_frames=1500)
    try:
        sigs = [omel.speechlike(3.0, seed=300 + i) for i in range(20)]
        t_embed = omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim)
        exp = [tiny_oracle.transcribe_streaming(omel.mel_tensor_from_audio(omel.peak_normalize(s)), t_embed) for s in sigs]
        for b in (9, 12, 20):
            got = m.transcribe_pcm(np.stack(sigs[:b]))
            assert got.shape == (b, len(exp[0]))
            for i in range(b):
                assert got[i].tolist() == exp[i], (b, i)
        m.debug("graph_off")
        got = m.transcribe_pcm(np.stack(sigs[:12]))
        m.debug("graph_on")
        for i in range(12):
            assert got[i].tolist() == exp[i], i
    finally:
        m.close()


def test_generate_step_with_cache_parity(tiny_model, tiny_oracle):
    """Incremental API (model.rs:857-867): prefill M=5 then single steps; logits vs oracle."""
    cfg = tiny_oracle.cfg
    t_embed = omel.time_embedding(6.0, cfg.dec_dim)
    ada = tiny_oracle.ada_scales(t_embed)
    cache = tiny_oracle.new_cache()
    tiny_model.reset_cache()
    ids = [1, 32, 77, 400, 9]
    h = tiny_oracle.decoder_forward_with_cache(tiny_oracle.embed_tokens(ids), ada, cache)
    exp = tiny_oracle.lm_head(h).numpy()
    got = tiny_model.generate_step_with_cache(np.array([ids]))
    assert got.shape == (1, 5, cfg.vocab)
    assert np.abs(got[0] - exp).max() < 1e-3
    assert tiny_model.cache_len() == 5
    for tok in (123, 7):
        h = tiny_oracle.decoder_forward_with_cache(tiny_oracle.embed_tokens([tok]), ada, cache)
        exp = tiny_oracle.lm_head(h).numpy()
        got = tiny_model.generate_step_with_cache(np.array([[tok]]))
        assert np.abs(got[0] - exp).max() < 1e-3
        assert int(got[0, 0].argmax()) == int(exp[0].argmax())
    assert tiny_model.cache_len() == 7
    # different fed-back token => different logits (feedback path is live)
    a = tiny_model.generate_step_with_cache(np.array([[5]]))
    tiny_model.reset_cache()
    assert tiny_model.cache_len() == 0
    b = tiny_model.generate_step_with_cache(np.array([[6]]))
    assert np.abs(a - b).max() > 1e-3


def test_device_side_incremental_api(tiny_model, tiny_oracle):
    """vox_prefill + vox_decode_step (SURVEY 8(b); model.rs:857-867 with the argmax kept on the device): driving the
    decoder step by step reproduces transcribe_streaming, with device feedback (tok=None), with host-fed tokens,
    batched, and without audio (== argmax of generate_step_with_cache's logits)."""
    sigs = [omel.peak_normalize(omel.speechlike(4.0, 50 + i)) for i in range(3)]
    mels = np.concatenate([omel.mel_tensor_from_audio(a) for a in sigs])
    want = tiny_model.transcribe_streaming(mels)                  # [3, n]
    n = want.shape[1]
    t_embed = omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim)
    assert want[0].tolist() == tiny_oracle.transcribe_streaming(mels[:1], t_embed)
    prefix = np.array([[1] + [32] * 37] * 3, np.int32)
    # (a) device feedback, batched
    tiny_model.encode_audio(mels)
    tiny_model.reset_cache()
    out = [tiny_model.prefill(prefix)]
    for _ in range(n - 2):
        tiny_model.decode_step(batch=3, read=False)               # fully asynchronous steps
        out.append(None)
    last = tiny_model.decode_step(batch=3)
    assert tiny_model.cache_len() == 38 + n - 1
    assert np.array_equal(out[0], want[:, 0]) and np.array_equal(last, want[:, n - 1])
    # (b) host-fed tokens (teacher forcing with the known ids), single stream
    tiny_model.encode_audio(mels[1:2])
    tiny_model.reset_cache()
    got = [int(tiny_model.prefill(prefix[:1])[0])]
    for j in range(1, n):
        got.append(int(tiny_model.decode_step(tok=[int(want[1, j - 1])])[0]))
    assert got == want[1].tolist()
    # (c) token-only (no audio): equals the argmax of generate_step_with_cache
    ids = np.array([[1, 32, 77, 400, 9]], np.int32)
    tiny_model.reset_cache()
    lg = tiny_model.generate_step_with_cache(ids)
    tiny_model.reset_cache()
    nxt = tiny_model.prefill(ids, add_audio=False)
    assert int(nxt[0]) == int(lg[0, -1].argmax())
    lg2 = tiny_model.generate_step_with_cache(np.array([[int(nxt[0])]]))
    tiny_model.reset_cache()
    tiny_model.prefill(ids, add_audio=False)
    assert int(tiny_model.decode_step(batch=1, add_audio=False)[0]) == int(lg2[0, 0].argmax())
    # argument checking: audio positions exhausted / wrong batch
    tiny_model.encode_audio(mels[:1])
    tiny_model.reset_cache()
    with pytest.raises(Exception, match="add_audio"):
        tiny_model.prefill(prefix[:2])


def test_forward_streaming_parity(tiny_model, tiny_oracle):
    """forward_streaming (model.rs:801-814): teacher-forced logits for every position vs the oracle."""
    _, mel = _mel(4.0, seed=9)
    emb = tiny_oracle.encode_audio(mel)
    s4 = emb.shape[0]
    rng = np.random.default_rng(0)
    ids = rng.integers(0, tiny_oracle.cfg.vocab, size=s4).astype(np.int32)
    ids[0] = 1
    exp = tiny_oracle.forward_streaming(mel, ids.tolist(), omel.time_embedding(6.0, tiny_oracle.cfg.dec_dim), audio_embeds=emb).numpy()
    got = tiny_model.forward_streaming(mel, ids[None])[0]
    assert got.shape == exp.shape
    assert np.abs(got - exp).max() < 1e-3
    assert np.array_equal(got.argmax(1), exp.argmax(1))
    assert tiny_model.cache_len() == s4


def test_set_delay_changes_ada(tiny_model, tiny_oracle):
    cfg = tiny_oracle.cfg
    for delay in (6.0, 2.0):
        tiny_model.set_delay(delay)
        ada = np.stack([a.numpy() for a in tiny_oracle.ada_scales(omel.time_embedding(delay, cfg.dec_dim))])
        got = tiny_model.debug("ada").reshape(ada.shape)
        assert np.abs(got - ada).max() < 1e-5
    tiny_model.set_delay(6.0)


def test_loader_errors(vx, tiny_gguf, tmp_path):
    with pytest.raises(vx.VoxtralError, match="Failed to open"):
        vx.Q4ModelLoader.from_file(str(tmp_path / "missing.gguf"))
    # a GGUF lacking a required tensor -> "Tensor '...' not found"
    from oracle import gguf_synth, q4 as oq4
    raw = oq4.quantize_f32_to_q4_0(np.ones(32 * 32, np.float32))
    data = gguf_synth.build_gguf_bytes([("weight_a", 2, (32, 32), raw)])
    with pytest.raises(vx.VoxtralError, match="not found"):
        vx.Q4ModelLoader.from_bytes(data).load(0)
