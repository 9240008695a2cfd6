"""Host side of unbounded streaming pools (max_seconds = 0), and the suffix reference (tests/suffix_reference.py) the
GPU tests use to follow sessions past the model's RoPE tables."""
import ctypes as C

import numpy as np
import pytest

from oracle import mel as omel
from oracle.model import OracleModel, rope_tables
from oracle.streaming import StreamingOracle
from suffix_reference import dec_warmup_positions, enc_warmup_positions, suffix_reference
from voxtral_mini_realtime_rs_b200 import api

VOX_EINVAL, VOX_ECUDA = 1, 4


def test_new_entry_points_without_a_device_or_handle(vx, have_gpu):
    lib = vx.lib()
    out = (C.c_float * 8)()
    info = api._StreamSessionInfo()
    want = VOX_EINVAL if have_gpu else VOX_ECUDA       # no device: VOX_ECUDA first, as every compute entry point
    assert lib.vox_stream_audio_embeds_range(None, 0, 0, 1, out, 8) == want
    assert lib.vox_stream_session_info(None, 0, C.byref(info)) == want
    assert (b"null argument" if have_gpu else b"no CUDA device") in lib.vox_last_error()


def test_session_info_layout():
    # int64 x 7 + int32, padded to 8 bytes: the C struct, the ctypes mirror and rust/voxtral_sys.rs agree
    assert C.sizeof(api._StreamSessionInfo) == 64
    names = [f[0] for f in api._StreamSessionInfo._fields_]
    assert names == ["samples", "mel_frames", "encoder_frames", "audio_embeds", "first_audio_embed", "decoder_positions",
                     "ids_emitted", "kv_pages"]


@pytest.mark.parametrize("head_dim,rows", [(32, 4096), (64, 4096), (32, 16384), (128, 16384)])
def test_extended_rope_rows_equal_the_tables(head_dim, rows):
    """Rows past the model's tables come from the same f32 formula; inside them they are bitwise the tables."""
    c0, s0 = rope_tables(head_dim, rows, 1e6)
    c1, s1 = rope_tables(head_dim, rows + 70000, 1e6)
    assert np.array_equal(c0.numpy(), c1[:rows].numpy()) and np.array_equal(s0.numpy(), s1[:rows].numpy())


@pytest.fixture(scope="module")
def window_oracle(tmp_path_factory):
    from voxtral_mini_realtime_rs_b200 import synth
    p = str(tmp_path_factory.mktemp("tinyw") / "tiny_w48.gguf")
    synth.write_synthetic_gguf(p, synth.tiny_window_config(48), seed=3)
    return OracleModel(p)


def test_suffix_reference_equals_the_full_stream(window_oracle):
    """A 40 s stream of the tiny model with decoder window 48: the suffix started 15.4 s into the padded signal gives
    the full streaming oracle's audio embeddings and (teacher-forced along the full oracle's ids) its ids once past
    the warm-up."""
    m = window_oracle
    t_embed = omel.time_embedding(6.0, m.cfg.dec_dim)
    full = StreamingOracle(m, t_embed)
    audio = omel.peak_normalize(omel.speechlike(40.0, 77))
    for a in range(0, audio.size, 16000):
        full.feed(audio[a:a + 16000])
    ref_emb = np.stack([e.numpy() for e in full.audio_embeds])
    s0 = 96 * 2560
    p0, emb, out = suffix_reference(m, t_embed, full.samples, s0, full.ids)
    ew, dw = enc_warmup_positions(m.cfg), dec_warmup_positions(m.cfg)
    n = min(emb.shape[0], ref_emb.shape[0] - p0)
    assert n > ew + 50
    assert np.abs(emb[ew:n] - ref_emb[p0 + ew:p0 + n]).max() <= 1e-4
    checked = [p for p in out if p >= p0 + dw]
    assert len(checked) > 40
    for p in checked:
        tok, margin = out[p]
        assert margin < 2e-3 or tok == full.ids[p - 37], (p, tok, full.ids[p - 37], margin)
