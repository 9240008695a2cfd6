"""The wgmma GEMM (K3) at prefill and encoder shapes: single token tiles up to 320 rows and the stream-K schedule.

Operator level (vox_q4_matmul, the launch_q4_linear path the session takes: M > 8 runs split_tiles + K3) against a
float64 product of the dequantised weights, with the bound test_q4_gpu.py's K3 test uses.  Shapes: the decoder's four
GEMMs (wqkv 6144 x 3072, wo 3072 x 4096, w13 18432 x 3072, w2 3072 x 9216) and the encoder's FFN-in (5120 x 1280),
at M across the token-tile widths (64, 128, 192, 256 and 320 rows in one tile; 321 and 586 take 128-row tiles).  On a
132-SM launch every one of them splits tiles: wqkv at M <= 320 has 48 tiles x 48 k-steps over 132 CTAs (17-18 k-steps
each), so every tile is shared by three or more CTAs and most CTAs cross a tile boundary; the encoder shape at M = 586
gives CTAs of 30 k-steps over 20-step tiles, whole tiles and split ones in one launch.  The same call twice is bitwise
equal (split tiles are summed in slice order).

Model level: on synth.decoder_geometry_config, a teacher-forced 38-row pass per stream (vox_generate_step_with_cache,
the prefill's shapes: M = 38 * B through wqkv, wo and w2 with the in-place residual, w13 with SiLU * up) agrees with
OracleModel(dtype=float64) within LOGIT_REL_BOUND at every one of the 38 rows, for B = 1..8 at decoder window 8192, and
at B = 1, 3 and 8 at windows 40 and 8, where the mask of dec_attention_kernel bites inside the 38 prefill rows.
"""
import numpy as np
import pytest
import torch

from oracle.model import PREFIX_LEN, OracleModel
from oracle import mel as omel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes, rel_err

pytestmark = pytest.mark.gpu

SHAPES = {"wqkv": (6144, 3072), "wo": (3072, 4096), "w13": (18432, 3072), "w2": (3072, 9216), "enc_w1": (5120, 1280)}
DEC_M = (9, 38, 64, 65, 200, 250, 304, 320, 321)
ENC_M = (65, 304, 321, 586)


@pytest.fixture(scope="module")
def weights(vx):
    from voxtral_mini_realtime_rs_b200 import synth
    out = {}
    for name, (n, k) in SHAPES.items():
        rng = np.random.default_rng(n + k)
        t = vx.Q4Tensor.from_q4_bytes(synth.random_q4_blocks(rng, n * k, 1.0 / np.sqrt(k)), (n, k))
        out[name] = (t, t.dequantize().astype(np.float64))
    yield out


def _case(weights, name, m):
    t, w = weights[name]
    n, k = t.shape()
    rng = np.random.default_rng(1000 * m + n)
    x = (rng.standard_normal((1, m, k)) * rng.uniform(0.1, 3.0, (1, m, 1))).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    return t, x, bias, x[0].astype(np.float64) @ w.T + bias


@pytest.mark.parametrize("name,m", [(s, m) for s in ("wqkv", "wo", "w13", "w2") for m in DEC_M] +
                         [("enc_w1", m) for m in ENC_M])
def test_k3_matches_f64(vx, weights, name, m):
    t, x, bias, exp = _case(weights, name, m)
    out = vx.q4_matmul(x, t, bias)[0]
    err = np.abs(out - exp).max()
    assert err < 3e-5 * np.abs(exp).max() + 1e-5, err
    again = vx.q4_matmul(x, t, bias)[0]
    assert np.array_equal(out.view(np.uint32), again.view(np.uint32))


@pytest.fixture(scope="module")
def geometry(vx):
    """one model at a time, by decoder window"""
    held = {}

    def get(window):
        if window not in held:
            for m, _ in held.values():
                m.close()
            held.clear()
            data = geometry_model_bytes(window)
            held[window] = (vx.Q4ModelLoader.from_bytes(data).load(0, max_batch=8, max_mel_frames=1200),
                            OracleModel(data, dtype=torch.float64))
        return held[window]
    yield get
    for m, _ in held.values():
        m.close()


@pytest.mark.parametrize("window,B", [(8192, b) for b in range(1, 9)] + [(w, b) for w in (40, 8) for b in (1, 3, 8)])
def test_prefill_rows_match_f64(geometry, window, B):
    model, o64 = geometry(window)
    vocab = model.info["vocab"]
    rng = np.random.default_rng(B)
    ids = rng.integers(0, vocab, (B, PREFIX_LEN)).astype(np.int32)
    model.reset_cache()
    got = model.generate_step_with_cache(ids)                     # [B, 38, V]: no audio added
    t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
    zeros = torch.zeros(PREFIX_LEN, o64.cfg.dec_dim, dtype=torch.float64)
    for s in range(B):
        ref = o64.forward_streaming(None, ids[s].tolist(), t_embed, audio_embeds=zeros).numpy()
        err = rel_err(got[s], ref)
        assert err.max() <= LOGIT_REL_BOUND, (s, int(err.argmax()), float(err.max()))
