"""The Q4 kernels on the whole Q4_0 format against float64 (tests/test_q4_format_edges_ref.py holds the CPU side).

Operator level (vox_q4_matmul), each case in two kernel modes: "tc" (the tensor-core matvec K2a at M <= 8, the wgmma
GEMM K3 at M > 8 where N % 128 = K % 64 = 0 and every |d| < 32, else the SIMT GEMM) and "simt" (the SIMT matvec K2b and
the SIMT GEMM K3b).  Weight sets: scales of random sign, f16-subnormal scales, +-0 blocks, blocks heavy in nibbles 0
and 15, and |d| in {8, 31.98, 32, 64, 1000, 65504}.  Activation sets: Gaussian, a 1e4 outlier inside a block, blocks at
1e+-5, zero blocks and rows, -0.0, f32 subnormals inside rows of normal magnitude, rows at 1e-30 and at 1e30.  Per output
    |y - y64| <= 2^-20 * sum_k (|w_k| + 16 |d_b|) |x_k| + 2^-15 * max_k (|w_k| + 16 |d_b|) |x_k| + |bias| * 2^-23:
the error scale of the re-associated matvec form (tests/test_fragment_numerics.py) plus the floor of accumulation when
one term dominates the row (f64_and_bound); the numpy models of both tensor-core algorithms stay below a quarter of it
on every set.  The worst ratio is printed per kernel and separately for the outlier rows.  Shapes: the decoder's and
encoder's GEMMs, K = 4192 (131 blocks: K2a's last block pair is half empty, and at M >= 5 its 66 pairs leave a short last
split-K slice), K = 96, and N = 1, 17, 208.  Weights with |d| >= 32 on K3-capable shapes must take the SIMT GEMM: in
"tc" mode they give bitwise the "simt" result, in-domain weights do not (K3 still runs them).

Model level, on the sign-flipped twin (about a third of every Q4 tensor's blocks carry a negative scale; the dequantised
weights are the original's):
  * decoder geometry, window 40: the encoder is bitwise the original's (every encoder and adapter linear runs at
    M > 8 on a GEMM that builds the same f32 weights); teacher-forced decoding and prefill rows meet the decode geometry
    bound against the f64 reference; greedy ids equal the original's up to the first near-tie;
  * encoder geometry, window 750: the offline encoder layer by layer, and a streaming pool fed 80 ms per tick (2 rows:
    the tensor-core and the SIMT matvec), within the bounds of test_encoder_geometry_gpu.py.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
import test_encoder_geometry_gpu as encg
from test_decode_geometry_gpu import MEL_FRAMES, N_STREAMS, Geometry
from test_encoder_geometry_ref import EMBED_REL_BOUND, encoder_geometry_bytes
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes, rel_err
from test_golden_gpu import NEAR_TIE
from test_q4_format_edges_ref import (ACT_SETS, TWIN_SEED, WEIGHT_SETS, f64_and_bound, large_d, make_acts,
                                      make_weights, pairs, sign_flipped_twin)

pytestmark = pytest.mark.gpu

MODES = {"tc": 0, "simt": 3}
# (N, K, weight set): decoder wqkv, wo, w13, w2 and the encoder's FFN-in (K3-capable: two of them carry |d| >= 32
# scales, which the fix routes to the SIMT GEMM); K = 4192 (131 blocks); K = 96; N = 1, 17, 208
SHAPES = [(6144, 3072, "signed"), (3072, 4096, "d64"), (18432, 3072, "zero_blocks"), (3072, 9216, "d32"),
          (5120, 1280, "d65504"), (256, 4192, "f16_subnormal"), (128, 96, "nibbles_0_15"), (1, 4192, "d1000"),
          (17, 4192, "d8"), (208, 2304, "d31.98")]
assert sorted(w for _, _, w in SHAPES) == sorted(WEIGHT_SETS)
MS = (1, 2, 5, 8, 9, 38, 65, 320, 321)

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for key in sorted(_worst):
        print(f"\n[q4 format edges] {key}: worst |y - y64| / bound = {_worst[key]:.3f}")


def _run(vx, mode, raw, n, k, x, bias=None):
    assert vx.lib().vox_q4_set_matvec_mode(MODES[mode]) == 0
    try:
        return vx.q4_matmul(x[None], vx.Q4Tensor.from_q4_bytes(raw, (n, k)), bias)[0]
    finally:
        vx.lib().vox_q4_set_matvec_mode(0)


def _check(vx, group, mode, raw, n, k, x, bias, aset):
    out = _run(vx, mode, raw, n, k, x, bias).astype(np.float64)
    y64, bound = f64_and_bound(raw, n, k, x, bias)
    assert np.all(np.isfinite(out)), (group, mode, np.argwhere(~np.isfinite(out))[:4])
    err = np.abs(out - y64)
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))
    key = f"{group:5s} {mode:4s} {'M<=8' if x.shape[0] <= 8 else 'M>8 '}{' outlier rows' if aset == 'outlier_1e4' else ''}"
    _worst[key] = max(_worst.get(key, 0.0), float(ratio.max()))
    worst = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    assert ratio.max() <= 1.0, (group, mode, worst, float(ratio.max()), out[worst], y64[worst])


def _grid():
    """Every shape at every M, each shape with its weight set; the M rotate through the activation sets."""
    out = []
    for i, (n, k, wset) in enumerate(SHAPES):
        acts = [a for a in ACT_SETS if not (large_d(wset) and a == "rows_1e30")]
        for j, m in enumerate(MS):
            for mode in MODES:
                out.append((n, k, m, wset, acts[(i + j) % len(acts)], mode))
    return out


_weights = {}


def _shape_weights(wset, n, k):
    """One cached weight at a time (tests run shape by shape): the large shapes' f64 products are the cost."""
    key = (wset, n, k)
    if key not in _weights:
        _weights.clear()
        _weights[key] = make_weights(wset, n, k, n + k)
    return _weights[key]


@pytest.mark.parametrize("n,k,m,wset,aset,mode", _grid())
def test_shapes_and_rows(vx, n, k, m, wset, aset, mode):
    raw = _shape_weights(wset, n, k)
    x = make_acts(aset, m, k, 7 * m + k)
    bias = np.random.default_rng(m).standard_normal(n).astype(np.float32)
    _check(vx, "grid", mode, raw, n, k, x, bias, aset)


@pytest.mark.parametrize("wset,aset", pairs())
@pytest.mark.parametrize("mode", list(MODES))
def test_weight_and_activation_sets(vx, wset, aset, mode):
    """Every pair of sets: N = 256, K = 4160 (both tensor-core kernels' shapes) at M = 5 and 38, and N = 208,
    K = 4192 (odd block count) at M = 8 and 9."""
    for n, k, ms in ((256, 4160, (5, 38)), (208, 4192, (8, 9))):
        raw = make_weights(wset, n, k, 11 + k)
        for m in ms:
            x = make_acts(aset, m, k, 13 * m + k)
            bias = np.random.default_rng(k + m).standard_normal(n).astype(np.float32)
            _check(vx, "sets", mode, raw, n, k, x, bias, aset)


@pytest.mark.parametrize("wset,k3", [("d31.98", True), ("signed", True), ("d32", False), ("d65504", False)])
def test_k3_runs_exactly_the_in_domain_weights(vx, wset, k3):
    """At M = 38 on a K3-capable shape, "tc" mode runs K3 for weights with every |d| < 32 (its result differs from the
    SIMT GEMM's in the last bits) and the SIMT GEMM for the others (bitwise the "simt" mode result)."""
    n, k = 256, 4160
    raw = make_weights(wset, n, k, 5)
    x = make_acts("gauss", 38, k, 6)
    tc, simt = _run(vx, "tc", raw, n, k, x), _run(vx, "simt", raw, n, k, x)
    assert np.array_equal(tc.view(np.uint32), simt.view(np.uint32)) != k3, wset


# ---------------------------------------------------------------------------------- model level: the twin


@pytest.fixture(scope="module")
def twin(vx):
    """(Geometry over the twin, the original model).  The twin's f64 reference is the original's: the dequantised
    weights are equal (tests/test_q4_format_edges_ref.py)."""
    data = geometry_model_bytes(40)
    g = Geometry(vx, 40, data=sign_flipped_twin(data, TWIN_SEED))
    orig = vx.Q4ModelLoader.from_bytes(data).load(0, max_batch=N_STREAMS, max_mel_frames=MEL_FRAMES)
    yield g, orig, data
    orig.close()
    g.model.close()


def test_twin_encoder_is_bitwise_equal(twin):
    g, orig, _ = twin
    for b in (1, 3):
        a, t = orig.encode_audio(g.mels[:b]), g.model.encode_audio(g.mels[:b])
        assert np.array_equal(a.view(np.uint32), t.view(np.uint32)), b


@pytest.mark.parametrize("B", [1, 5, 8, 11])
def test_twin_persistent_kernel_vs_f64_reference(twin, B):
    g = twin[0]
    g.model.debug("mega_auto")
    logits, toks, launches = g.teacher_forced(B)
    g.check("twin mega", B, logits, toks)
    assert np.all(launches == (B + 7) // 8), (B, np.unique(launches))


@pytest.mark.parametrize("path,B", [("mega_off", 3), ("tc_off", 1)])
def test_twin_per_op_paths_vs_f64_reference(twin, path, B):
    g = twin[0]
    g.model.debug(path)
    try:
        logits, toks, launches = g.teacher_forced(B)
    finally:
        g.model.debug("tc_on" if path == "tc_off" else "mega_auto")
    g.check(f"twin {path}", B, logits, toks)
    assert np.all(launches > 2 * g.model.info["dec_layers"])


@pytest.mark.parametrize("B", [1, 8])
def test_twin_prefill_rows_match_f64(twin, B):
    """38 teacher-forced rows per stream through the token-embedding gather and the prefill's GEMMs (residual and
    SiLU * up epilogues), against the f64 reference."""
    g, _, data = twin
    o64 = OracleModel(data, dtype=torch.float64)
    model, vocab = g.model, g.vocab
    ids = np.random.default_rng(B).integers(0, vocab, (B, PREFIX_LEN)).astype(np.int32)
    model.reset_cache()
    got = model.generate_step_with_cache(ids)
    t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
    zeros = torch.zeros(PREFIX_LEN, o64.cfg.dec_dim, dtype=torch.float64)
    worst = 0.0
    for s in range(B):
        ref = o64.forward_streaming(None, ids[s].tolist(), t_embed, audio_embeds=zeros).numpy()
        err = rel_err(got[s], ref)
        worst = max(worst, float(err.max()))
        assert err.max() <= LOGIT_REL_BOUND, (s, int(err.argmax()), float(err.max()))
    print(f"\n[twin prefill] B={B}: max |dlogit| / max(1, max|ref|) = {worst:.2e}")


def test_twin_greedy_ids_equal_the_original(twin):
    """The original's greedy ids equal the twin's up to the first difference, which must be a near-tie of the f64
    reference (both ids its top two, margin < NEAR_TIE): after it the histories differ."""
    g, orig, _ = twin
    ids = orig.transcribe_streaming(g.mels)
    same = 0
    for i in range(N_STREAMS):
        diff = np.nonzero(ids[i] != g.free[i])[0]
        if diff.size == 0:
            same += 1
            continue
        j = int(diff[0])
        r = g.ref[i, j]
        top2 = np.argsort(r)[-2:]
        assert set(top2.tolist()) == {int(ids[i, j]), int(g.free[i, j])}, (i, j)
        assert r[top2[1]] - r[top2[0]] < NEAR_TIE, (i, j, r[top2[1]] - r[top2[0]])
    print(f"\n[twin ids] {same}/{N_STREAMS} streams: all greedy ids equal the original's")


# ------------------------------------------------------------------------------ the twin at encoder geometry


@pytest.fixture(scope="module")
def enc_twin(vx):
    """test_encoder_geometry_gpu.Geometry over the twin of the encoder-geometry model at window 750; its f64 reference
    is the original's."""
    g = encg.Geometry(vx, 750, data=sign_flipped_twin(encoder_geometry_bytes(750), TWIN_SEED))
    yield g
    g.model.close()


@pytest.mark.parametrize("path", ["tc", "gemm_simt"])
def test_twin_offline_encoder_layer_by_layer(enc_twin, path):
    """S = 995 at B = 1: every encoder and adapter linear at M > 8 (K3, or the SIMT GEMM), stage by stage against the
    f64 reference within test_encoder_geometry_gpu.py's bounds."""
    encg._offline(enc_twin, encg.INPUTS["S995"], path, 1, "twin")


@pytest.mark.parametrize("env", [None, ("VOX_MATVEC", "simt")], ids=["matvec_tc", "matvec_simt"])
def test_twin_streaming_pool_vs_f64(vx, enc_twin, monkeypatch, env):
    """One 20 s session fed 80 ms per tick: 2 encoder rows per tick through the tensor-core matvec (or the SIMT matvec),
    the window biting from encoder frame 751 on; every embedding against the f64 encode_audio of the GPU's own mel."""
    if env is not None:
        monkeypatch.setenv(*env)
    audio = omel.peak_normalize(omel.speechlike(20.0, 951))
    embs, rows = encg._run_pool(vx, enc_twin.model, [audio], (0,), 1280)
    assert int(np.median(rows[rows > 0])) == 2
    ref = enc_twin.o64.encode_audio(encg._gpu_mel(vx, audio)).numpy()
    assert embs[0].shape == ref.shape
    encg._report(f"window 750 twin pool 80ms {env} embeds", encg.rel_err(embs[0], ref), EMBED_REL_BOUND)
