"""GPU parity of the Q4 operator seam (vox_q4_tensor_* / vox_q4_matmul) against the oracle.

Mirrors the reference's kernel tests 1:1 (closed-form inputs, same tolerances):
  src/gguf/tests.rs  test_q4_dequantize_gpu 332-364 (1e-5), test_q4_matmul_small 371-411 (1e-3),
  test_q4_matmul_shapes 414-478 (1e-2), test_q4_linear_forward_with_bias 507-562 (1e-3),
  test_q4_matmul_batch 643-694 (1e-3);  tests/gguf_integration.rs 74-130 (0.5 vs unquantised).
Plus what the reference lacks: every M in 1..9 (matvec/GEMM dispatch boundary), nibble value 0
(-8*d, never produced by the reference's test quantiser), ragged N, K-chunked staging.
"""
import numpy as np
import pytest

from oracle import q4 as oq4
from conftest import closed_form_weights

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True, params=["tc", "simt"])
def matvec_mode(request, vx):
    """Every test runs with both kernel families: tensor-core paths (mma.sync matvec for M<=8, wgmma
    GEMM for M>8; default) and the SIMT matvec / SIMT tiled GEMM."""
    assert vx.lib().vox_q4_set_matvec_mode(3 if request.param == "simt" else 0) == 0
    yield request.param
    vx.lib().vox_q4_set_matvec_mode(0)


def _ref(x2d, raw, n, k, bias=None):
    return oq4.q4_matmul_c(x2d, raw, n, k, bias)


def test_q4_dequantize_gpu(vx):
    rows = cols = 16
    orig = (np.sin(np.arange(rows * cols, dtype=np.float32) * np.float32(0.05) - np.float32(6.4)) * np.float32(0.3))
    raw = oq4.quantize_f32_to_q4_0(orig.astype(np.float32))
    # 16x16: K=16 is not block aligned per row -> the product requires K % 32 == 0; use [8,32] view
    t = vx.Q4Tensor.from_q4_bytes(raw, (8, 32))
    assert np.abs(t.dequantize().reshape(-1) - oq4.dequantize_q4_0(raw)).max() < 1e-5


def test_q4_matmul_small(vx):
    k = n = 32
    wf = (np.sin(np.arange(n * k, dtype=np.float32) * np.float32(0.1)) * np.float32(0.5)).astype(np.float32)
    raw = oq4.quantize_f32_to_q4_0(wf)
    act = (np.arange(k, dtype=np.float32) * np.float32(0.1)).reshape(1, 1, k)
    expected = oq4.reference_matmul(act.reshape(1, k), oq4.dequantize_q4_0(raw), 1, k, n)
    out = vx.q4_matmul(act, vx.Q4Tensor.from_q4_bytes(raw, (n, k)))
    assert out.shape == (1, 1, n)
    assert np.abs(out.reshape(1, n) - expected).max() < 1e-3


@pytest.mark.parametrize("batch,seq,k,n,tol", [(1, 1, 128, 64, 1e-2), (1, 10, 3072, 3072, 1e-2),
                                               (1, 1, 3072, 9216, 1e-2), (1, 1, 3072, 8192, 1e-2),
                                               (1, 38, 3072, 3072, 1e-2), (1, 1, 1280, 5120, 1e-2),
                                               (1, 100, 1280, 1280, 1e-2)])
def test_q4_matmul_shapes(vx, batch, seq, k, n, tol):
    i = np.arange(batch * seq * k, dtype=np.float32)
    act = (np.sin(i * np.float32(0.001)) * np.float32(0.1)).astype(np.float32).reshape(batch, seq, k)
    raw = oq4.quantize_f32_to_q4_0(closed_form_weights(n, k))
    expected = _ref(act.reshape(-1, k), raw, n, k)
    out = vx.q4_matmul(act, vx.Q4Tensor.from_q4_bytes(raw, (n, k)))
    assert out.shape == (batch, seq, n)
    assert np.abs(out.reshape(-1, n) - expected).max() < tol
    # and much tighter than the reference's bound: f32 summation-order differences only
    assert np.abs(out.reshape(-1, n) - expected).max() < 2e-4 * max(1.0, np.abs(expected).max())


def test_q4_matmul_batch(vx):
    batch, seq, k, n = 4, 10, 128, 64
    i = np.arange(batch * seq * k, dtype=np.float32)
    act = (np.sin(i * np.float32(0.001)) * np.float32(0.1)).astype(np.float32).reshape(batch, seq, k)
    raw = oq4.quantize_f32_to_q4_0(closed_form_weights(n, k))
    out = vx.q4_matmul(act, vx.Q4Tensor.from_q4_bytes(raw, (n, k)))
    assert np.abs(out.reshape(-1, n) - _ref(act.reshape(-1, k), raw, n, k)).max() < 1e-3


def test_q4_linear_forward_with_bias(vx):
    k, n = 64, 32
    wf = (np.sin(np.arange(n * k, dtype=np.float32) * np.float32(0.001)) * np.float32(0.1)).astype(np.float32)
    raw = oq4.quantize_f32_to_q4_0(wf)
    bias = (np.arange(n, dtype=np.float32) * np.float32(0.01)).astype(np.float32)
    act = (np.arange(k, dtype=np.float32) * np.float32(0.1)).reshape(1, 1, k)
    lin = vx.Q4Linear(vx.Q4Tensor.from_q4_bytes(raw, (n, k)), bias)
    expected = oq4.reference_matmul(act.reshape(1, k), oq4.dequantize_q4_0(raw), 1, k, n) + bias
    assert np.abs(lin.forward(act).reshape(1, n) - expected).max() < 1e-3


def test_q4_vs_unquantised_f32(vx):
    """tests/gguf_integration.rs:74-130: quantise -> q4_matmul vs f32 matmul, tol 0.5."""
    k, n, m = 256, 128, 4
    rng = np.random.default_rng(0)
    w = (rng.standard_normal((n, k)) * 0.1).astype(np.float32)
    x = (rng.standard_normal((1, m, k)) * 0.5).astype(np.float32)
    raw = oq4.quantize_f32_to_q4_0(w)
    out = vx.q4_matmul(x, vx.Q4Tensor.from_q4_bytes(raw, (n, k)))
    assert np.abs(out[0] - x[0] @ w.T).max() < 0.5


@pytest.mark.parametrize("m", list(range(1, 10)) + [17, 64, 65])
def test_q4_matmul_all_m_random_blocks(vx, m):
    """Random nibbles (all 16 values incl. 0) and random scales of either sign (real files carry negative ones);
    matvec (M<=8) and GEMM (M>8)."""
    n, k = 208, 2304  # N not a multiple of 16/64, K = 72 blocks (lanes unevenly loaded)
    rng = np.random.default_rng(m)
    raw = np.empty((n * k // 32, 18), np.uint8)
    d = rng.uniform(0.001, 0.02, n * k // 32) * rng.choice([-1.0, 1.0], n * k // 32)
    raw[:, :2] = d.astype(np.float16).view(np.uint8).reshape(-1, 2)
    raw[:, 2:] = rng.integers(0, 256, (n * k // 32, 16), dtype=np.uint8)
    raw[::7, 2:] = 0  # whole blocks of nibble 0 => -8*d
    raw = raw.reshape(-1)
    x = rng.standard_normal((1, m, k)).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    out = vx.q4_matmul(x, vx.Q4Tensor.from_q4_bytes(raw, (n, k)), bias)
    exp = _ref(x[0], raw, n, k, bias)
    scale = np.abs(exp).max()
    assert np.abs(out[0] - exp).max() < 2e-5 * scale + 1e-5


@pytest.mark.parametrize("m,n,k", [(130, 256, 1280), (586, 1280, 2048), (38, 384, 3072), (257, 128, 64)])
def test_q4_gemm_large_m_accuracy(vx, m, n, k):
    """Encoder / prefill sized GEMMs (N % 128 == 0, K % 64 == 0 => wgmma path in 'tc' mode): the
    2x2 f16 split keeps f32-grade accuracy (error ~ f32 summation-order noise, far below 1e-3)."""
    rng = np.random.default_rng(m + n)
    raw = np.empty((n * k // 32, 18), np.uint8)
    d = rng.uniform(0.002, 0.02, n * k // 32) * rng.choice([-1.0, 1.0], n * k // 32)
    raw[:, :2] = d.astype(np.float16).view(np.uint8).reshape(-1, 2)
    raw[:, 2:] = rng.integers(0, 256, (n * k // 32, 16), dtype=np.uint8)
    raw = raw.reshape(-1)
    x = (rng.standard_normal((1, m, k)) * rng.uniform(0.1, 3.0, (1, m, 1))).astype(np.float32)
    bias = rng.standard_normal(n).astype(np.float32)
    out = vx.q4_matmul(x, vx.Q4Tensor.from_q4_bytes(raw, (n, k)), bias)
    exp = _ref(x[0], raw, n, k, bias)
    err = np.abs(out[0] - exp).max()
    assert err < 3e-5 * np.abs(exp).max() + 1e-5, err


def test_q4_matvec_k_chunked(vx):
    """M=8 with K=9216 exceeds the shared-memory x tile => exercises the K-chunk path."""
    n, k, m = 64, 9216, 8
    rng = np.random.default_rng(5)
    raw = oq4.quantize_f32_to_q4_0((rng.standard_normal(n * k) * 0.02).astype(np.float32))
    x = rng.standard_normal((1, m, k)).astype(np.float32)
    out = vx.q4_matmul(x, vx.Q4Tensor.from_q4_bytes(raw, (n, k)))
    exp = _ref(x[0], raw, n, k)
    assert np.abs(out[0] - exp).max() < 2e-5 * np.abs(exp).max() + 1e-5


def test_q4_tensor_create_errors(vx):
    raw = np.zeros(18 * 4, np.uint8)
    with pytest.raises(vx.VoxtralError, match="byte count mismatch"):
        vx.Q4Tensor.from_q4_bytes(raw, (8, 32))
    with pytest.raises(vx.VoxtralError, match="divisible by 32|multiple of 32"):
        vx.Q4Tensor.from_q4_bytes(raw, (3, 17))
    t = vx.Q4Tensor.from_q4_bytes(raw, (4, 32))
    with pytest.raises(vx.VoxtralError, match="K dimension mismatch"):
        vx.q4_matmul(np.zeros((1, 1, 64), np.float32), t)
