"""CPU side of the fused linear-layer tests (tests/test_linear_forms_gpu.py runs vox_q4_linear on the same inputs).

Every linear layer of the model is  y[r] = epi(norm(x[r]) . W^T + bias) (+ res[r])  on one of four Q4 kernels
(launch_q4_linear).  This file holds the float64 reference of every form and its per-output error bound, and checks
that the bound is both safe (numpy models of the kernels' f32 arithmetic stay below a quarter of it) and tight (six
planted mistakes each exceed it).

The reference, in f64 on the f32 inputs:
    xh  = x / sqrt(mean(x^2) + eps) * gamma * ada[r // m]
    v   = xh . W64^T + bias
    y   = v | v + res | gelu_erf(v) | silu(v[:, 2i]) * v[:, 2i+1]

The bound (LinearRef.forward):
  * product: f64_and_bound (tests/test_q4_format_edges_ref.py) applied to xh: B_v;
  * norm: eps_rms(K) * |v64 - bias| + 2^-22 * |xh| . |W|^T.  The f32 rms is one factor common to the whole row, so
    its error scales the row's product, not the spread sum.  The per-element term covers the divide (or the
    reciprocal multiply) and the gamma and ADA products: three f32 roundings, 3 * 2^-24 < 2^-22;
  * residual: + 2^-22 |y64|.  The f32 add rounds at up to 2^-24 |y|; an exactly rounded result already reaches that,
    so the term carries the same factor 4 of margin the numpy models below are held to;
  * GELU: 1.13 B_v + 2^-22 |y64| + 2^-23 (max |gelu'| = 1.129; a few ulps of erff and the products);
  * SiLU*up: 1.1 B_g (|u64| + B_u) + |silu(g64)| B_u + 2^-21 |y64| + 2^-148 (max |silu'| = 1.0998; the last term is
    two roundings onto the f32 subnormal grid, 2^-150 each, for products that underflow: rows whose norm is eps).

eps_rms (rms_rel_bound): each kernel sums K squares in f32 (fmaf, or a rounded square then an add) as a chain of
sequential partial sums followed by a tree.  A recursive sum of d non-negative terms has relative error at most
gamma_d = d u / (1 - d u), u = 2^-24, with d the depth of the longest chain (+1 for a rounded square):
  * launch_rmsnorm: 256 threads, K/256 sequential terms each, then two 32-wide butterflies: d = K/256 + 10;
  * split_tiles_kernel (wgmma GEMM operand split): 32 threads per row, K/32 sequential terms each, then the 32
    partials added in order: d = K/32 + 32;
  * the hand-off (tensor-core matvec, ssq_in): 16 squares per tile in order, then ceil(K/16)/32 = K/512 partials per
    lane, then a 32-lane butterfly: d = 16 + 1 + K/512 + 5.
The deepest is split_tiles' for every K >= 64.  Then s / K, + eps and sqrt round once each (the sqrt halves the
relative error of its argument), and the reciprocal once more: eps_rms = (gamma_d + 2u) / 2 + 2u.

Activation sets that are run with a norm are those whose f32 sum of squares stays inside the f32 range: rows at 1e30
are run without one.  The kernels' f32 RMSNorm overflows there exactly as the reference model's does, so there is
nothing to compare.  Likewise a form whose f64 output leaves the f32 range (SiLU*up of rows at 1e30) is not run.
"""
import math

import numpy as np
import pytest

from oracle import q4 as oq4
from test_fragment_numerics import gemm_split_model, tc_matvec_model
from test_q4_format_edges_ref import f64_and_bound, largest_term, make_acts, make_weights, scales_of
from voxtral_mini_realtime_rs_b200.synth import random_q4_blocks

F32 = np.float32
U = 2.0 ** -24
EPS = 1e-5                                  # the model's norm_eps
EPIS = ("none", "residual", "silu_mul", "gelu")

# activation sets: make_acts' sets, and four that only matter under a norm
NORM_SETS = ("near_eps", "rows_1e15", "zero_rows", "outlier_row")
ACT_SETS = ("gauss", "outlier_1e4", "blocks_1e5", "zeros", "neg_zero", "f32_subnormal", "rows_1e-30", "rows_1e30") + \
    NORM_SETS


def norm_allowed(aset: str) -> bool:
    """rows at 1e30: the f32 sum of squares overflows (in the kernels and in the reference model alike)."""
    return aset != "rows_1e30"


def acts(aset: str, m: int, k: int, seed: int) -> np.ndarray:
    if aset not in NORM_SETS:
        return make_acts(aset, m, k, seed)
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((m, k)) * rng.uniform(0.5, 2.0, (m, 1))
    if aset == "near_eps":                  # mean square 0.3 .. 3 eps: eps decides the rms
        x = rng.standard_normal((m, k)) * math.sqrt(EPS) * np.geomspace(0.55, 1.7, m)[:, None]
    elif aset == "rows_1e15":               # sum of squares ~1e33 K: large, finite in f32
        x *= 1e15
    elif aset == "zero_rows":
        x[::2] = 0.0
    elif aset == "outlier_row":             # one element 1e6 in row 1: after the norm it is ~sqrt(K), the rest ~1e-6
        x[min(1, m - 1), k // 3] = 1e6
    return x.astype(F32)


# ------------------------------------------------------------------------------------------ the inputs of a layer


def make_gamma(k: int, seed: int) -> np.ndarray:
    """around 1, with a few zeros and negative entries"""
    rng = np.random.default_rng(seed)
    g = 1.0 + 0.2 * rng.standard_normal(k)
    g[rng.integers(0, k, max(1, k // 97))] = 0.0
    g[rng.integers(0, k, max(1, k // 53))] *= -1.0
    return g.astype(F32)


def make_ada(streams: int, k: int, seed: int) -> np.ndarray:
    """one vector per stream, all distinct (1 + w2(gelu(w0 t)) is near 1); stream 1's has zeros"""
    rng = np.random.default_rng(seed)
    a = 1.0 + 0.5 * rng.standard_normal((streams, k))
    if streams > 1:
        a[1, ::7] = 0.0
    return a.astype(F32)


def make_res(m: int, n: int, seed: int) -> np.ndarray:
    """rows of varied magnitude, 1e-3 .. 1e3"""
    rng = np.random.default_rng(seed)
    return (rng.standard_normal((m, n)) * np.geomspace(1e-3, 1e3, m)[:, None]).astype(F32)


def make_bias(n: int, seed: int) -> np.ndarray:
    return np.random.default_rng(seed).standard_normal(n).astype(F32)


def weights(kind: str, n: int, k: int, seed: int) -> np.ndarray:
    """Q4_0 bytes: random_q4_blocks (the synthetic model's weights) or the format-edges "signed" set (negative
    scales)"""
    if kind == "signed":
        return make_weights("signed", n, k, seed)
    return random_q4_blocks(np.random.default_rng(seed), n * k, 0.02)


# ----------------------------------------------------------------------------------------- reference and bound


def rms_rel_bound(k: int) -> float:
    d = max(k / 256 + 10, k / 32 + 32, 16 + 1 + math.ceil(math.ceil(k / 16) / 32) + 5)
    gam = d * U / (1 - d * U)
    return (gam + 2 * U) / 2 + 2 * U


def gelu64(v):
    from scipy.special import erf
    return 0.5 * v * (1.0 + erf(v / math.sqrt(2.0)))


def silu64(v):
    with np.errstate(over="ignore"):                  # exp(-v) = inf: silu(v) = -0
        return v / (1.0 + np.exp(-v))


class LinearRef:
    """One Q4 weight, dequantised once, and the f64 reference + bound of any fused form over it."""

    def __init__(self, raw: np.ndarray, n: int, k: int):
        self.raw, self.n, self.k = raw, n, k
        self.w = oq4.dequantize_q4_0(raw).reshape(n, k).astype(np.float64)
        self.aw = np.abs(self.w)
        self.wd = self.aw + 16.0 * np.abs(scales_of(raw, n, k))

    def product(self, x64: np.ndarray, bias=None):
        """f64_and_bound over this weight (the same formula, without dequantising again)"""
        y = x64 @ self.w.T
        bound = 2.0 ** -20 * (np.abs(x64) @ self.wd.T) + 2.0 ** -15 * largest_term(x64, self.wd)
        if bias is not None:
            y = y + bias.astype(np.float64)
            bound = bound + np.abs(bias.astype(np.float64)) * 2.0 ** -23
        return y, bound

    @staticmethod
    def normed(x, gamma, eps=EPS, ada=None, ada_m=1, perturb=None):
        x64 = x.astype(np.float64)
        ms = np.mean(x64 * x64, axis=1, keepdims=True)
        e = 0.0 if perturb == "no_eps" else float(F32(eps))
        rms = np.sqrt(ms + e)                         # a zero row without eps gives NaN: a planted mistake
        if perturb == "rms_next":
            rms = np.roll(rms, -1, axis=0)
        with np.errstate(invalid="ignore"):
            xh = x64 / rms * gamma.astype(np.float64)
        if ada is not None:
            s = np.arange(x.shape[0]) // ada_m
            if perturb == "ada_next":
                s = (s + 1) % ada.shape[0]
            xh = xh * ada.astype(np.float64)[s]
        return xh

    def forward(self, x, epi="none", bias=None, res=None, gamma=None, eps=EPS, ada=None, ada_m=1, perturb=None):
        """(y64, bound) of the form; `perturb` names a planted mistake (the bound stays the correct form's)"""
        if gamma is not None:
            xh = self.normed(x, gamma, eps, ada, ada_m)
            v, bv = self.product(xh, bias)
            vb = v - (0.0 if bias is None else bias.astype(np.float64))
            bv = bv + rms_rel_bound(self.k) * np.abs(vb) + 2.0 ** -22 * (np.abs(xh) @ self.aw.T)
            if perturb in ("no_eps", "rms_next", "ada_next"):
                v = self.normed(x, gamma, eps, ada, ada_m, perturb) @ self.w.T + (0.0 if bias is None else bias)
        else:
            v, bv = self.product(x.astype(np.float64), bias)
        if epi == "none":
            return v, bv
        if epi == "residual":
            y = v + res.astype(np.float64)
            yp = y + res.astype(np.float64) if perturb == "res_twice" else y
            return yp, bv + 2.0 ** -22 * np.abs(y)
        if epi == "gelu":
            y = gelu64(v)
            yp = 0.5 * v * (1.0 + np.tanh(math.sqrt(2.0 / math.pi) * (v + 0.044715 * v ** 3))) \
                if perturb == "gelu_tanh" else y
            return yp, 1.13 * bv + 2.0 ** -22 * np.abs(y) + 2.0 ** -23
        assert epi == "silu_mul"
        g, u, bg, bu = v[:, 0::2], v[:, 1::2], bv[:, 0::2], bv[:, 1::2]
        y = silu64(g) * u
        yp = silu64(u) * g if perturb == "swap_gate_up" else y
        return yp, 1.1 * bg * (np.abs(u) + bu) + np.abs(silu64(g)) * bu + 2.0 ** -21 * np.abs(y) + 2.0 ** -148


# ------------------------------------------------------------------- numpy models of the kernels' f32 arithmetic


def _butterfly(v: np.ndarray) -> np.ndarray:
    """warp_sum over the last axis (32 lanes): v += shfl_xor(v, o) for o = 16 .. 1; every lane ends with the sum"""
    v = v.astype(F32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(F32)
    return v[..., 0]


def _seq_sum(terms: np.ndarray, fma: bool) -> np.ndarray:
    """sequential f32 sum over axis 1 of [rows, n, ...]: s = fmaf(t, t, s) (fma) or s += t"""
    s = np.zeros((terms.shape[0],) + terms.shape[2:], F32)
    for j in range(terms.shape[1]):
        t = terms[:, j].astype(np.float64)
        s = ((t * t if fma else t) + s.astype(np.float64)).astype(F32)
    return s


def ssq_rmsnorm(x: np.ndarray) -> np.ndarray:
    """launch_rmsnorm: thread t of 256 runs fmaf over i = t, t + 256, ..; two butterflies over 8 warps of 32"""
    m, k = x.shape
    xp = np.zeros((m, -(-k // 256) * 256), F32)
    xp[:, :k] = x
    part = _seq_sum(xp.reshape(m, -1, 256), fma=True)             # [m, 256]
    warp = _butterfly(part.reshape(m, 8, 32))                     # [m, 8]
    red = np.zeros((m, 32), F32)
    red[:, :8] = warp
    return _butterfly(red)


def ssq_split_tiles(x: np.ndarray) -> np.ndarray:
    """split_tiles_kernel: thread cth of 32 runs fmaf over the 8 elements of chunks cth, cth + 32, ..; then the 32
    partials in order"""
    m, k = x.shape
    t = x.reshape(m, k // 256, 32, 8).transpose(0, 1, 3, 2).reshape(m, -1, 32)   # [m, step, cth]
    part = _seq_sum(t, fma=True)                                  # [m, 32]
    return _seq_sum(part[:, :, None], fma=False)[:, 0]


def ssq_parts(y: np.ndarray) -> np.ndarray:
    """the residual epilogue's hand-off: [ceil(N/16)][rows] sums of 16 rounded squares in order (zeros past N)"""
    m, n = y.shape
    yp = np.zeros((m, -(-n // 16) * 16), F32)
    yp[:, :n] = y
    sq = (yp.astype(F32) * yp.astype(F32)).astype(F32).reshape(m, -1, 16)
    return _seq_sum(sq.transpose(0, 2, 1), fma=False).T           # [parts, m]


def ssq_handoff(parts: np.ndarray) -> np.ndarray:
    """q4_matvec_tc_kernel with ssq_in: lane l adds parts l, l + 32, .. in order, then a butterfly"""
    p, m = parts.shape
    pp = np.zeros((-(-p // 32) * 32, m), F32)
    pp[:p] = parts
    lane = _seq_sum(pp.reshape(-1, 32, m).transpose(2, 0, 1), fma=False)   # [m, 32]
    return _butterfly(lane)


def norm_model(x, gamma, eps, ada, ada_m, ssq, recip: bool) -> np.ndarray:
    """f32 x / rms * gamma * ada from a row's f32 sum of squares: x / rms (launch_rmsnorm, split_tiles) or
    x * (1 / rms) (the tensor-core matvec)"""
    m, k = x.shape
    rms = np.sqrt((ssq / F32(k)).astype(F32) + F32(eps)).astype(F32)[:, None]
    if recip:
        v = (x * (F32(1.0) / rms).astype(F32)).astype(F32)
    else:
        v = (x / rms).astype(F32)
    v = (v * gamma).astype(F32)
    if ada is not None:
        v = (v * ada[np.arange(m) // ada_m]).astype(F32)
    return v


def epilogue_model(v: np.ndarray, epi: str, bias, res) -> np.ndarray:
    """the kernels' f32 epilogue on f32 products v [m, n]"""
    from scipy.special import erf
    if epi == "silu_mul":
        g, u = v[:, 0::2].astype(F32), v[:, 1::2].astype(F32)
        return ((g / (F32(1.0) + np.exp(-g).astype(F32))).astype(F32) * u).astype(F32)
    if bias is not None:
        v = (v + bias).astype(F32)
    if epi == "residual":
        v = (v + res).astype(F32)
    if epi == "gelu":
        v = (F32(0.5) * v * (F32(1.0) + erf(v.astype(np.float64) / math.sqrt(2.0)).astype(F32))).astype(F32)
    return v.astype(F32)


def kernel_model(kernel: str, ref: LinearRef, x, epi="none", bias=None, res=None, gamma=None, eps=EPS, ada=None,
                 ada_m=1) -> np.ndarray:
    """numpy model of one form on one kernel path:
       "tc": launch_rmsnorm then the tensor-core matvec; "handoff": the matvec's own norm from ssq_in;
       "gemm": split_tiles' norm then the wgmma GEMM"""
    x = x.astype(F32)
    if gamma is not None:
        if kernel == "tc":
            x = norm_model(x, gamma, eps, ada, ada_m, ssq_rmsnorm(x), recip=False)
        elif kernel == "handoff":
            x = norm_model(x, gamma, eps, ada, ada_m, ssq_handoff(ssq_parts(x)), recip=True)
        else:
            x = norm_model(x, gamma, eps, ada, ada_m, ssq_split_tiles(x), recip=False)
    with np.errstate(all="ignore"):
        if kernel == "gemm":
            v = gemm_split_model(x, ref.raw, ref.n, ref.k).astype(F32)
        else:
            v = np.stack([tc_matvec_model(x[i], ref.raw, ref.n, ref.k) for i in range(x.shape[0])]).astype(F32)
        return epilogue_model(v, epi, bias, res)


def ratio(got, y64, bound) -> np.ndarray:
    err = np.abs(np.asarray(got, np.float64) - y64)
    return np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), np.where(err > 0, np.inf, 0.0))


# --------------------------------------------------------------------------------------------------- the tests

N, K, M, STREAMS = 32, 3072, 6, 3          # ada_m = 2: rows (0, 1), (2, 3), (4, 5) are three streams


def _inputs(aset, seed=0):
    x = acts(aset, M, K, 100 + seed)
    return dict(x=x, bias=make_bias(N, 1 + seed), res=make_res(M, N, 2 + seed), gamma=make_gamma(K, 3 + seed),
                ada=make_ada(STREAMS, K, 4 + seed))


@pytest.fixture(scope="module", params=["random", "signed"])
def ref(request):
    return LinearRef(weights(request.param, N, K, 5), N, K)


def _forms(inp, aset):
    """(name, kwargs) of every form: each epilogue, without a norm, with a norm, with a norm and ADA"""
    out = []
    for epi in EPIS:
        base = dict(epi=epi, bias=None if epi == "silu_mul" else inp["bias"],
                    res=inp["res"] if epi == "residual" else None)
        if epi != "silu_mul" or aset != "rows_1e30":
            out.append((f"{epi}", base))
        if norm_allowed(aset):
            out.append((f"{epi}+norm", dict(base, gamma=inp["gamma"])))
            out.append((f"{epi}+norm+ada", dict(base, gamma=inp["gamma"], ada=inp["ada"], ada_m=M // STREAMS)))
    return out


def test_product_bound_is_f64_and_bound():
    raw = weights("signed", 24, 256, 9)
    r = LinearRef(raw, 24, 256)
    x = acts("outlier_1e4", 3, 256, 1)
    b = make_bias(24, 2)
    y, bd = r.product(x.astype(np.float64), b)
    y2, bd2 = f64_and_bound(raw, 24, 256, x, b)
    assert np.array_equal(y, y2) and np.array_equal(bd, bd2)


def test_rms_bound_takes_the_deepest_sum():
    for k in (96, 1280, 3072, 4192, 5120, 9216):
        d = k / 32 + 32
        assert d >= k / 256 + 10 and d >= 22 + k / 512
        assert d * U / 2 < rms_rel_bound(k) < (d / 2 + 4) * U, k    # half the chain's gamma_d, plus four roundings


def test_ssq_models_agree_with_f64():
    """the four f32 sums of squares are f32 sums of the same terms: within their depth's gamma_d of the f64 sum"""
    x = acts("gauss", M, K, 3)
    s64 = np.sum(x.astype(np.float64) ** 2, axis=1)
    for name, s in (("rmsnorm", ssq_rmsnorm(x)), ("split", ssq_split_tiles(x)),
                    ("handoff", ssq_handoff(ssq_parts(x)))):
        rel = np.abs(s.astype(np.float64) - s64) / s64
        assert rel.max() < 2 * rms_rel_bound(K), (name, rel.max())
        assert rel.max() > 0, name                                 # f32 arithmetic, not exact


@pytest.mark.parametrize("aset", ACT_SETS)
def test_models_within_a_quarter_of_the_bound(ref, aset):
    """Every form on the models of the kernels that run it: "tc" (launch_rmsnorm + the tensor-core matvec),
    "handoff" (the matvec's norm from the residual epilogue's sums of squares) and "gemm" (split_tiles + the wgmma
    GEMM, in-domain weights only)."""
    inp = _inputs(aset)
    worst = {}
    for name, kw in _forms(inp, aset):
        y64, bound = ref.forward(inp["x"], **kw)
        kernels = ["tc", "gemm"] + (["handoff"] if "norm" in name else [])
        for kern in kernels:
            got = kernel_model(kern, ref, inp["x"], **kw)
            r = float(ratio(got, y64, bound).max())
            worst[f"{kern} {name}"] = r
    top = sorted(worst.items(), key=lambda kv: -kv[1])[:3]
    print(f"\n[linear forms model / bound] {aset:>13s}: " + "  ".join(f"{k} {v:.3f}" for k, v in top))
    assert max(worst.values()) < 0.25, top


PLANTED = {
    "no_eps": dict(epi="none", norm=True),
    "ada_next": dict(epi="none", norm=True, ada=True),
    "rms_next": dict(epi="none", norm=True),
    "swap_gate_up": dict(epi="silu_mul", norm=True),
    "res_twice": dict(epi="residual", norm=False),
    "gelu_tanh": dict(epi="gelu", norm=False),
}


@pytest.mark.parametrize("perturb", list(PLANTED))
def test_planted_mistakes_exceed_the_bound(ref, perturb):
    """Each planted mistake, applied to the f64 reference, exceeds the correct form's bound on at least one output of
    the activation sets (the GELU one on its outputs near |v| ~ 2, eps on the near_eps rows)."""
    p = PLANTED[perturb]
    worst = {}
    for aset in ACT_SETS:
        if p["norm"] and not norm_allowed(aset):
            continue
        inp = _inputs(aset)
        kw = dict(epi=p["epi"], bias=None if p["epi"] == "silu_mul" else inp["bias"],
                  res=inp["res"] if p["epi"] == "residual" else None)
        if p["norm"]:
            kw["gamma"] = inp["gamma"]
        if p.get("ada"):
            kw.update(ada=inp["ada"], ada_m=M // STREAMS)
        y64, bound = ref.forward(inp["x"], **kw)
        yp, _ = ref.forward(inp["x"], perturb=perturb, **kw)
        worst[aset] = float(ratio(yp, y64, bound).max())
    best = max(worst, key=worst.get)
    print(f"\n[planted {perturb}] largest |planted - y64| / bound = {worst[best]:.3g} ({best})")
    assert worst[best] > 1.0, worst
    if perturb == "no_eps":
        assert worst["near_eps"] > 1.0
