"""CPU side of the decoder attention tests (tests/test_dec_attention_gpu.py runs vox_dec_attention on the same kind of
inputs).

The decoder attention kernels -- K5 fused (dec_attn_fused_kernel, decode_attn.cu) and K5 prefill (dec_rope_append_kernel
then dec_attention_kernel, kernels.cu) -- compute, per (row, head h), at position p:
    q' = RoPE(q, p),  o = sum_j softmax_j(scale q' . K_j) V_j  over the keys j in max(0, p - window) .. p
of kv head h / G (G = H / Hkv), where K_j and V_j are what the cache holds (K after RoPE), read through the row's page
table.  This file holds the float64 reference, its per-output bound, numpy models of both kernels' f32 arithmetic in
their own order, and planted mistakes.

The reference (f64_and_bound) takes q in f32 before RoPE and the caller's f32 cos / sin row, rotates q in float64, and
reads K and V as stored, decoded exactly (f32 as is, f16 widened, q8 as d * q), so the rounding of the storage rule
never enters the bound.  Per output (row, d):
  * scores: ds_j = |scale| (2^-22 sum_d R_d |K_jd| + gamma_dot sum_d |q'_d K_jd|) + 2^-21 (|s_j| + |m|) + 2^-21.
    R_d = |x_r c| + |x_i s| (resp. |x_r s| + |x_i c|) is the size of q'_d's rotation terms: the f32 rotation is off by
    at most 2^-22 R_d with or without FMA contraction.  gamma_dot = gamma(n) with n the dot product's depth: hd / 32 + 5
    in the fused kernel (per-lane FMAs, then a 5-level xor butterfly), hd in dec_attention_kernel (one sequential fmaf
    chain) -- at hd 128 that is 2^-17, looser than the encoder file's 2^-20.  The rest covers the scale multiply, the
    subtraction of the maximum and a few ulps of expf.  A score error moves o by sum_j p_j ds_j |V_jd - o_d|;
  * sums: (gamma(n_sum) + 2^-21) (sum_j p_j |V_jd| + |o_d|).  Fused: n_sum = 4 ceil(n / 8) + 24 -- each warp's online
    softmax rounds acc * alpha and the FMA at every key, and each fresh alpha = expf(m_old - m_new) (a new one at every
    key where the running max rises) weights the earlier keys by up to 2 ulps differently from the later ones; then 8
    warp states merge.  Prefill: n_sum = n + ceil(n / 32) + 16 -- a two-pass softmax with a sequential P V over all n
    keys and lane-strided sums of p;
  * floor: 2^-100 max |V| + 2^-126, for p underflowing far below the maximum.

Checked here: both models stay below a quarter of the bound on every operand set; each planted mistake exceeds it by at
least SEPARATION (10).
"""
import numpy as np
import pytest
import torch

from test_attention_ref import _tree32, expf, f32, fma, ratio
from test_kv_q8_ref import kv8_decode, kv8_quant

U = 2.0 ** -24
SEPARATION = 10
F32 = np.float32
WARPS = 8             # dec_attn_fused_kernel's DA_WARPS
THETA = 1e6           # the decoder's RoPE base (oracle/model.py rope_tables)


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1 - n * U)


def rope_rows(positions, hd):
    """f32 cos / sin rows [len(positions), hd / 2] of the decoder's RoPE (oracle/model.py rope_tables' rule)"""
    half = hd // 2
    inv = np.array([F32(1.0) / np.power(F32(THETA), F32(2 * i) / F32(hd)) for i in range(half)], F32)
    fr = (np.asarray(positions, F32)[:, None] * inv[None, :]).astype(F32)
    return np.cos(fr).astype(F32), np.sin(fr).astype(F32)


def rotate64(x, c, s):
    """RoPE in float64 of f32 x [..., hd] by f32 rows c, s [..., hd / 2] -> (x', R), R the rotation terms' size"""
    x, c, s = (np.asarray(a, np.float64) for a in (x, c, s))
    xr, xi = x[..., 0::2], x[..., 1::2]
    out, mag = np.empty_like(x), np.empty_like(x)
    out[..., 0::2], out[..., 1::2] = xr * c - xi * s, xr * s + xi * c
    mag[..., 0::2], mag[..., 1::2] = np.abs(xr * c) + np.abs(xi * s), np.abs(xr * s) + np.abs(xi * c)
    return out, mag


def unrotate(xr, c, s):
    """the f32 x whose float64 RoPE is (close to) the wanted xr: operand sets are defined after RoPE"""
    xr, c, s = (np.asarray(a, np.float64) for a in (xr, c, s))
    a, b = xr[..., 0::2], xr[..., 1::2]
    out = np.empty_like(xr)
    out[..., 0::2], out[..., 1::2] = a * c + b * s, b * c - a * s
    return out.astype(F32)


def f64_and_bound(kernel, q, c, s, k, v, mask, scale):
    """Rows of one head: q [nq, hd] f32 before RoPE, c / s [nq, hd / 2] f32, k and v [m, hd] as stored (exact in f64),
    mask [nq, m] the keys each row sees -> (o64, bound), both [nq, hd].  kernel: "fused" or "prefill"."""
    hd = q.shape[-1]
    qr, mag = rotate64(q, c, s)
    k64, v64 = np.asarray(k, np.float64), np.asarray(v, np.float64)
    scale = float(F32(scale))
    sc = scale * (qr @ k64.T)
    sc = np.where(mask, sc, -np.inf)
    mx = sc.max(1, keepdims=True)
    e = np.where(mask, np.exp(sc - mx), 0.0)
    p = e / e.sum(1, keepdims=True)
    o = p @ v64
    ak, av = np.abs(k64), np.abs(v64)
    n = mask.sum(1, keepdims=True).astype(np.float64)
    g_dot = gamma(hd // 32 + 5 if kernel == "fused" else hd)
    ds = abs(scale) * (2.0 ** -22 * (mag @ ak.T) + g_dot * ((np.abs(qr) + 2.0 ** -22 * mag) @ ak.T))
    ds = ds + 2.0 ** -21 * (np.abs(np.where(mask, sc, 0.0)) + np.abs(mx)) + 2.0 ** -21
    w = p * ds
    sens = np.empty_like(o)
    step = max(1, (1 << 22) // max(1, k64.size))
    for i0 in range(0, len(o), step):                    # sum_j w_ij |v_jd - o_id|, a few rows at a time
        sl = slice(i0, i0 + step)
        sens[sl] = torch.einsum("ij,ijd->id", torch.from_numpy(w[sl]),
                                (torch.from_numpy(v64)[None] - torch.from_numpy(o[sl])[:, None]).abs()).numpy()
    n_sum = 4 * np.ceil(n / WARPS) + 24 if kernel == "fused" else n + np.ceil(n / 32) + 16
    vmax = np.where(mask[:, :, None], av[None], 0.0).max((1, 2))[:, None]
    return o, sens + (gamma(n_sum) + 2.0 ** -21) * (p @ av + np.abs(o)) + 2.0 ** -100 * vmax + 2.0 ** -126


# ------------------------------------------------------------------------------------------------ operand sets

OPERAND_SETS = ("gauss", "one_hot", "edge_key", "outside_key", "v_offset", "qk_2^-16", "qk_2^+16", "v_2^-16", "v_2^+16",
                "rising", "q8_blocks", "f16_range")


def operands(aset, nq, n_keys, hd, seed, edge=None):
    """One head: q' [nq, hd] (after RoPE), K and V [n_keys, hd] (K after RoPE), float64; the queries sit at the last nq
    keys.  edge: the key index of the last query's oldest visible key (edge_key and outside_key put a dominant key there
    or one before it).  f16_range: K and V past the f16 range, which an f16 cache stores clamped to +-65504."""
    rng = np.random.default_rng(seed)
    q, k, v = rng.standard_normal((nq, hd)), rng.standard_normal((n_keys, hd)), rng.standard_normal((n_keys, hd))
    if aset.startswith("qk_"):
        f = 2.0 ** float(aset.split("^")[1])
        q, k = q * f, k * f
    elif aset.startswith("v_2"):
        v = v * 2.0 ** float(aset.split("^")[1])
    elif aset == "one_hot":                        # each query's own key wins by a score gap of 120 over the one before
        q[:, 0] = 40.0 * np.sqrt(hd)
        k[:, 0] = 3.0 * np.arange(n_keys)
    elif aset in ("edge_key", "outside_key"):      # a dominant key at the oldest visible position (or one before it)
        at = (0 if edge is None else edge) - (aset == "outside_key")
        if 0 <= at < n_keys:
            k[at] = 6.0 * q[-1] / np.sqrt(hd)
    elif aset == "v_offset":                       # |v - o| << |v|
        v = 1000.0 + 0.01 * v
    elif aset == "rising":                         # scores rise by 0.25 key by key: the running max moves at every key
        q = 0.01 * q
        q[:, 0] = 4.0
        k[:, 0] = 0.25 * np.arange(n_keys) / (4.0 / np.sqrt(hd))
    elif aset == "q8_blocks":                      # an all-zero 16-dim block of K and of V, and a block with one outlier
        k[:, 16:32], v[:, :16] = 0.0, 0.0
        k[:, 3] *= 300.0
        v[:, 20] *= 300.0
    elif aset == "f16_range":
        q = q / 65536.0
        k[:, ::3] *= 70000.0
        v[:, ::5] *= 70000.0
    return q, k, v


# ------------------------------------------------------------------------------------------------ f32 models


def rope_f32(x, c, s):
    """the kernels' f32 rotation, each product rounded (no FMA contraction)"""
    xr, xi = x[..., 0::2], x[..., 1::2]
    out = np.empty(x.shape, F32)
    out[..., 0::2] = f32(f32(xr * c) - f32(xi * s))
    out[..., 1::2] = f32(f32(xr * s) + f32(xi * c))
    return out


def model_fused(q, c, s, k, v, scale, mistake=None):
    """dec_attn_fused_kernel for one row and the G heads of a kv group: q [G, hd] f32 before RoPE, c / s [hd / 2], k / v
    [n, hd] the visible keys in order (key t of the window goes to warp t % 8).  Lane l owns dims l * hd/32 ..; a key's
    score is a per-lane fmaf chain and the xor butterfly; online softmax per key; the 8 warp states merge in order
    through expf(m_w - mx).  mistake: "alpha_acc", "alpha_l" (that rescale dropped), "merge_factor" (warps merged
    without their factor)."""
    G, hd = q.shape
    dpl = hd // 32
    scale = F32(scale)
    qr = rope_f32(q, c, s).reshape(G, 32, dpl)
    kk = np.asarray(k, F32).reshape(-1, 32, dpl)
    part = np.zeros((len(kk), G, 32), F32)
    for i in range(dpl):
        part = fma(qr[None, :, :, i], kk[:, None, :, i], part)
    sc = f32(_tree32(part) * scale)                       # [n, G]
    vv = np.asarray(v, F32)
    ms, ls, accs = [], [], []
    for w in range(WARPS):
        m, l, acc = np.full(G, -np.inf, F32), np.zeros(G, F32), np.zeros((G, hd), F32)
        for t in range(w, len(kk), WARPS):
            m_new = np.maximum(m, sc[t])
            alpha, p = expf(m - m_new), expf(sc[t] - m_new)
            l = fma(l, F32(1) if mistake == "alpha_l" else alpha, p)
            m = m_new
            acc = fma(p[:, None], vv[t][None], acc if mistake == "alpha_acc" else f32(acc * alpha[:, None]))
        ms.append(m), ls.append(l), accs.append(acc)
    mx = np.max(ms, 0)
    num, den = np.zeros((G, hd), F32), np.zeros(G, F32)
    for w in range(WARPS):
        f = np.where(ms[w] == -np.inf, F32(0), F32(1) if mistake == "merge_factor" else expf(ms[w] - mx))
        num, den = fma(accs[w], f[:, None], num), fma(ls[w], f, den)
    return f32(num / den[:, None])


def model_prefill(q, c, s, k, v, scale):
    """dec_attention_kernel (after dec_rope_append_kernel's rotation) for one row and the G heads of a kv group: one warp
    per head, lane l scores keys l, l + 32, .. with a sequential fmaf over hd; the warp max, expf, lane sums and the xor
    butterfly; then per dim a sequential fmaf P V over all keys, times 1 / sum."""
    G, hd = q.shape
    scale = F32(scale)
    qr = rope_f32(q, c, s)
    kk, vv = np.asarray(k, F32), np.asarray(v, F32)
    n = len(kk)
    acc = np.zeros((G, n), F32)
    for d in range(hd):
        acc = fma(qr[:, d:d + 1], kk[None, :, d], acc)
    sc = f32(acc * scale)
    mx = sc.max(1, keepdims=True)
    p = expf(sc - mx)
    lanes = np.zeros((G, 32), F32)
    for t0 in range(0, n, 32):
        blk = p[:, t0:t0 + 32]
        lanes[:, :blk.shape[1]] = f32(lanes[:, :blk.shape[1]] + blk)
    inv = f32(F32(1) / _tree32(lanes))
    o = np.zeros((G, hd), F32)
    for t in range(n):
        o = fma(p[:, t:t + 1], vv[t][None], o)
    return f32(o * inv[:, None])


MODELS = {"fused": model_fused, "prefill": model_prefill}


# ------------------------------------------------------------------------------------------------ scenarios


class Scene:
    """One row of one kv group: G query heads at position pos, the cache's keys 0 .. pos of kv head 0 (and a second kv
    head and a second row holding other keys, for the mistakes that read them), stored as f32 or q8."""

    def __init__(self, aset, G, hd, pos, window, seed, kv="f32", rope_ring=None):
        self.G, self.hd, self.pos, self.window = G, hd, pos, window
        self.j_lo = max(0, pos - window)
        n = pos + 1
        self.scale = float(F32(hd) ** F32(-0.5))
        qs, ks, vs = zip(*(operands(aset, 1, n, hd, seed + h, edge=self.j_lo) for h in range(G)))
        k = np.stack([ks[0], operands("gauss", 1, n, hd, seed + 99)[1]])       # [kv head, n, hd]
        v = np.stack([vs[0], operands("gauss", 1, n, hd, seed + 98)[2]])
        self.c, self.s = (t[0] for t in rope_rows([pos], hd))
        self.rope_ring = rope_ring
        self.q = unrotate(np.concatenate(qs), self.c, self.s)                   # [G, hd] f32 before RoPE
        self.kv = kv
        if kv == "q8":
            (self.kq, self.kd), (self.vq, self.vd) = kv8_quant(k.astype(F32)), kv8_quant(v.astype(F32))
            self.k, self.v = kv8_decode(self.kq, self.kd), kv8_decode(self.vq, self.vd)
        else:
            self.k, self.v = k.astype(F32), v.astype(F32)
        self.other_row = (f32(operands("gauss", 1, n, hd, seed + 97)[1]), f32(operands("gauss", 1, n, hd, seed + 96)[2]))

    def keys(self):
        return np.arange(self.j_lo, self.pos + 1)

    def ref(self, kernel):
        """(o64, bound) [G, hd]"""
        j = self.keys()
        mask = np.ones((1, len(j)), bool)
        outs = [f64_and_bound(kernel, self.q[h:h + 1], self.c[None], self.s[None], self.k[0, j], self.v[0, j], mask,
                              self.scale) for h in range(self.G)]
        return np.concatenate([o for o, _ in outs]), np.concatenate([b for _, b in outs])

    def model(self, kernel, mistake=None):
        j = self.keys()
        kw = {"mistake": mistake} if mistake else {}
        return MODELS[kernel](self.q, self.c, self.s, self.k[0, j], self.v[0, j], self.scale, **kw)

    def f64(self, q=None, c=None, s=None, k=None, v=None, keys=None, heads_kv=None):
        """float64 attention of every head with one thing changed (a planted mistake)"""
        q = self.q if q is None else q
        c, s = (self.c if c is None else c), (self.s if s is None else s)
        j = self.keys() if keys is None else keys
        out = []
        for h in range(self.G):
            g = 0 if heads_kv is None else heads_kv[h]
            kk = (self.k[g] if k is None else k)[j]
            vv = (self.v[g] if v is None else v)[j]
            out.append(f64_and_bound("fused", q[h:h + 1], c[None], s[None], kk, vv, np.ones((1, len(j)), bool),
                                     self.scale)[0])
        return np.concatenate(out)


def _q8_shifted(q, d, how):
    """q8 values decoded with a neighbouring scale: of the next block, or of the next position"""
    if how == "block":
        d = d[..., np.arange(d.shape[-1]) ^ 1]
    else:
        d = np.concatenate([d[..., 1:, :], d[..., -2:-1, :]], -2)
    return kv8_decode(q, d)


# ------------------------------------------------------------------------------------------------ checks


PROBES = [  # (G, hd, pos, window)
    (4, 128, 300, 8192), (4, 128, 300, 40), (2, 64, 130, 7), (1, 32, 97, 8), (4, 32, 600, 383), (1, 128, 12, 0),
]


@pytest.mark.parametrize("aset", OPERAND_SETS)
def test_models_within_a_quarter_of_the_bound(aset):
    worst = {}
    for kv in ("f32", "q8"):
        for G, hd, pos, window in PROBES:
            sc = Scene(aset, G, hd, pos, window, G + hd + pos + window, kv=kv)
            for kernel in MODELS:
                o64, bound = sc.ref(kernel)
                r = float(ratio(sc.model(kernel), o64, bound).max())
                worst[kernel] = max(worst.get(kernel, 0.0), r)
    for kernel, w in worst.items():
        print(f"\n[dec attention models] {aset:12s} {kernel:8s} worst |model - o64| / bound = {w:.3f}")
        assert w < 0.25, (aset, kernel, w)


def test_bound_is_looser_for_the_sequential_dot_product():
    """at hd 128 the prefill kernel's hd-deep fmaf chain gets gamma(128) ~ 2^-17, the fused kernel gamma(9)"""
    sc = Scene("gauss", 1, 128, 200, 8192, 5)
    assert np.all(sc.ref("prefill")[1] > sc.ref("fused")[1])


def _planted(mistake, aset, G, hd, pos, window, seed):
    kv = "q8" if mistake.startswith("q8_") else "f32"
    sc = Scene(aset, G, hd, pos, window, seed, kv=kv)
    kernel = "prefill" if mistake == "prefill_row0_pos" else "fused"
    o64, bound = sc.ref(kernel)
    j = sc.keys()
    if mistake in ("window-1", "window+1"):
        w = window + int(mistake[6:])
        got = sc.f64(keys=np.arange(max(0, pos - w), pos + 1))
    elif mistake == "j<pos":
        got = sc.f64(keys=j[:-1])
    elif mistake == "prefill_row0_pos":       # row i of a prefill scoring the keys of row 0 (pos - 5): i = 5
        got = sc.f64(keys=np.arange(max(0, pos - 5 - window), pos - 5 + 1))
    elif mistake == "rope_row+1":
        c, s = (t[0] for t in rope_rows([pos + 1], hd))
        got = sc.f64(c=c, s=s)
    elif mistake == "rope_unwrapped":         # row pos of a 4096-row ring table: a row filled for another position
        c, s = (t[0] for t in rope_rows([pos - 4096], hd))
        got = sc.f64(c=c, s=s)
    elif mistake == "q_unrotated":
        got = sc.f64(c=np.ones(hd // 2, F32), s=np.zeros(hd // 2, F32))
    elif mistake == "kv_head_h%Hkv":          # Hkv = 2: head h reads kv head h % 2 in place of h / G
        got = sc.f64(heads_kv=[h % 2 for h in range(G)])
    elif mistake == "page_row_b-1":           # the keys of the row before, through its page table
        got = sc.f64(k=sc.other_row[0], v=sc.other_row[1])
    elif mistake == "ring_page+1":            # a ring sized as DecoderKv sizes it, read one page (16 slots) on: the
        cap = ((window + 64) // 16 + 1) * 16  # slot holds the latest position of the same residue
        got = sc.f64(keys=np.where(j + 16 <= pos, j + 16, j + 16 - cap))
    elif mistake in ("alpha_acc", "alpha_l", "merge_factor"):
        got = sc.model("fused", mistake)
    elif mistake in ("q8_scale_block", "q8_scale_pos"):
        how = mistake.split("_")[-1]
        got = sc.f64(k=_q8_shifted(sc.kq, sc.kd, how)[0], v=_q8_shifted(sc.vq, sc.vd, how)[0])
    return float(ratio(got, o64, bound).max())


PLANTED = {  # mistake: probes (operand set, G, hd, pos, window)
    "window-1": [("gauss", 4, 128, 300, 40), ("edge_key", 2, 64, 130, 7)],
    "window+1": [("gauss", 4, 128, 300, 40), ("outside_key", 2, 64, 130, 7)],
    "j<pos": [("gauss", 4, 128, 300, 40), ("gauss", 1, 32, 97, 8)],
    "prefill_row0_pos": [("gauss", 4, 128, 300, 40), ("gauss", 2, 64, 130, 31)],
    "rope_row+1": [("gauss", 4, 128, 300, 40), ("gauss", 1, 32, 97, 8)],
    "rope_unwrapped": [("gauss", 4, 128, 5000, 40), ("gauss", 1, 32, 4200, 8)],
    "q_unrotated": [("gauss", 4, 128, 300, 40), ("gauss", 1, 32, 97, 8)],
    "kv_head_h%Hkv": [("gauss", 4, 128, 300, 40), ("gauss", 2, 64, 130, 7)],
    "page_row_b-1": [("gauss", 4, 128, 300, 40), ("gauss", 1, 32, 97, 8)],
    "ring_page+1": [("gauss", 4, 128, 300, 40), ("gauss", 2, 64, 130, 7)],
    "alpha_acc": [("rising", 4, 128, 300, 8192), ("qk_2^+16", 1, 64, 130, 100)],
    "alpha_l": [("rising", 4, 128, 300, 8192), ("qk_2^+16", 1, 64, 130, 100)],
    "merge_factor": [("rising", 4, 128, 300, 8192), ("gauss", 2, 64, 130, 100)],
    "q8_scale_block": [("gauss", 4, 128, 300, 40), ("gauss", 1, 32, 97, 8)],
    "q8_scale_pos": [("gauss", 4, 128, 300, 40), ("gauss", 1, 32, 97, 8)],
}


@pytest.mark.parametrize("mistake", list(PLANTED))
def test_planted_mistake_exceeds_the_bound(mistake):
    worst = max(_planted(mistake, aset, G, hd, pos, w, 7 + pos + w) for aset, G, hd, pos, w in PLANTED[mistake])
    print(f"\n[dec attention planted] {mistake:16s} worst |planted - o64| / bound = {worst:.1f}")
    assert worst >= SEPARATION, (mistake, worst)
