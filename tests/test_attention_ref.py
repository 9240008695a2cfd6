"""CPU side of the encoder attention tests (tests/test_attention_gpu.py runs vox_attention on the same inputs).

The three encoder attention kernels -- K4-TC (enc_attn_tc.cu), K4 (kernels.cu) and K4-S (stream.cu) -- compute, per
(stream, head), o_i = sum_j p_ij v_j with p_i = softmax_j(scale q_i . k_j) over the keys j visible to query i: j <= i and
i - j <= window (K4-S: key position p of a session sits in ring slot p % ring).  This file holds the float64 reference,
its per-output bound, numpy models of each kernel's f32 arithmetic in its own order, and planted mistakes.

The bound (f64_and_bound), per output (i, d), on the f32 inputs:
  * scores: ds_ij = |scale| * (2^-20 sum_d |q_id k_jd| + 2^-32 |q_i|_1 max|k|) + 2^-21 (|s_ij| + |m_i|) + 2^-21.  The
    first term is the f32 dot product over hd (and, for K4-TC, the two f16 pieces and the dropped lo.lo term, 3 x 2^-22
    relative); the second the pieces of keys far below their tile's largest; the rest the scale multiply, the
    subtraction of the running max and a few ulps of expf.  A score error moves o_i by sum_j p_ij ds_ij |v_jd - o_id|
    (the softmax's sensitivity to its scores);
  * sums: (gamma_d + 2^-21) (sum_j p_ij |v_jd| + |o_id|), gamma_d = d u / (1 - d u), u = 2^-24, d = n_i + n_i / 64 + 8
    with n_i the visible keys: the deepest f32 chain of the P V and l sums is K4's sequential fmaf over all keys plus
    one alpha rescale per tile.  2^-21 covers the V and P pieces, 1 / l and the final products;
  * floor: 2^-28 max |v| + 2^-126, the max over floor_keys: pieces of values far below the largest V a kernel scales
    them with.  K4-TC scales V by the largest over the keys some query of its 64-row block can see (block_keys); the
    other kernels need only the row's visible keys, the default.

Checked here: the reference agrees with OracleModel._attention in float64; the three models stay below a quarter of the
bound on every operand set (worst 0.11); thirteen planted mistakes exceed it by >= SEPARATION (10, the window pins'
factor in tests/test_encoder_geometry_ref.py); a two-piece split without powers of two (K4-TC's earlier form) exceeds it
once V is scaled to 2^-8 (80x the bound; 18000x at 2^-16), which enc_attn_tc.cu's powers of two fixed. A diagnostic prints the encoder-geometry model's Q, K and V magnitudes per layer against the 2^-3 edge below
which unscaled pieces lose bits.
"""
import numpy as np
import pytest
import torch

U = 2.0 ** -24
SEPARATION = 10
F32 = np.float32


def visible(qpos, kpos, window):
    qpos, kpos = np.asarray(qpos)[:, None], np.asarray(kpos)[None, :]
    return (kpos <= qpos) & (qpos - kpos <= window)


def block_keys(n, window):
    """[n, n]: the keys some query of query i's 64-row block (K4-TC's CTA) can see"""
    q0 = 64 * (np.arange(n) // 64)[:, None]
    j = np.arange(n)[None, :]
    return (j >= q0 - window) & (j <= q0 + 63)


def f64_and_bound(q, k, v, mask, scale, floor_keys=None):
    """One head: q [n, hd], k and v [m, hd] (f32), mask [n, m] -> (o64, bound), both [n, hd]."""
    q64, k64, v64 = (np.asarray(a, np.float64) for a in (q, k, v))
    s = scale * (q64 @ k64.T)
    s = np.where(mask, s, -np.inf)
    mx = s.max(1, keepdims=True)
    e = np.where(mask, np.exp(s - mx), 0.0)
    p = e / e.sum(1, keepdims=True)
    o = p @ v64
    aq, ak, av = np.abs(q64), np.abs(k64), np.abs(v64)
    ds = abs(scale) * (2.0 ** -20 * (aq @ ak.T) + 2.0 ** -32 * aq.sum(1, keepdims=True) * ak.max(initial=0.0))
    ds = ds + 2.0 ** -21 * (np.abs(np.where(mask, s, 0.0)) + np.abs(mx)) + 2.0 ** -21
    w = p * ds                                               # zero off the mask
    sens = np.empty_like(o)
    for i0 in range(0, len(o), 64):                          # sum_j w_ij |v_jd - o_id|, 64 queries at a time
        sl = slice(i0, i0 + 64)
        sens[sl] = torch.einsum("ij,ijd->id", torch.from_numpy(w[sl]),
                                (torch.from_numpy(v64)[None] - torch.from_numpy(o[sl])[:, None]).abs()).numpy()
    n = mask.sum(1, keepdims=True).astype(np.float64)
    d = n + n // 64 + 8
    gam = d * U / (1 - d * U) + 2.0 ** -21
    vmax = np.where((mask if floor_keys is None else floor_keys)[:, :, None], av[None], 0.0).max((1, 2))[:, None]
    return o, sens + gam * (p @ av + np.abs(o)) + 2.0 ** -28 * vmax + 2.0 ** -126


def ratio(got, o64, bound):
    """|got - o64| / bound, inf where got is not finite"""
    got = np.asarray(got, np.float64)
    with np.errstate(invalid="ignore"):
        return np.where(np.isfinite(got), np.abs(got - o64) / bound, np.inf)


# ------------------------------------------------------------------------------------------------ layouts and cases


def enc_heads(qkv, h, hd, q_off, k_off, v_off):
    """[rows, ld] -> q, k, v [rows, h, hd]"""
    return tuple(qkv[:, off:off + h * hd].reshape(-1, h, hd) for off in (q_off, k_off, v_off))


def encoder_ref(qkv, h, hd, q_off, k_off, v_off, starts, lens, window, scale):
    """f64 reference and bound of the encoder kernels: streams of rows [starts[t], starts[t] + lens[t])."""
    q, k, v = enc_heads(qkv, h, hd, q_off, k_off, v_off)
    o = np.zeros((q.shape[0], h * hd))
    b = np.zeros_like(o)
    for r0, n in zip(starts, lens):
        mask, fk = visible(np.arange(n), np.arange(n), window), block_keys(n, window)
        for hh in range(h):
            sl = slice(r0, r0 + n)
            oo, bb = f64_and_bound(q[sl, hh], k[sl, hh], v[sl, hh], mask, scale, fk)
            o[sl, hh * hd:(hh + 1) * hd], b[sl, hh * hd:(hh + 1) * hd] = oo, bb
    return o, b


def ring_keys(k_ring, slot, pos, window, ring, shift=0):
    """key positions and the ring rows of a K4-S query row: positions max(0, pos - window) .. pos at (p + shift) % ring"""
    kp = np.arange(max(0, pos - window), pos + 1)
    return kp, k_ring[slot, (kp + shift) % ring]


def ring_ref(qkv, h, hd, row_slot, row_pos, k_ring, v_ring, window, scale, shift=0):
    ring = k_ring.shape[1]
    o = np.zeros((qkv.shape[0], h * hd))
    b = np.zeros_like(o)
    for r, (slot, pos) in enumerate(zip(row_slot, row_pos)):
        kp, kr = ring_keys(k_ring, slot, pos, window, ring, shift)
        _, vr = ring_keys(v_ring, slot, pos, window, ring, shift)
        for hh in range(h):
            c = slice(hh * hd, (hh + 1) * hd)
            oo, bb = f64_and_bound(qkv[r:r + 1, c], kr[:, c], vr[:, c], np.ones((1, len(kp)), bool), scale)
            o[r, c], b[r, c] = oo[0], bb[0]
    return o, b


OPERAND_SETS = ("gauss", "qk_2^-16", "qk_2^-8", "qk_2^+8", "v_2^-16", "v_2^-8", "v_2^+8", "one_hot", "uniform",
                "edge_key", "outside_key", "v_offset", "hidden_v",
                "v_tile_range")


def operands(aset, n, h, hd, seed, window=64):
    """q, k, v [n, h, hd] f32 for one operand set (positions 0..n-1 of one stream)."""
    rng = np.random.default_rng(seed)
    q, k, v = (rng.standard_normal((n, h, hd)) for _ in range(3))
    if aset.startswith("qk_"):
        f = 2.0 ** float(aset.split("^")[1])
        q, k = q * f, k * f
    elif aset.startswith("v_2"):
        v = v * 2.0 ** float(aset.split("^")[1])
    elif aset == "one_hot":                        # each query's own key wins by a score gap of 120 over the one before
        q[:, :, 0] = 40.0 * np.sqrt(hd)
        k[:, :, 0] = 3.0 * np.arange(n)[:, None]
    elif aset == "uniform":                        # all keys identical: a uniform softmax
        k[:] = k[:1]
    elif aset in ("edge_key", "outside_key"):      # a dominant key at i - window (or one before it) of the last query
        at = max(0, n - 1 - window - (aset == "outside_key"))
        k[at] = 6.0 * q[n - 1] / np.sqrt(hd)
    elif aset == "v_offset":                       # |v - o| << |v|
        v = 1000.0 + 0.01 * v
    elif aset == "hidden_v":                       # V of 2^60 at the key just before the first one the 64-row block
        q0 = 64 * ((window + 64) // 64)            # q0 can see (q0 - window, in 1 .. 64): for window % 64 != 0 it
        at = q0 - window - 1                       # sits in the first tile that block loads
        if 0 <= at < n:
            v[at] *= 2.0 ** 60
    elif aset == "v_tile_range":                   # V of every other 64-key tile 2^-100 times smaller
        v[(np.arange(n) // 64) % 2 == 1] *= 2.0 ** -100
    return q.astype(F32), k.astype(F32), v.astype(F32)


# ------------------------------------------------------------------------------------------------ f32 models


def f32(x):
    return np.asarray(x, np.float64).astype(F32)


def fma(a, b, c):
    return f32(np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64))


def expf(x):
    with np.errstate(invalid="ignore"):
        return f32(np.exp(np.asarray(x, np.float64)))


def model_simt(q, k, v, window, scale, mistake=None):
    """K4 (enc_attention_kernel): 32-query blocks, 64-key tiles, lane c of a query row takes keys c, c+4, ..; fmaf dot
    products, online softmax with the alpha rescale, sequential fmaf P V.  One stream, one head: q, k, v [S, hd]."""
    S, hd = q.shape
    out = np.zeros((S, hd), F32)
    scale = F32(scale)
    for q0 in range(0, S, 32):
        rows = np.arange(q0, min(q0 + 32, S))
        qb = q[rows]
        m = np.full(len(rows), -np.inf, F32)
        l = np.zeros(len(rows), F32)
        o = np.zeros((len(rows), hd), F32)
        j_begin = max(q0 - window, 0) // 64 * 64 + (64 if mistake == "j_begin" else 0)
        for j0 in range(j_begin, min(q0 + 31, S - 1) + 1, 64):
            keys = np.arange(j0, j0 + 64)
            kt = np.where((keys < S)[:, None], k[np.minimum(keys, S - 1)], 0).astype(F32)
            vt = np.where((keys < S)[:, None], v[np.minimum(keys, S - 1)], 0).astype(F32)
            acc = np.zeros((len(rows), 64), F32)
            for d in range(hd):
                acc = fma(qb[:, d:d + 1], kt[None, :, d], acc)
            valid = (keys[None] < S) & visible(rows, keys, window)
            s = np.where(valid, f32(acc * scale), F32(-np.inf))
            m_new = np.maximum(m, s.max(1))
            dead = m_new == -np.inf
            alpha = np.where(dead, F32(1), expf(m - np.where(dead, 0, m_new)))
            p = np.where(dead[:, None], F32(0), expf(s - np.where(dead, 0, m_new)[:, None]))
            part = np.zeros((len(rows), 4), F32)
            for jj in range(16):
                part = f32(part + p[:, jj * 4:jj * 4 + 4])
            psum = f32(f32(part[:, 0] + part[:, 1]) + f32(part[:, 2] + part[:, 3]))
            l = fma(l, F32(1) if mistake == "alpha_l" else alpha, psum)
            m = m_new
            if mistake != "alpha_o":
                o = f32(o * alpha[:, None])
            for kk in range(64):
                o = fma(p[:, kk:kk + 1], vt[kk][None], o)
        with np.errstate(divide="ignore", invalid="ignore"):    # a planted j_begin can leave a row no key
            out[rows] = f32(o * f32(F32(1) / l)[:, None])
    return out


def _tree32(x):
    """the xor butterfly of a warp sum (__shfl_xor 16, 8, 4, 2, 1): lane 0's value; x [..., 32]"""
    for off in (16, 8, 4, 2, 1):
        x = f32(x + x[..., np.arange(32) ^ off])
    return x[..., 0]


def model_stream(q, kp, kr, vr, scale):
    """K4-S (stream_enc_attn_kernel) for one (row, head): keys kp (ascending positions), rows kr / vr [n, hd]; key t
    of the window goes to warp t % 4; a warp's dot product is per-lane fmaf over hd / 32 dims and a butterfly; the four
    warps' (m, l, acc) merge through -inf-guarded factors."""
    hd = q.shape[0]
    dpl = hd // 32
    scale = F32(scale)
    ms, ls, accs = [], [], []
    for w in range(4):
        m, l, acc = F32(-np.inf), F32(0), np.zeros(hd, F32)
        for t in range(w, len(kp), 4):
            part = np.zeros(32, F32)
            for i in range(dpl):
                part = fma(q[i::dpl], kr[t, i::dpl], part)
            s = f32(_tree32(part) * scale)
            m_new = max(m, s)
            alpha, p = expf(m - m_new), expf(s - m_new)
            l = fma(l, alpha, p)
            m = m_new
            acc = fma(p, vr[t], f32(acc * alpha))
        ms.append(m), ls.append(l), accs.append(acc)
    mx = max(ms)
    num, den = np.zeros(hd, F32), F32(0)
    for w in range(4):
        f = F32(0) if ms[w] == -np.inf else expf(ms[w] - mx)
        num, den = fma(accs[w], f, num), fma(ls[w], f, den)
    return f32(num / den)


def f16(x):
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def split2(x, lose_lo=False):
    hi = f16(x)
    with np.errstate(invalid="ignore"):
        lo = np.zeros_like(hi) if lose_lo else f16(f32(np.asarray(x, np.float64) - hi))
    return hi, lo


def split_exp(mx, keep=0):
    """enc_attn_tc.cu split_exp: 2^e brings mx into [2^14, 2^15)"""
    if not (mx > 0) or not np.isfinite(mx):
        return keep
    return int(min(max(14 - int(np.floor(np.log2(np.float64(mx)))), -126), 126))


def _mma3(c, ah, al, bh, bl):
    """c += A B over k-steps of 16 as three MMAs each (hi.hi, hi.lo, lo.hi): each MMA's 16 products summed exactly, then
    added to the f32 accumulator with one rounding.  a [rows, K], b [K, cols]"""
    for k0 in range(0, ah.shape[1], 16):
        ks = slice(k0, k0 + 16)
        for a, b in ((ah, bh), (ah, bl), (al, bh)):
            c = f32(c + a[:, ks] @ b[ks])
    return c


def model_tc(q, k, v, window, scale, scaled=True, lose=(), all_keys=False):
    """K4-TC (enc_attention_tc_kernel) for one stream and head: 64-query blocks, 64-key tiles, two-piece f16 operands and
    three MMAs per product.  scaled: the powers of two of enc_attn_tc.cu (Q per row, K per key tile, V by the running
    tile maximum, P * 2^15; keys no query of the block sees load as zeros);
    False is the plain split K4-TC had before.  lose: operands ("q", "k", "v", "p") whose lo piece is dropped.  all_keys: the
    scaled split over every key of a tile, masked ones included (a planted mistake)."""
    S, hd = q.shape
    out = np.zeros((S, hd), F32)
    scale = F32(scale)
    ps = 2.0 ** 15 if scaled else 1.0
    for q0 in range(0, S, 64):
        rows = np.arange(q0, q0 + 64)
        qb = np.where((rows < S)[:, None], q[np.minimum(rows, S - 1)], 0).astype(F32)
        eq = np.array([split_exp(np.abs(r).max()) if scaled else 0 for r in qb])
        qh, ql = split2(f32(qb * 2.0 ** eq[:, None]), "q" in lose)
        sc = f32(scale * 2.0 ** -eq.astype(np.float64))
        m = np.full(64, -np.inf, F32)
        l4 = np.zeros((64, 4), F32)                    # quad-partial sums: lane t holds keys 8n + 2t + {0, 1}
        o = np.zeros((64, hd), F32)
        ev_run = 126 if scaled else 0
        q_last = min(q0 + 63, S - 1)
        j_begin = max(q0 - window, 0) // 64 * 64
        for j0 in range(j_begin, q_last + 1, 64):
            keys = np.arange(j0, j0 + 64)
            # the scaled kernel loads only keys some query of the block can see, the plain split every key below S
            load = (keys >= q0 - window) & (keys <= q_last) if scaled and not all_keys else keys < S
            kt = np.where(load[:, None], k[np.minimum(keys, S - 1)], 0).astype(F32)
            vt = np.where(load[:, None], v[np.minimum(keys, S - 1)], 0).astype(F32)
            ek = split_exp(np.abs(kt).max()) if scaled else 0
            ev = min(ev_run, split_exp(np.abs(vt).max(), ev_run)) if scaled else 0
            kh, kl = split2(f32(kt * 2.0 ** ek), "k" in lose)
            vh, vl = split2(f32(vt * 2.0 ** ev), "v" in lose)
            s = _mma3(np.zeros((64, 64), F32), qh, ql, kh.T, kl.T)
            valid = (keys[None] < S) & visible(rows, keys, window)
            s = np.where(valid, f32(s * f32(sc * 2.0 ** -ek)[:, None]), F32(-np.inf))
            m_new = np.maximum(m, s.max(1))
            dead = m_new == -np.inf
            alpha = np.where(dead, F32(1), expf(m - np.where(dead, 0, m_new)))
            p = np.where(dead[:, None], F32(0), expf(s - np.where(dead, 0, m_new)[:, None]))
            psum = np.zeros((64, 4), F32)
            for n in range(8):
                for e in range(2):
                    psum = f32(psum + p[:, 8 * n + 2 * np.arange(4) + e])
            l4 = fma(l4, alpha[:, None], psum)
            m = m_new
            ph, pl = split2(f32(p * ps), "p" in lose)
            o = f32(o * f32(alpha * 2.0 ** (ev - ev_run))[:, None])
            ev_run = ev
            o = _mma3(o, ph, pl, vh, vl)
        l = f32(f32(l4[:, 0] + l4[:, 1]) + f32(l4[:, 2] + l4[:, 3]))
        res = f32(f32(o * f32(F32(1) / l)[:, None]) * (2.0 ** -(ev_run + (15 if scaled else 0))))
        keep = rows < S
        out[rows[keep]] = res[keep]
    return out


# ------------------------------------------------------------------------------------------------ checks


def _one_head(aset, S, hd, window, seed):
    q, k, v = operands(aset, S, 1, hd, seed, window)
    return q[:, 0], k[:, 0], v[:, 0]


SCALE = {32: float(F32(32) ** F32(-0.5)), 64: float(F32(64) ** F32(-0.5))}
PROBES = [(130, 32, 8), (130, 64, 1), (200, 64, 70), (200, 32, 1000)]     # (S, hd, window)


def test_reference_matches_oracle_attention():
    from oracle.model import OracleModel
    S, h, hd, window = 150, 3, 32, 40
    q, k, v = operands("gauss", S, h, hd, 1, window)
    got = OracleModel._attention(None, *(torch.from_numpy(a.astype(np.float64)) for a in (q, k, v)), SCALE[hd], 0,
                                 window).numpy()
    qkv = np.concatenate([a.reshape(S, h * hd) for a in (q, k, v)], 1)
    o, b = encoder_ref(qkv, h, hd, 0, h * hd, 2 * h * hd, [0], [S], window, SCALE[hd])
    assert np.abs(got - o).max() <= 1e-12 * np.abs(o).max()
    assert np.all(b > 0) and np.all(b < 1e-5 * np.abs(v).max())


@pytest.mark.parametrize("aset", OPERAND_SETS)
def test_models_within_a_quarter_of_the_bound(aset):
    worst = {}
    for S, hd, window in PROBES:
        q, k, v = _one_head(aset, S, hd, window, S + hd + window)
        o64, bound = f64_and_bound(q, k, v, visible(np.arange(S), np.arange(S), window), SCALE[hd], block_keys(S, window))
        for name, fn in (("K4-TC", model_tc), ("K4", model_simt)):
            worst[name] = max(worst.get(name, 0.0), float(ratio(fn(q, k, v, window, SCALE[hd]), o64, bound).max()))
        # K4-S over the same keys: the last 8 rows
        r = []
        for i in range(S - 8, S):
            kp = np.arange(max(0, i - window), i + 1)
            r.append(ratio(model_stream(q[i], kp, k[kp], v[kp], SCALE[hd]), o64[i], bound[i]).max())
        worst["K4-S"] = max(worst.get("K4-S", 0.0), float(max(r)))
    for name, w in worst.items():
        print(f"\n[attention models] {aset:12s} {name:6s} worst |model - o64| / bound = {w:.3f}")
        assert w < 0.25, (aset, name, w)


def _planted(mistake, S, hd, window, aset, seed):
    q, k, v = _one_head(aset, S, hd, window, seed)
    pos = np.arange(S)
    o64, bound = f64_and_bound(q, k, v, visible(pos, pos, window), SCALE[hd], block_keys(S, window))
    if mistake.startswith("lo_"):
        got = model_tc(q, k, v, window, SCALE[hd], lose=(mistake[3:],))
    elif mistake == "tile_max_all_keys":               # K4-TC's V power of two over keys no query of the block sees
        got = model_tc(q, k, v, window, SCALE[hd], all_keys=True)
    elif mistake in ("j_begin", "alpha_o", "alpha_l"):
        got = model_simt(q, k, v, window, SCALE[hd], mistake)
    elif mistake in ("window-1", "window+1"):
        got = f64_and_bound(q, k, v, visible(pos, pos, window + int(mistake[6:])), SCALE[hd])[0]
    elif mistake == "j<i":
        with np.errstate(invalid="ignore"):
            got = f64_and_bound(q, k, v, visible(pos, pos, window) & (pos[None] < pos[:, None]), SCALE[hd])[0][1:]
        o64, bound = o64[1:], bound[1:]                   # row 0 sees no key at all
    elif mistake == "prev_stream_key":                    # key -1: the previous stream's last row
        k2 = np.concatenate([f32(np.random.default_rng(seed).standard_normal((1, hd))), k])
        v2 = np.concatenate([f32(np.random.default_rng(seed + 1).standard_normal((1, hd))), v])
        got = f64_and_bound(q, k2, v2, visible(pos, np.arange(-1, S), window), SCALE[hd])[0]
    elif mistake == "ring_slot+1":
        ring = window + 256
        rng = np.random.default_rng(seed)
        kr, vr = f32(rng.standard_normal((1, ring, hd))), f32(rng.standard_normal((1, ring, hd)))
        slot, p = np.zeros(8, int), np.arange(ring - 4, ring + 4) + 3 * ring
        o64, bound = ring_ref(q[:8], 1, hd, slot, p, kr, vr, window, SCALE[hd])
        got = ring_ref(q[:8], 1, hd, slot, p, kr, vr, window, SCALE[hd], shift=1)[0]
    return float(ratio(got, o64, bound).max())


PLANTED = {  # mistake: probes (S, hd, window, operand set)
    "lo_q": [(130, 64, 1, "gauss"), (130, 32, 8, "gauss")],
    "lo_k": [(130, 64, 1, "gauss"), (130, 32, 8, "gauss")],
    "lo_v": [(130, 64, 1, "gauss"), (130, 32, 1, "gauss")],
    "lo_p": [(130, 64, 1, "gauss"), (130, 32, 2, "gauss")],
    "window-1": [(130, 64, 8, "gauss")],
    "window+1": [(130, 64, 8, "gauss")],
    "j<i": [(130, 64, 8, "gauss")],
    "j_begin": [(200, 64, 70, "gauss")],
    "alpha_o": [(200, 64, 1000, "qk_2^+8")],
    "alpha_l": [(200, 64, 1000, "qk_2^+8")],
    "prev_stream_key": [(130, 64, 8, "gauss")],
    "ring_slot+1": [(130, 64, 3, "gauss"), (130, 64, 750, "gauss")],
    "tile_max_all_keys": [(200, 64, 63, "hidden_v"), (200, 32, 8, "hidden_v")],
}


@pytest.mark.parametrize("mistake", list(PLANTED))
def test_planted_mistake_exceeds_the_bound(mistake):
    worst = max(_planted(mistake, S, hd, w, aset, 7 + S + w) for S, hd, w, aset in PLANTED[mistake])
    print(f"\n[attention planted] {mistake:16s} worst |planted - o64| / bound = {worst:.1f}")
    assert worst >= SEPARATION, (mistake, worst)


@pytest.mark.parametrize("aset", ["v_2^-8", "v_2^-16"])
def test_unscaled_split_exceeds_the_bound_at_small_scales(aset):
    """The two-piece split without powers of two (K4-TC before they were added) loses bits once lo leaves f16's normal
    range; the scaled split (model_tc) holds the bound on the same operands (test_models_within_a_quarter_of_the_bound)."""
    S, hd, window = 130, 64, 130
    q, k, v = _one_head(aset, S, hd, window, 3)
    o64, bound = f64_and_bound(q, k, v, visible(np.arange(S), np.arange(S), window), SCALE[hd], block_keys(S, window))
    w = float(ratio(model_tc(q, k, v, window, SCALE[hd], scaled=False), o64, bound).max())
    print(f"\n[attention unscaled split] {aset:9s} worst |model - o64| / bound = {w:.1f}")
    assert w > 1.0


def test_encoder_geometry_operand_magnitudes():
    """Diagnostic: per layer of the encoder-geometry model (f64 oracle, 12 s of speech-like audio), the RMS and max |.|
    of Q, K (after RoPE) and V over heads, against the 2^-3 edge below which an unscaled lo piece is subnormal."""
    from oracle.model import OracleModel, apply_rope, rms_norm
    from test_encoder_geometry_ref import encoder_geometry_bytes, geometry_mel
    o = OracleModel(encoder_geometry_bytes(750), dtype=torch.float64)
    c = o.cfg
    x = o.conv_stem(geometry_mel(12.0, 3))
    pre = "mm_streams_embeddings.embedding_module.whisper_encoder"
    for i in range(c.enc_layers):
        p = f"{pre}.transformer.layers.{i}"
        h = rms_norm(x, o.param(f"{p}.attention_norm.weight"), c.norm_eps)
        s = h.shape[0]
        q = apply_rope(o.linear(h, f"{p}.attention.wq.weight", f"{p}.attention.wq.bias").reshape(s, c.enc_heads, -1),
                       o.enc_cos, o.enc_sin, 0)
        k = apply_rope(o.linear(h, f"{p}.attention.wk.weight").reshape(s, c.enc_heads, -1), o.enc_cos, o.enc_sin, 0)
        v = o.linear(h, f"{p}.attention.wv.weight", f"{p}.attention.wv.bias").reshape(s, c.enc_heads, -1)
        line = []
        for name, t in (("q", q), ("k", k), ("v", v)):
            rms = t.pow(2).mean((0, 2)).sqrt()
            line.append(f"{name} rms {float(rms.min()):.2e}..{float(rms.max()):.2e} max {float(t.abs().max()):.2e}")
        print(f"\n[encoder geometry operands] layer {i}: " + "; ".join(line) + f" (edge 2^-3 = {2.0 ** -3:.3f})")
        x = o.encoder_layer(x, i)
