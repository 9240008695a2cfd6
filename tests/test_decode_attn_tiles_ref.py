"""CPU pins of the persistent decode kernel's attention schedule (decode_mega.cu, the MG_ATTN phase) for
tests/test_decode_attn_tiles_gpu.py.

The kernel splits the keys [j_lo, pos] of one (stream, kv head), j_lo = max(0, pos - window), into NC key chunks of
per = ceil((pos - j_lo + 1) / NC) keys (the last ones may be short or empty).  A CTA walks its chunk in tiles of KT keys
with an online softmax: a running max per head, and the unnormalised P.V (o_acc) and sum of P (o_sum) rescaled by
alpha = exp(m_old - m_new) at every tile.  P.V takes two keys per iteration plus a one-key tail.  The last chunk's CTA
merges the chunks: its own state first, then chunks 0 .. NC-2 in ascending order, an empty chunk being m = -inf.
KT and NC depend on the rows of the launch (TILING, for the decoder geometry on a 132-SM H100).

  * chunked_attention is that schedule in float64.  It equals plain softmax attention to ~1e-12 at every position
    0..1100, windows 8, 383, 400 and 8192, and every (KT, NC) of TILING.  The sweep meets empty last chunks, one-key
    tails, full final tiles and chunks of 3 or more tiles.
  * Sensitivity: each of these kernel mistakes, applied in both layers to 16 consecutive rows of the decoder-geometry
    model, moves the f64 logits of some row by more than 20x LOGIT_REL_BOUND, the GPU test's bound, at every
    (rows, window, positions) probe where the mistake changes the computation at all:
      1. no_rescale       -- alpha = 1: the earlier tiles are never rescaled;
      2. sum_not_rescaled -- o_acc is rescaled but o_sum is not;
      3. odd_tail         -- the P.V tail is lost: the last key of every odd-length tile is dropped;
      4. stale_v          -- tile t+1's probabilities are applied to tile t's V rows;
      5. ring_lap         -- (KV ring of RING_POSITIONS positions) when a tile straddles the ring wrap, the keys past
                             the wrap are read from the previous lap (key j taken from j - RING_POSITIONS).
    A mistake that changes nothing at a probe is not caught there, and cannot be: mistakes 1, 2 and 4 need a chunk of
    two or more tiles, 3 an odd-length tile and 5 a tile across the wrap.  At window 383 with 3 or 4 rows (KT 96, NC 4)
    a chunk holds at most 96 keys, one tile, so mistakes 1, 2 and 4 cannot occur there at any position (the GPU test
    meets them at 3 and 4 rows at the other windows); once the window bites every chunk is one full tile, which the
    GPU test checks against the reference.  The test prints, per probe, each mistake's largest effect.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes

# rows in one persistent launch -> (keys per tile KT, key chunks per (stream, kv head) NC); 11 rows run as 8 + 3
TILING = {1: (32, 4), 2: (64, 4), 3: (96, 4), 4: (96, 4), 5: (96, 3), 8: (96, 2)}
SWEEP_WINDOWS = (8, 383, 400, 8192)
RING_POSITIONS = 480           # KV ring of the window-400 decoder: (400 + 64) / 16 + 1 = 30 pages of 16 positions
MISTAKES = ("no_rescale", "sum_not_rescaled", "odd_tail", "stale_v")
PROBE_ROWS = 16
# decode positions the GPU test reaches at every window (S4 = 984 for its 150 s streams), 16 rows from each start
PROBES = {8192: (360, 900), 383: (360, 900), 400: (360, 600, 900)}
RING_PROBE = (400, 600)        # keys [200.., 600..] hold the ring wrap at 480


def chunk_bounds(pos, window, NC):
    """[(j0, j1)] of the NC key chunks of position pos (j1 <= j0 for an empty chunk)."""
    j_lo = max(0, pos - window)
    per = (pos - j_lo + NC) // NC
    return [(j_lo + ch * per, min(pos + 1, j_lo + ch * per + per)) for ch in range(NC)]


def chunk_tiles(pos, window, NC, KT):
    """Per chunk, the lengths of its tiles in walk order."""
    return [[min(KT, j1 - jt) for jt in range(j0, j1, KT)] for j0, j1 in chunk_bounds(pos, window, NC)]


def mistake_applies(mistake, tiles, pos=None, window=None, NC=None, KT=None, ring=RING_POSITIONS):
    """Whether the mistake changes the schedule of a position with these chunk tiles."""
    if mistake in ("no_rescale", "sum_not_rescaled", "stale_v"):
        return any(len(t) > 1 for t in tiles)
    if mistake == "odd_tail":
        return any(n % 2 for t in tiles for n in t)
    assert mistake == "ring_lap"
    return any(_wrap_in_tile(jt, min(KT, j1 - jt), ring) is not None
               for j0, j1 in chunk_bounds(pos, window, NC) for jt in range(j0, j1, KT))


def _wrap_in_tile(jt, n, ring):
    """Index in the tile [jt, jt + n) of its first key at a ring wrap (key % ring == 0), if not the tile's first key."""
    w = -jt % ring
    return w if 0 < w < n else None


def chunked_attention(q, k, v, scale, pos, window, NC, KT, mistake=None, ring=RING_POSITIONS):
    """The kernel's schedule in float64 for one query position: q [H, hd], k / v [>= pos + 1, Hkv, hd] (key j in row j)
    -> [H, hd].  `mistake`: one of MISTAKES or "ring_lap" (module docstring)."""
    H, hd = q.shape
    Hkv = k.shape[1]
    qg = np.asarray(q, np.float64).reshape(Hkv, H // Hkv, hd)
    k, v = np.asarray(k, np.float64), np.asarray(v, np.float64)
    states = []
    for j0, j1 in chunk_bounds(pos, window, NC):
        m = np.full(qg.shape[:2], -np.inf)
        o_acc = np.zeros(qg.shape)
        o_sum = np.zeros(qg.shape[:2])
        v_prev = None
        for jt in range(j0, j1, KT):
            n = min(KT, j1 - jt)
            keys = np.arange(jt, jt + n)
            w = _wrap_in_tile(jt, n, ring) if mistake == "ring_lap" else None
            if w is not None:
                keys[w:] -= ring
            kt, vt = k[keys], v[keys]                                  # [n, Hkv, hd]
            s = np.einsum("hgd,nhd->hgn", qg, kt) * scale
            m_new = np.maximum(m, s.max(-1))
            p = np.exp(s - m_new[..., None])
            alpha = np.exp(m - m_new)                                  # 0 on the first tile
            v_used = v_prev[:n] if mistake == "stale_v" and v_prev is not None else vt
            if mistake == "odd_tail" and n % 2:
                p, v_used = p[..., :n - 1], v_used[:n - 1]
            a_acc = np.ones_like(alpha) if mistake == "no_rescale" else alpha
            a_sum = np.ones_like(alpha) if mistake in ("no_rescale", "sum_not_rescaled") else alpha
            o_acc = o_acc * a_acc[..., None] + np.einsum("hgn,nhd->hgd", p, v_used)
            o_sum = o_sum * a_sum + p.sum(-1)
            m, v_prev = m_new, vt
        states.append((m, o_acc, o_sum))
    m_all, num, den = states[-1]
    for mc, ac, sc in states[:-1]:
        m_new = np.maximum(m_all, mc)
        with np.errstate(invalid="ignore"):
            fo = np.where(m_all == -np.inf, 0.0, np.exp(m_all - m_new))
            fc = np.where(mc == -np.inf, 0.0, np.exp(mc - m_new))
        num, den, m_all = num * fo[..., None] + ac * fc[..., None], den * fo + sc * fc, m_new
    return (num / den[..., None]).reshape(H, hd)


def plain_attention(q, k, v, scale, pos, window):
    H, hd = q.shape
    Hkv = k.shape[1]
    j_lo = max(0, pos - window)
    kk = np.repeat(np.asarray(k[j_lo:pos + 1], np.float64), H // Hkv, axis=1)   # [n, H, hd]
    vv = np.repeat(np.asarray(v[j_lo:pos + 1], np.float64), H // Hkv, axis=1)
    s = np.einsum("hd,nhd->hn", np.asarray(q, np.float64), kk) * scale
    p = np.exp(s - s.max(-1, keepdims=True))
    return np.einsum("hn,nhd->hd", p / p.sum(-1, keepdims=True), vv)


def test_chunked_schedule_equals_softmax_attention():
    """Positions 0..1100, windows 8, 383, 400, 8192, every (KT, NC) of TILING: the f64 schedule == plain attention."""
    rng = np.random.default_rng(0)
    H, Hkv, hd, P = 8, 2, 16, 1101
    k = rng.standard_normal((P, Hkv, hd))
    v = rng.standard_normal((P, Hkv, hd))
    qs = rng.standard_normal((P, H, hd)) * 2.0        # scores of spread ~ 8 at scale 1/sqrt(hd)
    scale = hd ** -0.5
    worst = 0.0
    seen = {"empty chunk": 0, "one-key tail": 0, "full final tile": 0, "3+ tiles": 0}
    for KT, NC in sorted(set(TILING.values())):
        for window in SWEEP_WINDOWS:
            for pos in range(P):
                tiles = chunk_tiles(pos, window, NC, KT)
                seen["empty chunk"] += any(not t for t in tiles)
                seen["one-key tail"] += any(len(t) > 1 and t[-1] == 1 for t in tiles)
                seen["full final tile"] += any(len(t) > 1 and t[-1] == KT for t in tiles)
                seen["3+ tiles"] += any(len(t) >= 3 for t in tiles)
                assert sum(map(sum, tiles)) == pos - max(0, pos - window) + 1
                got = chunked_attention(qs[pos], k, v, scale, pos, window, NC, KT)
                worst = max(worst, float(np.abs(got - plain_attention(qs[pos], k, v, scale, pos, window)).max()))
    print(f"\n[attention schedule] f64 emulation vs plain softmax attention: max |d| = {worst:.1e}; positions with "
          + ", ".join(f"{what}: {n}" for what, n in seen.items()))
    assert worst < 1e-12
    assert all(seen.values()), seen


def test_mistakes_change_the_emulation_only_where_they_apply():
    """Each mistake leaves the f64 schedule bit-identical where mistake_applies() says it does not apply (synthetic q,
    k, v), and moves it at some positions where it does.  (Where it applies it need not move the result: dropping alpha
    changes nothing while no later tile raises a head's running max.)"""
    rng = np.random.default_rng(1)
    H, Hkv, hd, P = 8, 2, 16, 1000
    k, v = rng.standard_normal((P, Hkv, hd)), rng.standard_normal((P, Hkv, hd))
    scale = hd ** -0.5
    moved = dict.fromkeys(MISTAKES + ("ring_lap",), 0)
    for KT, NC in sorted(set(TILING.values())):
        for window in (383, 400, 8192):
            for pos in (40, 100, 382, 383, 500, 611, 997):
                q = rng.standard_normal((H, hd)) * 2.0
                ok = chunked_attention(q, k, v, scale, pos, window, NC, KT)
                for mistake in moved:
                    d = np.abs(chunked_attention(q, k, v, scale, pos, window, NC, KT, mistake) - ok).max()
                    if not mistake_applies(mistake, chunk_tiles(pos, window, NC, KT), pos, window, NC, KT):
                        assert d == 0, (mistake, KT, NC, window, pos, d)
                    moved[mistake] += d > 1e-6
    assert all(moved.values()), moved


# ---------------------------------------------------------------------------------------------------------------------
# Sensitivity on the decoder-geometry model

@pytest.fixture(scope="module")
def geometry_oracle():
    """f64 oracle of the decoder-geometry model (the same weights at every window), the f32 oracle's audio embeddings of
    a 150 s utterance (984 positions, as the GPU test) and random teacher tokens."""
    data = geometry_model_bytes(8192)
    o64 = OracleModel(data, dtype=torch.float64)
    mel = omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(150.0, 4321)))
    emb = OracleModel(data).encode_audio(mel)
    ids = np.random.default_rng(2).integers(0, o64.cfg.vocab, emb.shape[0])
    ids[:PREFIX_LEN] = [1] + [32] * (PREFIX_LEN - 1)
    x = torch.as_tensor(emb).to(torch.float64) + o64.embed_tokens(ids.tolist())
    return o64, x, o64.ada_scales(omel.time_embedding(6.0, o64.cfg.dec_dim))


def _rows_with(monkeypatch, o64, x, ada, cache, p0, NC=None, KT=None, mistake=None):
    """Logits of rows [p0, p0 + PROBE_ROWS) on a copy of the cache of rows [0, p0); with NC given, every layer's
    attention of those rows runs chunked_attention(NC, KT, mistake)."""
    def attention(self, q, k, v, scale, q_offset, window, causal=True):
        out = [chunked_attention(q[i].numpy(), k.numpy(), v.numpy(), scale, q_offset + i, window, NC, KT, mistake)
               for i in range(q.shape[0])]
        return torch.from_numpy(np.stack(out)).reshape(q.shape[0], -1)
    with monkeypatch.context() as mp:
        if NC is not None:
            mp.setattr(OracleModel, "_attention", attention)
        h = o64.decoder_forward_with_cache(x[p0:p0 + PROBE_ROWS], ada, [dict(c) for c in cache])
    return o64.lm_head(h).numpy()


@pytest.mark.parametrize("window", sorted(PROBES))
def test_attention_mistakes_exceed_logit_bound(geometry_oracle, monkeypatch, window):
    o64, x, ada = geometry_oracle
    saved = o64.cfg.dec_window
    o64.cfg.dec_window = window
    try:
        cache, done = o64.new_cache(), 0
        rows_out = []
        for p0 in PROBES[window]:
            o64.decoder_forward_with_cache(x[done:p0], ada, cache)
            done = p0
            ref = _rows_with(monkeypatch, o64, x, ada, cache, p0)
            bound = LOGIT_REL_BOUND * np.maximum(1.0, np.abs(ref).max(-1))
            exact = _rows_with(monkeypatch, o64, x, ada, cache, p0, NC=4, KT=32)
            assert (np.abs(exact - ref).max(-1) / bound).max() < 1e-3   # the emulation itself is the reference
            cases = [(B, m) for B in (1, 2, 3, 5, 8) for m in MISTAKES]
            if (window, p0) == RING_PROBE:
                cases += [(B, "ring_lap") for B in (1, 3, 8)]
            for B, mistake in cases:
                KT, NC = TILING[B]
                applies = [mistake_applies(mistake, chunk_tiles(p, window, NC, KT), p, window, NC, KT)
                           for p in range(p0, p0 + PROBE_ROWS)]
                if not any(applies):
                    rows_out.append((p0, B, mistake, None))
                    continue
                got = _rows_with(monkeypatch, o64, x, ada, cache, p0, NC, KT, mistake)
                ratio = np.abs(got - ref).max(-1) / bound
                rows_out.append((p0, B, mistake, ratio.max()))
                assert ratio.max() > 20, (window, p0, B, mistake, ratio.max())
    finally:
        o64.cfg.dec_window = saved
    print(f"\n[attention mistakes] window {window}: largest logit change in 16 rows, as a multiple of the GPU bound "
          "('-': the mistake does not occur there)")
    for p0, B, mistake, r in rows_out:
        print(f"  positions {p0}..{p0 + PROBE_ROWS - 1} B={B} (KT {TILING[B][0]}, NC {TILING[B][1]}) {mistake:>16s}: "
              + ("-" if r is None else f"{r:.0f}x"))
    # every mistake occurs, and is caught, at every tiling somewhere on this window's probes, except where the module
    # docstring says it cannot occur
    for B in (1, 2, 3, 5, 8):
        for mistake in MISTAKES:
            if window == 383 and B == 3 and mistake != "odd_tail":
                continue
            assert any(r is not None for p0, b, m, r in rows_out if b == B and m == mistake), (window, B, mistake)
