"""The decoder attention kernels at operator level (vox_dec_attention) against float64: K5 fused (dec_attn_fused_kernel,
decode_attn.cu) and K5 prefill (dec_rope_append_kernel + dec_attention_kernel, kernels.cu), over f32, f16 and q8 caches,
paged and ring-indexed.

The reference and its per-output bound are tests/test_dec_attention_ref.py's (f64_and_bound).  Each case builds a
cache whose rows sit on shuffled physical pages (beam-style rows share the full pages below their position), writes
the keys a row can see directly in the stored domain (f32, f16 bits, int8 codes and f16 scales), and fills every slot
no row may read with NaN (NaN scales for q8): keys before pos - window, slots after the last appended position, and
pages in no table.  A read outside the window or the row's table then shows up as NaN.  Every call checks:
  1. the output within the bound (NaN fails);
  2. the output's guard row, pre-filled with a NaN sentinel, bitwise untouched;
  3. both pools bitwise unchanged except at the appended (page, kv head, slot) rows (for q8 the row's values and scales);
  4. the appended V bitwise the storage rule of the f32 v;
  5. the appended K inside the interval the rotation bound allows: FMA contraction of x_r c - x_i s may differ between
     instantiations, so K is never required bit-exact; for q8 the block scale lies in the range the block's absmax
     allows and each code in [rint(lo / d), rint(hi / d)] for the stored d;
  6. qkv afterwards: prefill rotates q in place (within the rotation bound) and leaves k and v bitwise; the fused kernel
     leaves all of qkv bitwise;
  7. the same call again (qkv re-uploaded) gives bitwise the same output and pools.
Cases: the fused kernel at the production geometry (H 32, Hkv 8, hd 128) at B 1, 3, 8 with per-row positions around
page edges and the 64-entry shared page-table cache, every one of its 54 instantiations, ring caches sized as
DecoderKv sizes them at positions up to a day of audio, the prefill at M 1 .. 130 over all three caches, ring and not,
the largest capacity its 200 KB of shared memory accepts, both kernels on identical M = 1 inputs, and the seam's
refusals.  The worst error / bound ratio is printed per kernel x cache type x operand set.
"""
import ctypes as C

import numpy as np
import pytest

from test_dec_attention_ref import (OPERAND_SETS, F32, f64_and_bound, operands, ratio, rope_rows, rotate64,
                                    unrotate)
from test_kv_half_ref import kv16_from_f32
from test_kv_q8_ref import kv8_quant

pytestmark = pytest.mark.gpu

SENTINEL = np.uint32(0x7FC5A5A5).view(np.float32)
PAGE = 16
ROPE_RING = 4096                       # stream.cu's RoPE ring rows
KV_DT = {"f32": np.float32, "f16": np.float16}
_worst, _ran = {}, set()


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for key in sorted(_worst):
        print(f"\n[dec attention] {key}: worst |out - o64| / bound = {_worst[key]:.3f}")
    print(f"\n[dec attention] instantiations run: {sorted(_ran)}")


def ring_capacity(window, launch):
    """DecoderKv::create's ring: ((window + launch) / 16 + 1) * 16 positions, launch at least 64"""
    return ((window + max(launch, 64)) // PAGE + 1) * PAGE


# ------------------------------------------------------------------------------------------------ the cache


class Pool:
    """[pages][hkv] units of 16 positions in a cache's stored form, as bytes; positions written through a page table"""

    def __init__(self, kv, n_pages, hkv, hd):
        self.kv, self.hkv, self.hd = kv, hkv, hd
        if kv == "q8":
            self.unit = PAGE * hd + PAGE * (hd // 16) * 2
            self.k, self.v = (np.zeros((n_pages, hkv, self.unit), np.uint8) for _ in range(2))
            for a in (self.k, self.v):
                a[..., :PAGE * hd] = 0x55                                        # codes of NaN scales
                a[..., PAGE * hd:].view(np.float16)[:] = np.float16(np.nan)
        else:
            self.k, self.v = (np.full((n_pages, hkv, PAGE, hd), np.nan, KV_DT[kv]) for _ in range(2))

    def row_index(self, page, g, slot):
        """where one position is held: [values] or, for q8, [values, scales] (byte ranges of the unit)"""
        if self.kv != "q8":
            return [(page, g, slot)]
        hd, sb = self.hd, (self.hd // 16) * 2
        return [(page, g, slice(slot * hd, (slot + 1) * hd)),
                (page, g, slice(PAGE * hd + slot * sb, PAGE * hd + (slot + 1) * sb))]

    def row_bytes(self, a, page, g, slot):
        """views of the bytes that hold one position: [values] or [values, scales]"""
        return [a[i].view(np.uint8) for i in self.row_index(page, g, slot)]

    def write(self, a, page, g, slot, x):
        """store f32 values x [hd] by the cache's rule"""
        if self.kv == "q8":
            q, d = kv8_quant(x)
            vals, sc = self.row_bytes(a, page, g, slot)
            vals[:], sc[:] = q.view(np.uint8), d.view(np.uint8)
        elif self.kv == "f16":
            a[page, g, slot] = kv16_from_f32(x)
        else:
            a[page, g, slot] = x

    def read(self, a, page, g, slot):
        """the stored values at one position, decoded exactly, float64 [hd]"""
        if self.kv == "q8":
            vals, sc = self.row_bytes(a, page, g, slot)
            q = vals.view(np.int8).astype(np.float64).reshape(-1, 16)
            return (sc.view(np.float16).astype(np.float32).astype(np.float64)[:, None] * q).reshape(-1)
        return a[page, g, slot].astype(np.float64)


class Case:
    def __init__(self, kernel, kv, G, hkv, hd, starts, M, window, aset, seed, ring=False, capacity=None, beam=False,
                 rope_ring=None):
        self.kernel, self.kv, self.G, self.hkv, self.hd = kernel, kv, G, hkv, hd
        self.H = G * hkv
        self.starts, self.M, self.window, self.aset, self.ring = list(starts), M, window, aset, ring
        B = self.B = len(starts)
        self.beam = beam and not ring
        ends = [s + M - 1 for s in starts]
        if capacity is None:
            capacity = ring_capacity(window, M) if ring else (max(ends) // PAGE + 2) * PAGE
        self.capacity, self.max_pages = capacity, capacity // PAGE
        rng = np.random.default_rng(seed)
        # ---- page tables: slot 0 of the pool is a NaN page every unreachable table entry points at; a few pages are
        # in no table at all
        table = np.zeros((B, self.max_pages), np.int32)
        need = []                                            # (row, table slot) that get a page of their own
        for b, (s, e) in enumerate(zip(starts, ends)):
            lo = max(0, s - window)
            lps = range(lo // PAGE, e // PAGE + 1)
            slots = sorted({lp % self.max_pages for lp in lps}) if ring else list(lps)
            for t in slots:
                if not (self.sibling(b) and t < s // PAGE):
                    need.append((b, t))
        ids = rng.permutation(len(need) + 3) + 1
        for (b, t), p in zip(need, ids):
            table[b, t] = p
        for b in range(B):                                   # beam siblings: the full pages below the position
            if self.sibling(b):
                for t in range(starts[b] // PAGE):
                    if table[b, t] == 0:
                        table[b, t] = table[b - 1, t]
        self.table = table
        self.pool = Pool(kv, len(need) + 4, hkv, hd)
        # ---- RoPE: a full table, or a 4096-row ring filled for the launch's positions (NaN elsewhere)
        pos_all = np.concatenate([np.arange(s, s + M) for s in starts])
        if ring:
            rows = rope_ring or ROPE_RING
            self.cos, self.sin = (np.full((rows, hd // 2), np.nan, F32) for _ in range(2))
            distinct = np.unique(pos_all)
            assert len(np.unique(distinct % rows)) == len(distinct), "two of the launch's positions share a RoPE row"
            c, s_ = rope_rows(pos_all, hd)
            self.cos[pos_all % rows], self.sin[pos_all % rows] = c, s_
        else:
            self.cos, self.sin = rope_rows(np.arange(max(ends) + 1 + (rng.integers(0, 3))), hd)
        # ---- operands after RoPE, per (row, kv head): the keys lo .. end and the M queries of each of the G heads
        ld = self.ld = (self.H + 2 * hkv) * hd
        qkv = np.full((B * M, ld), np.nan, F32)
        self.keys = {}
        for b, s in enumerate(starts):
            lo = max(0, s - window)
            n = ends[b] - lo + 1
            c, sn = self.rope(np.arange(s, s + M))
            kv_row = b - 1 if self.sibling(b) else b      # beam siblings hold the same keys (their pages are shared)
            for g in range(hkv):
                sd = seed + 1000 * b + 10 * g
                qh = operands(aset, M, n, hd, sd, edge=ends[b] - window - lo)[0]
                k, v = operands(aset, M, n, hd, seed + 1000 * kv_row + 10 * g, edge=ends[b] - window - lo)[1:]
                k, v = k.astype(F32).astype(np.float64), v.astype(F32)
                for hh in range(G):
                    qq = qh if hh == 0 else operands(aset, M, n, hd, sd + hh)[0]
                    h = g * G + hh
                    qkv[b * M:(b + 1) * M, h * hd:(h + 1) * hd] = unrotate(qq, c, sn)
                kk = self.H * hd + g * hd
                qkv[b * M:(b + 1) * M, kk:kk + hd] = unrotate(k[n - M:], c, sn)
                vv = (self.H + hkv) * hd + g * hd
                qkv[b * M:(b + 1) * M, vv:vv + hd] = v[n - M:]
                for j in range(lo, s):                       # visible keys before the launch, in the stored domain
                    page, slot = self.where(b, j)
                    self.pool.write(self.pool.k, page, g, slot, k[j - lo].astype(F32))
                    self.pool.write(self.pool.v, page, g, slot, v[j - lo])
        self.qkv = qkv
        self.scale = float(F32(hd) ** F32(-0.5))

    def sibling(self, b):
        """row b is a beam sibling of row b - 1: the same position, the full pages below it shared"""
        return self.beam and b % 2 == 1 and self.starts[b - 1] == self.starts[b]

    def rope(self, positions):
        rows = self.cos.shape[0]
        r = np.asarray(positions) % rows if self.ring else np.asarray(positions)
        return self.cos[r], self.sin[r]

    def where(self, b, j):
        lp = j // PAGE
        return self.table[b, lp % self.max_pages if self.ring else lp], j % PAGE

    def launch(self, vx, qkv=None):
        return vx.dec_attention(self.kernel, self.qkv if qkv is None else qkv, b=self.B, m=self.M, h=self.H,
                                hkv=self.hkv, hd=self.hd, kv_dtype=self.kv, k_pool=self.pool.k, v_pool=self.pool.v,
                                page_table=self.table, pos=np.array(self.starts, np.int32), cos=self.cos, sin=self.sin,
                                window=self.window, scale=self.scale, ring=self.ring, out_rows=self.B * self.M + 1,
                                sentinel=SENTINEL)


# ------------------------------------------------------------------------------------------------ checks


def _k_interval_ok(pool, stored_bytes, k32, c, s):
    """the appended K (one position, one kv head) against the interval RoPE's f32 rounding allows"""
    k64, mag = rotate64(k32, c, s)
    lo, hi = k64 - 2.0 ** -22 * mag, k64 + 2.0 ** -22 * mag
    if pool.kv == "f32":
        got = stored_bytes[0].view(np.float32).astype(np.float64)
        return bool(np.all((got >= lo) & (got <= hi)))
    if pool.kv == "f16":
        got = stored_bytes[0].view(np.float16).astype(np.float64)
        rule = lambda x: np.clip(x, -65504.0, 65504.0).astype(np.float16).astype(np.float64)   # noqa: E731
        return bool(np.all((got >= rule(lo)) & (got <= rule(hi))))
    codes = stored_bytes[0].view(np.int8).astype(np.float64).reshape(-1, 16)
    d = stored_bytes[1].view(np.float16)
    lo32 = np.nextafter(lo.astype(F32), F32(-np.inf)).reshape(-1, 16)
    hi32 = np.nextafter(hi.astype(F32), F32(np.inf)).reshape(-1, 16)
    amin = np.where((lo32 <= 0) & (hi32 >= 0), F32(0), np.minimum(np.abs(lo32), np.abs(hi32))).max(1)
    amax = np.maximum(np.abs(lo32), np.abs(hi32)).max(1)
    d_rule = lambda a: np.minimum(a / F32(127), F32(65504)).astype(np.float16).astype(F32)   # noqa: E731
    df = d.astype(F32)
    if not np.all((df >= d_rule(amin)) & (df <= d_rule(amax))):
        return False
    with np.errstate(divide="ignore", invalid="ignore"):
        qlo = np.clip(np.rint(lo32 / df[:, None]), -127, 127)
        qhi = np.clip(np.rint(hi32 / df[:, None]), -127, 127)
    qlo[df == 0], qhi[df == 0] = 0, 0
    return bool(np.all((codes >= qlo) & (codes <= qhi)))


def _v_bytes(pool, v32):
    if pool.kv == "q8":
        q, d = kv8_quant(v32)
        return [q.view(np.uint8), d.view(np.uint8)]
    return [(kv16_from_f32(v32) if pool.kv == "f16" else v32.astype(F32)).view(np.uint8)]


def run(vx, case, tag=None):
    """launch, check 1..7, return (out rows, o64, bound)"""
    cs, pool, hd, M = case, case.pool, case.hd, case.M
    what = (cs.kernel, cs.kv, cs.G, cs.hkv, hd, cs.ring, cs.starts, M, cs.window, cs.aset)
    out, qkv_after, k_after, v_after = cs.launch(vx)
    rows = cs.B * M
    assert np.all(out[rows:].view(np.uint32) == SENTINEL.view(np.uint32)), (what, "stray writes in the guard row")
    # ---- 3: pools changed only at the appended rows; 4, 5: what those rows hold
    touched = np.zeros(pool.k.shape, bool)           # the appended rows' elements (q8: bytes)
    for b, s in enumerate(cs.starts):
        for i in range(M):
            page, slot = cs.where(b, s + i)
            c, sn = cs.rope([s + i])
            for g in range(cs.hkv):
                for i_row in pool.row_index(page, g, slot):
                    touched[i_row] = True
                r = b * M + i
                k0, v0 = (cs.H + g) * hd, (cs.H + cs.hkv + g) * hd
                k32, v32 = cs.qkv[r, k0:k0 + hd], cs.qkv[r, v0:v0 + hd]
                got_v = pool.row_bytes(v_after, page, g, slot)
                for got, want in zip(got_v, _v_bytes(pool, v32)):
                    assert np.array_equal(got.view(np.uint8), want), (what, "appended V", b, i, g)
                assert _k_interval_ok(pool, pool.row_bytes(k_after, page, g, slot), k32, c[0], sn[0]), \
                    (what, "appended K outside the RoPE interval", b, i, g)
    bits = {1: np.uint8, 2: np.uint16, 4: np.uint32}[pool.k.itemsize]
    for name, before, after in (("K", pool.k, k_after), ("V", pool.v, v_after)):
        assert np.array_equal(before.view(bits)[~touched], after.view(bits)[~touched]), \
            (what, f"{name} pool changed outside the appended rows")
    # ---- 6: qkv afterwards
    hq = cs.H * hd
    if cs.kernel == "fused":
        assert np.array_equal(qkv_after.view(np.uint32), cs.qkv.view(np.uint32)), (what, "fused kernel changed qkv")
    else:
        assert np.array_equal(qkv_after[:, hq:].view(np.uint32), cs.qkv[:, hq:].view(np.uint32)), \
            (what, "prefill changed the k / v columns")
        for b, s in enumerate(cs.starts):
            c, sn = cs.rope(np.arange(s, s + M))
            q = cs.qkv[b * M:(b + 1) * M, :hq].reshape(M, cs.H, hd)
            q64, mag = rotate64(q, c[:, None], sn[:, None])
            got = qkv_after[b * M:(b + 1) * M, :hq].reshape(M, cs.H, hd).astype(np.float64)
            assert np.all(np.abs(got - q64) <= 2.0 ** -22 * mag), (what, "q rotated in place outside the bound")
    # ---- 1: the output against the reference over the stored keys
    o64, bound = np.zeros((rows, hq)), np.ones((rows, hq))
    for b, s in enumerate(cs.starts):
        lo = max(0, s - cs.window)
        j = np.arange(lo, s + M)
        p = np.arange(s, s + M)
        mask = (j[None] <= p[:, None]) & (p[:, None] - j[None] <= cs.window)
        c, sn = cs.rope(p)
        for g in range(cs.hkv):
            locs = [cs.where(b, jj) for jj in j]
            kk = np.stack([pool.read(k_after, pg, g, sl) for pg, sl in locs])
            vv = np.stack([pool.read(v_after, pg, g, sl) for pg, sl in locs])
            for hh in range(cs.G):
                h = g * cs.G + hh
                cols = slice(h * hd, (h + 1) * hd)
                o64[b * M:(b + 1) * M, cols], bound[b * M:(b + 1) * M, cols] = f64_and_bound(
                    cs.kernel, cs.qkv[b * M:(b + 1) * M, cols], c, sn, kk, vv, mask, cs.scale)
    r = ratio(out[:rows], o64, bound)
    _ran.add((cs.kernel, cs.G, hd, cs.ring, cs.kv))
    for key in (f"{cs.kernel:7s} {cs.kv}", f"{cs.kernel:7s} {cs.kv:3s} {tag or cs.aset}"):
        _worst[key] = max(_worst.get(key, 0.0), float(r.max()))
    at = np.unravel_index(int(np.argmax(r)), r.shape)
    assert r.max() <= 1.0, (what, at, float(r.max()), float(out[at]), float(o64[at]))
    # ---- 7: the same call again
    again = cs.launch(vx, cs.qkv.copy())
    assert np.array_equal(again[0].view(np.uint32), out.view(np.uint32)), (what, "output not reproducible")
    for got, first in zip(again[2:], (k_after, v_after)):
        assert np.array_equal(got.view(np.uint8), first.view(np.uint8)), (what, "pools not reproducible")
    return out[:rows], o64, bound


# ------------------------------------------------------------------------------------------------ fused kernel

FUSED_POS = (0, 1, 7, 8, 9, 15, 16, 17, 1023, 1024, 1025)
FUSED_CAP = 1280
SETS = OPERAND_SETS


def _sets_for(kv):
    return [s for s in SETS if (s != "q8_blocks" or kv == "q8") and (s != "f16_range" or kv == "f16")]


def _fused_prod():
    out, i = [], 0
    for kv in ("f32", "f16", "q8"):
        for B in (1, 3, 8):
            for w in (0, 1, 7, 8, 9, 383, 8192):
                out.append(pytest.param(kv, B, w, i, id=f"{kv}-B{B}-w{w}"))
                i += 1
    return out


@pytest.mark.parametrize("kv,B,window,i", _fused_prod())
def test_fused_production_geometry(vx, kv, B, window, i):
    """H 32, Hkv 8, hd 128: every row at its own position; 1024 and up read the page table from global memory"""
    pool = FUSED_POS + (FUSED_CAP - 1,)
    starts = [pool[(i + 5 * b) % len(pool)] for b in range(B)]
    if B == 8:                                           # beam-style: rows 2k and 2k + 1 share the pages below
        starts[1::2] = starts[0::2]
    sets = _sets_for(kv)
    run(vx, Case("fused", kv, 4, 8, 128, starts, 1, window, sets[i % len(sets)], 11 + i, capacity=FUSED_CAP,
                 beam=B == 8))


def _instantiations():
    out = []
    for G in (1, 2, 4):
        for hd in (32, 64, 128):
            for ring in (False, True):
                for kv in ("f32", "f16", "q8"):
                    out.append(pytest.param(G, hd, ring, kv, id=f"G{G}-hd{hd}-{'ring' if ring else 'paged'}-{kv}"))
    return out


FUSED_INST = _instantiations()


@pytest.mark.parametrize("G,hd,ring,kv", FUSED_INST)
def test_fused_every_instantiation(vx, G, hd, ring, kv):
    """window 40 bites and the keys cross pages; the ring (capacity 112) has wrapped"""
    starts = [300, 301] if ring else [100, 57]
    sets = _sets_for(kv)
    run(vx, Case("fused", kv, G, 2, hd, starts, 1, 40, sets[(G + hd + ring) % len(sets)], G * hd + ring, ring=ring))


# ------------------------------------------------------------------------------------------------ ring caches


RING_POS = {"before_wrap": 0, "straddle": 1, "1e5": 100000, "day": 1080000}


@pytest.mark.parametrize("kernel", ["fused", "prefill"])
@pytest.mark.parametrize("window", [40, 8192])
@pytest.mark.parametrize("where", list(RING_POS))
def test_ring(vx, kernel, window, where):
    """capacity ((window + L) / 16 + 1) * 16 with L = max(M, 64); a 4096-row RoPE ring; at 8192 past the first lap the
    ring is full"""
    M = 1 if kernel == "fused" else 64
    cap = ring_capacity(window, M)
    if where == "before_wrap":
        starts = [cap // 4, cap - M - 5]
    elif where == "straddle":
        starts = [cap - M // 2 - 1, 2 * cap - 7]
    else:
        starts = [RING_POS[where] + 13, RING_POS[where] + 3 * cap + 2]
    G, hkv, hd = (4, 2, 128) if kernel == "fused" else (2, 1, 128)
    for kv in ("f32", "f16", "q8"):
        run(vx, Case(kernel, kv, G, hkv, hd, starts, M, window, "gauss" if kv != "q8" else "rising",
                     window + len(where), ring=True))


# ------------------------------------------------------------------------------------------------ prefill


def _prefill():
    out, i = [], 0
    geoms = [(4, 8, 128), (1, 2, 32), (2, 2, 64), (4, 1, 32), (2, 1, 128), (1, 1, 64)]
    for M in (1, 2, 37, 38, 39, 64, 130):
        for w in (0, 1, 31, 32, 33, 40, 8192):
            kv = ("f32", "f16", "q8")[i % 3]
            ring = i % 2 == 1
            G, hkv, hd = geoms[0] if M <= 39 and i % 4 == 0 else geoms[1 + i % 5]
            B = (1, 3, 8)[(i // 3) % 3] if M <= 64 else 1
            out.append(pytest.param(M, w, kv, ring, G, hkv, hd, B, i,
                                    id=f"M{M}-w{w}-{kv}-{'ring' if ring else 'paged'}-G{G}h{hkv}d{hd}-B{B}"))
            i += 1
    return out


@pytest.mark.parametrize("M,window,kv,ring,G,hkv,hd,B,i", _prefill())
def test_prefill(vx, M, window, kv, ring, G, hkv, hd, B, i):
    """per-row starts that differ: 0, 5, 1000 and across a page"""
    starts = [(0, 5, 1000, 14, 1000, 5, 30, 47)[(b + i) % 8] for b in range(B)]
    if B == 8 and not ring:                              # beam-style: rows 2k and 2k + 1 share the pages below
        starts[1::2] = starts[0::2]
    if ring:
        starts = [s + (ring_capacity(window, M) if b % 2 else 0) for b, s in enumerate(starts)]
    sets = _sets_for(kv)
    run(vx, Case("prefill", kv, G, hkv, hd, starts, M, window, sets[i % len(sets)], 3 + i, ring=ring, beam=B >= 3))


PREFILL_MAX_CAP = (200 * 1024 // 4 // 4 - 128) // PAGE * PAGE     # G = 4, hd = 128: 12672 positions


@pytest.mark.parametrize("kv", ["f32", "f16", "q8"])
def test_prefill_largest_capacity(vx, kv):
    """the largest cache the prefill's 200 KB of shared memory holds at G 4, hd 128, full to its last position"""
    run(vx, Case("prefill", kv, 4, 1, 128, [PREFILL_MAX_CAP - 2], 2, 8192, "gauss", 5, capacity=PREFILL_MAX_CAP))


@pytest.mark.parametrize("kv", ["f32", "f16", "q8"])
@pytest.mark.parametrize("ring", [False, True])
def test_both_kernels_same_inputs(vx, kv, ring):
    """M = 1: the fused and prefill kernels on identical inputs, each within the bound"""
    for kernel in ("fused", "prefill"):
        run(vx, Case(kernel, kv, 4, 2, 128, [700, 33, 1500], 1, 383, "rising", 21, ring=ring), tag="same_inputs")


def test_instantiation_coverage():
    """the cases above run all 54 fused instantiations and all 6 of the prefill kernels"""
    fused = {(p.values[0], p.values[1], p.values[2], p.values[3]) for p in FUSED_INST}
    assert len(fused) == 54
    prefill = {(p.values[2], p.values[3]) for p in _prefill()}
    assert prefill == {(kv, r) for kv in ("f32", "f16", "q8") for r in (False, True)}


# ------------------------------------------------------------------------------------------------ refusals


def test_refusals(vx):
    """vox_dec_attention refuses, with VOX_EINVAL and a reason, whatever the named kernel cannot honour -- before any
    launch -- and so do the launchers' ring guards"""
    from voxtral_mini_realtime_rs_b200.api import _DecAttnArgs
    dev = vx.DeviceBuffer
    H, hkv, hd, B, M = 8, 2, 64, 2, 4
    ld = (H + 2 * hkv) * hd
    max_pages = 8
    qkv = dev.from_numpy(np.ones((B * M, ld), np.float32))
    pools = {t: dev.from_numpy(np.zeros(max_pages * B * hkv * PAGE * hd * 4, np.uint8)) for t in "kv"}
    table = dev.from_numpy(np.arange(B * max_pages, dtype=np.int32))
    pos = dev.from_numpy(np.array([3, 100], np.int32))
    pos_far = dev.from_numpy(np.array([3, 126], np.int32))
    pos_neg = dev.from_numpy(np.array([-1, 3], np.int32))
    cos = dev.from_numpy(np.ones((200, hd // 2), np.float32))
    sin = dev.from_numpy(np.zeros((200, hd // 2), np.float32))
    out_host = np.full((B * M, H * hd), SENTINEL, np.float32)
    out = dev.from_numpy(out_host)
    lib = vx.lib()

    def rc(kernel, **kw):
        a = dict(qkv=qkv.ptr, ld=ld, b=B, m=1 if kernel == 0 else M, h=H, hkv=hkv, hd=hd, kv_dtype=0,
                 k_pool=pools["k"].ptr, v_pool=pools["v"].ptr, page_table=table.ptr, max_pages=max_pages, ring=0,
                 pos=pos.ptr, cos=cos.ptr, sin=sin.ptr, rope_rows=200, window=10, scale=0.125, out=out.ptr)
        a.update(kw)
        code = lib.vox_dec_attention(0, kernel, C.byref(_DecAttnArgs(**a)), None)
        assert lib.vox_dev_sync(0) == 0
        return code, lib.vox_last_error().decode()

    refused = {
        "unknown kernel 2": (2, {}),
        "unknown kernel -1": (-1, {}),
        "unknown kv dtype": (1, dict(kv_dtype=2)),
        "null qkv": (0, dict(qkv=None)),
        "null k_pool": (1, dict(k_pool=None)),
        "null v_pool": (0, dict(v_pool=None)),
        "null page_table": (1, dict(page_table=None)),
        "null pos": (0, dict(pos=None)),
        "null cos": (1, dict(cos=None)),
        "null sin": (0, dict(sin=None)),
        "null out": (1, dict(out=None)),
        "b < 1": (1, dict(b=0)),
        "m < 1": (1, dict(m=0)),
        "h < 1": (1, dict(h=0)),
        "hkv < 1": (1, dict(hkv=0)),
        "hd < 1": (1, dict(hd=0)),
        "max_pages < 1": (0, dict(max_pages=0)),
        "rope_rows < 1": (1, dict(rope_rows=0)),
        "h % hkv": (1, dict(h=7)),
        "ld short": (0, dict(ld=ld - 1)),
        "negative window": (1, dict(window=-1)),
        "fused: m = 2": (0, dict(m=2)),
        "fused: G = 8": (0, dict(hkv=1, ld=(H + 2) * hd)),
        "fused: hd 96": (0, dict(hd=96, ld=(H + 2 * hkv) * 96)),
        "fused: hd 16": (0, dict(hd=16)),
        "prefill: hd not a multiple of 4": (1, dict(hd=62)),
        "prefill: q8 hd not a multiple of 16": (1, dict(hd=56, kv_dtype=100)),
        "prefill: shared memory": (1, dict(max_pages=3200 // PAGE * 4, hkv=1, ld=(H + 2) * hd)),
        "paged: pos + m past capacity": (1, dict(pos=pos_far.ptr)),
        "paged: pos past capacity, fused": (0, dict(pos=pos_far.ptr, max_pages=7)),
        "paged: pos + m past rope_rows": (1, dict(rope_rows=103)),
        "paged: negative pos": (0, dict(pos=pos_neg.ptr)),
    }
    guards = {   # the launchers' own ring guards (kernels.cu launch_dec_attention, decode_attn.cu launch_dec_attn_fused)
        "ring, prefill: window + m > capacity": (1, dict(ring=1, window=8 * PAGE - M + 1), "dec_attention:"),
        "ring, fused: window >= capacity": (0, dict(ring=1, window=8 * PAGE), "dec_attn_fused:"),
    }
    assert rc(0)[0] == 0 and rc(1)[0] == 0
    assert rc(1, ring=1, window=8 * PAGE - M)[0] == 0 and rc(0, ring=1, window=8 * PAGE - 1)[0] == 0
    assert rc(1, pos=pos_far.ptr, m=2)[0] == 0 and rc(1, rope_rows=104)[0] == 0
    for why, (kernel, kw) in refused.items():
        out.free()
        out = dev.from_numpy(out_host)
        kw = {**kw, "out": None} if kw.get("out", 1) is None else {**kw, "out": out.ptr}
        qkv_before = qkv.to_numpy(np.float32, (B * M, ld))
        code, msg = rc(kernel, **kw)
        assert code == 1, (why, code, msg)
        assert msg.startswith("dec_attention:"), (why, msg)
        assert np.array_equal(out.to_numpy(np.float32, out_host.shape).view(np.uint32), out_host.view(np.uint32)), \
            (why, "a refused call wrote its output")
        assert np.array_equal(qkv.to_numpy(np.float32, (B * M, ld)), qkv_before), (why, "a refused call rotated q")
    not_refused = []
    for why, (kernel, kw, prefix) in guards.items():
        out.free()
        out = dev.from_numpy(out_host)
        qkv_before = qkv.to_numpy(np.float32, (B * M, ld))
        code, msg = rc(kernel, **kw, out=out.ptr)
        if not (code == 1 and msg.startswith(prefix)):
            not_refused.append((why, code, msg))
            continue
        assert np.array_equal(out.to_numpy(np.float32, out_host.shape).view(np.uint32), out_host.view(np.uint32)), \
            (why, "a refused call wrote its output")
        assert np.array_equal(qkv.to_numpy(np.float32, (B * M, ld)), qkv_before), (why, "a refused call rotated q")
    assert not not_refused, not_refused
    assert rc(1)[0] == 0 and rc(0)[0] == 0               # a refusal launches nothing and leaves the library usable
