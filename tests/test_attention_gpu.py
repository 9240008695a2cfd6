"""The encoder attention kernels at operator level (vox_attention) against float64: K4-TC (enc_attn_tc.cu), K4
(kernels.cu) and K4-S (stream.cu).

The reference and its per-output bound are tests/test_attention_ref.py's (f64_and_bound); K4-TC and K4 run every
encoder case against one reference.  Cases:
  * offline shapes: S in {1, 2, 63, 64, 65, 129, 995, 1500} x window in {0, 1, 63, 64, 65, 750, >= S} at hd 32 and 64 on
    both kernels and hd 128 on K4, two heads, the production layout (ld = 3 H hd, q, k, v at 0, H hd, 2 H hd); H = 32 at
    hd 64 at S = 995 and 1500; a second layout with four NaN columns ahead of q and v ahead of k;
  * batches: B = 3 uniform, and a segment table of lengths {1, 50, 64, 65, 995};
  * operand sets: every set of test_attention_ref.py plus whole-tensor scales 2^-16 .. 2^+8 of Q and K and of V;
  * K4-S: ring = window + 256 (as StreamPool), windows 0, 1, 2, 3 and 750, rows of three sessions in one launch (before
    the ring wraps, straddling the wrap, near position 10^5), and 256 consecutive rows of one session; the k and v
    columns of its qkv rows are NaN (the kernel reads only q there).
Every call checks the bound, that the same call twice is bitwise equal, and that the output's guard row (pre-filled
with a NaN sentinel) is bitwise the sentinel afterwards; where both encoder kernels ran on at least 64 rows at a
window above 0 (at 0 both return each row's own v exactly), K4-TC and K4 differ bitwise somewhere.  The worst
error / bound ratio is printed per kernel and per operand set.  Then the seam's refusals.
"""
import numpy as np
import pytest

from test_attention_ref import OPERAND_SETS, encoder_ref, operands, ratio, ring_ref

pytestmark = pytest.mark.gpu

SENTINEL = np.uint32(0x7FC5A5A5).view(np.float32)
SEQ = (1, 2, 63, 64, 65, 129, 995, 1500)
WINDOWS = (0, 1, 63, 64, 65, 750, 100000)
SCALE_SETS = tuple(f"{w}_2^{e:+d}" for w in ("qk", "v") for e in (-16, -12, -8, -4, 4, 8))
SETS = OPERAND_SETS + tuple(s for s in SCALE_SETS if s not in OPERAND_SETS)

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for key in sorted(_worst):
        print(f"\n[attention] {key}: worst |out - o64| / bound = {_worst[key]:.3f}")


def scale_of(hd):
    return float(np.float32(hd) ** np.float32(-0.5))


def check(out, rows, o64, bound, kernel, aset, what):
    guard = out[rows:].view(np.uint32)
    assert np.all(guard == SENTINEL.view(np.uint32)), (what, "stray writes in the guard row")
    r = ratio(out[:rows], o64, bound)
    for key in (kernel, f"{kernel:6s} {aset}"):
        _worst[key] = max(_worst.get(key, 0.0), float(r.max()))
    at = np.unravel_index(int(np.argmax(r)), r.shape)
    assert r.max() <= 1.0, (what, at, float(r.max()), float(out[at]), float(o64[at]))


def build_qkv(aset, lens, h, hd, seed, window, layout="prod"):
    """rows of all streams, [rows, ld], and the offsets: "prod" = q | k | v, "alt" = 4 NaN | q | v | k"""
    hq = h * hd
    parts = [operands(aset, n, h, hd, seed + t, window) for t, n in enumerate(lens)]
    q, k, v = (np.concatenate([p[i] for p in parts]).reshape(-1, hq) for i in range(3))
    if layout == "prod":
        return np.concatenate([q, k, v], 1), 0, hq, 2 * hq
    pad = np.full((q.shape[0], 4), np.nan, np.float32)
    return np.concatenate([pad, q, v, k], 1), 4, 4 + 2 * hq, 4 + hq


def run_encoder(vx, aset, lens, h, hd, window, seed, layout="prod", uniform=True):
    qkv, q_off, k_off, v_off = build_qkv(aset, lens, h, hd, seed, window, layout)
    rows = qkv.shape[0]
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(int)
    o64, bound = encoder_ref(qkv, h, hd, q_off, k_off, v_off, starts, lens, window, scale_of(hd))
    kw = dict(q_off=q_off, k_off=k_off, v_off=v_off, out_rows=rows + 1, sentinel=SENTINEL)
    if uniform:
        kw.update(b=len(lens), s=lens[0])
    else:
        kw.update(b=len(lens), seg=np.concatenate([[0], np.cumsum(lens)]))
    outs = {}
    for kernel in (("tc", "simt") if hd != 128 else ("simt",)):
        what = (kernel, aset, lens, h, hd, window, layout)
        out = vx.attention(kernel, qkv, h, hd, window, scale_of(hd), **kw)
        again = vx.attention(kernel, qkv, h, hd, window, scale_of(hd), **kw)
        assert np.array_equal(out.view(np.uint32), again.view(np.uint32)), (what, "not reproducible")
        check(out, rows, o64, bound, {"tc": "K4-TC", "simt": "K4"}[kernel], aset, what)
        outs[kernel] = out[:rows]
    if len(outs) == 2 and rows >= 64 and window > 0:   # at window 0 every output is its own v, exactly
        assert not np.array_equal(outs["tc"].view(np.uint32), outs["simt"].view(np.uint32)), \
            (aset, lens, hd, window, "K4-TC and K4 gave bitwise the same result")


def _offline():
    out, i = [], 0
    for S in SEQ:
        for w in WINDOWS:
            for hd in (32, 64, 128):
                out.append(pytest.param(S, w, hd, SETS[i % len(SETS)], id=f"S{S}-w{w}-hd{hd}"))
                i += 1
    return out


@pytest.mark.parametrize("S,window,hd,aset", _offline())
def test_offline_shapes(vx, S, window, hd, aset):
    run_encoder(vx, aset, [S], 2, hd, window, S + window + hd)


@pytest.mark.parametrize("S,window", [(995, 750), (1500, 750), (1500, 100000)])
def test_production_heads(vx, S, window):
    """H = 32, hd = 64: the encoder's layout"""
    run_encoder(vx, "gauss", [S], 32, 64, window, S)


@pytest.mark.parametrize("hd", [32, 64, 128])
@pytest.mark.parametrize("window", [1, 64, 750])
def test_second_layout(vx, hd, window):
    """four NaN columns ahead of q, v ahead of k: nothing but q, k and v may reach an output"""
    run_encoder(vx, "gauss", [200], 3, hd, window, 11 * hd + window, layout="alt")


@pytest.mark.parametrize("hd", [32, 64, 128])
@pytest.mark.parametrize("window", [0, 65, 750])
def test_batches(vx, hd, window):
    run_encoder(vx, "gauss", [130, 130, 130], 2, hd, window, 3 + window)
    run_encoder(vx, "v_offset", [1, 50, 64, 65, 995], 2, hd, window, 5 + window, uniform=False)


@pytest.mark.parametrize("aset", SETS)
@pytest.mark.parametrize("window", [63, 750])
def test_operand_sets(vx, aset, window):
    """every operand set at hd 64 and 32, S = 300: queries deep in a 64-row tile see a first key tile that is entirely
    masked for them at window 63"""
    for hd in (32, 64):
        run_encoder(vx, aset, [300], 2, hd, window, 17 + window)


# ------------------------------------------------------------------------------------------------------ K4-S


def run_stream(vx, aset, slots, positions, h, hd, window, seed):
    ring = window + 256
    hq = h * hd
    n_slots = int(max(slots)) + 1
    q, kr, vr = operands(aset, n_slots * ring, h, hd, seed, window)
    kr, vr = kr.reshape(n_slots, ring, hq), vr.reshape(n_slots, ring, hq)
    rows = len(slots)
    qkv = np.full((rows, 3 * hq), np.nan, np.float32)
    qkv[:, :hq] = q.reshape(-1, hq)[:rows]
    o64, bound = ring_ref(qkv, h, hd, slots, positions, kr, vr, window, scale_of(hd))
    kw = dict(row_slot=np.asarray(slots, np.int32), row_pos=np.asarray(positions, np.int32), k_ring=kr, v_ring=vr,
              out_rows=rows + 1, sentinel=SENTINEL)
    what = ("stream", aset, h, hd, window)
    out = vx.attention("stream", qkv, h, hd, window, scale_of(hd), **kw)
    again = vx.attention("stream", qkv, h, hd, window, scale_of(hd), **kw)
    assert np.array_equal(out.view(np.uint32), again.view(np.uint32)), (what, "not reproducible")
    check(out, rows, o64, bound, "K4-S", aset, what)


@pytest.mark.parametrize("hd", [32, 64, 128])
@pytest.mark.parametrize("window", [0, 1, 2, 3, 750])
def test_stream_sessions(vx, window, hd):
    """three sessions in one launch: positions before the ring wraps, straddling the wrap, and near 10^5"""
    ring = window + 256
    pos = ([0, 1, 2, 3, 5, 130] + list(range(ring - 3, ring + 4)) + [100000 + i for i in range(6)])
    slots = [0] * 6 + [1] * 7 + [2] * 6
    for aset in ("gauss", "v_2^-16", "qk_2^+8", "v_offset"):
        run_stream(vx, aset, slots, pos, 2, hd, window, window + hd)


@pytest.mark.parametrize("window", [0, 3, 750])
def test_stream_consecutive_rows(vx, window):
    """256 consecutive rows of one session (the most a ring of window + 256 holds), H = 32, hd = 64"""
    run_stream(vx, "gauss", [0] * 256, list(range(5000, 5256)), 32, 64, window, 9)


# ------------------------------------------------------------------------------------------------------ refusals


def test_refusals(vx):
    """vox_attention refuses, with VOX_EINVAL and a reason, whatever the named kernel cannot honour"""
    import ctypes as C
    from voxtral_mini_realtime_rs_b200.api import _AttnArgs
    dev = vx.DeviceBuffer
    h, hd, rows = 2, 64, 70
    hq = h * hd
    qkv = dev.from_numpy(np.ones((rows + 1, 3 * hq), np.float32))
    qkv128 = dev.from_numpy(np.ones((rows, 3 * 2 * 128), np.float32))   # rows of ld = 768 for the hd 128 launch
    out = dev.from_numpy(np.zeros((rows + 1, 4 * hq), np.float32))
    slot = dev.from_numpy(np.zeros(rows, np.int32))
    pos = dev.from_numpy(np.arange(rows, dtype=np.int32))
    ring = dev.from_numpy(np.ones((1, 300, hq), np.float32))
    lib = vx.lib()

    def rc(kernel, **kw):
        a = dict(qkv=qkv.ptr, ld=3 * hq, q_off=0, k_off=hq, v_off=2 * hq, b=1, s=rows, h=h, hd=hd, seg=None,
                 rows=rows, row_slot=slot.ptr, row_pos=pos.ptr, k_ring=ring.ptr, v_ring=ring.ptr, ring=300, window=10,
                 scale=0.125, out=out.ptr)
        a.update(kw)
        code = lib.vox_attention(0, kernel, C.byref(_AttnArgs(**a)), None)
        assert lib.vox_dev_sync(0) == 0
        return code, lib.vox_last_error().decode()

    for kernel in (0, 1, 2):
        assert rc(kernel)[0] == 0
    assert rc(1, qkv=qkv128.ptr, hd=128, ld=3 * 2 * 128, k_off=256, v_off=512)[0] == 0
    assert rc(2, hd=32)[0] == 0 and rc(2, window=299)[0] == 0
    odd = C.c_void_p(qkv.ptr.value + 4)
    refused = {
        "unknown kernel 3": (3, {}),
        "unknown kernel -1": (-1, {}),
        "null qkv": (0, dict(qkv=None)),
        "null out": (2, dict(out=None)),
        "h < 1": (1, dict(h=0)),
        "negative window": (0, dict(window=-1)),
        "negative window, ring": (2, dict(window=-1)),
        "tc: b < 1": (0, dict(b=0)),
        "simt: s < 1": (1, dict(s=0)),
        "tc: hd 128": (0, dict(hd=128, ld=768, k_off=256, v_off=512)),
        "tc: hd 16": (0, dict(hd=16)),
        "simt: hd 96": (1, dict(hd=96, ld=3 * 192, k_off=192, v_off=384)),
        "tc: ld not a multiple of 4": (0, dict(ld=3 * hq + 2)),
        "tc: q_off not a multiple of 4": (0, dict(ld=3 * hq + 4, q_off=2)),
        "tc: k_off not a multiple of 4": (0, dict(ld=3 * hq + 4, k_off=hq + 2)),
        "tc: v_off not a multiple of 4": (0, dict(ld=3 * hq + 4, v_off=2 * hq + 2)),
        "tc: qkv not 16-byte aligned": (0, dict(qkv=odd, ld=3 * hq)),
        "simt: v past ld": (1, dict(v_off=2 * hq + 1)),
        "stream: hd 16": (2, dict(hd=16)),
        "stream: hd 96": (2, dict(hd=96)),
        "stream: rows < 1": (2, dict(rows=0)),
        "stream: window >= ring": (2, dict(window=300)),
        "stream: null ring": (2, dict(k_ring=None)),
        "stream: null row_pos": (2, dict(row_pos=None)),
    }
    for why, (kernel, kw) in refused.items():
        code, msg = rc(kernel, **kw)
        assert code == 1, (why, code, msg)
        assert msg.startswith("attention:"), (why, msg)
    assert rc(0)[0] == 0                                # a refusal launches nothing and leaves the library usable
