"""Every fused linear-layer form the model runs, on all four Q4 kernels, against float64 (vox_q4_linear).

The reference and its bound are tests/test_linear_forms_ref.py's (LinearRef): y = epi(norm(x) . W^T + bias) (+ res)
with RMSNorm, per-stream ADA vectors, bias, in-place residual, GELU and SiLU*up.  Each (form, rows) case runs in mode
"tc" (the tensor-core matvec at rows <= 8, the wgmma GEMM above on its shapes) and mode "simt" (the SIMT matvec and
the SIMT GEMM), against one f64 reference shared by both.  Forms at their production shapes (csrc/encoder.cu layers
and adapt, csrc/model.cu decoder_forward, lm_head_rows and compute_ada; the lm_head with a reduced vocabulary so that its
f64 weights fit in host memory), plus odd shapes on the matvec and SIMT GEMM paths: N = 17 and 208 at K = 4192, and
N = 18 at K = 96 (SiLU*up over a partial 16-row tile).  The activation sets rotate over the cases; N = 256, K = 3072
runs every set with every form on each of the four kernels.

Every call also checks:
  * writes stay in bounds: y has ldy = N + 40 (SiLU*up: N/2 + 40) and a guard row, all pre-filled with a NaN
    sentinel, and everything outside [rows][N] (N/2) is bitwise the sentinel afterwards.  That covers the padded token
    rows of the wgmma GEMM's 64-row-rounded tile and the matvec's last partial 16-row tile;
  * reproducibility: the same call twice is bitwise equal;
  * in place: for a residual, y == res gives bitwise the out-of-place result (at 321 and 586 rows the wgmma GEMM
    splits tiles across CTAs);
  * the kernel choice is real: where the modes pick different kernels, "tc" and "simt" differ bitwise somewhere
    among the outputs the product shows in (rows of x not all zero, and for a residual not lost below res).
Then the sum-of-squares hand-off of the tensor-core matvec (a residual call's ssq_out, read by the next call's norm as
ssq_in), and the seam's refusals.  The worst error / bound ratio is printed per (kernel, epilogue, norm).
"""
import numpy as np
import pytest

from test_linear_forms_ref import (ACT_SETS, EPS, LinearRef, make_ada, make_bias, make_gamma, make_res, acts,
                                   norm_allowed, ratio, weights)

pytestmark = pytest.mark.gpu

MODES = {"tc": 0, "simt": 3}
SENTINEL = np.uint32(0x7FC5A5A5).view(np.float32)
PAD = 40
ENC_ROWS = (1, 3, 8, 65, 320, 586)
DEC_ROWS = (1, 2, 5, 8, 9, 38, 114, 304, 321)
PREFILL = 38                               # decoder rows per stream of a prefill

# name: (N, K, epilogue, bias, norm, ada, rows)
FORMS = {
    "enc_wqkv": (6144, 1280, "none", True, True, False, ENC_ROWS),
    "enc_wo": (1280, 2048, "residual", True, False, False, ENC_ROWS),
    "enc_w13": (10240, 1280, "silu_mul", False, True, False, ENC_ROWS),
    "enc_w2": (1280, 5120, "residual", True, False, False, ENC_ROWS),
    "adapter0": (3072, 5120, "gelu", False, False, False, (8, 65, 304)),
    "adapter2": (3072, 3072, "none", False, False, False, (8, 65, 304)),
    "dec_wqkv": (6144, 3072, "none", False, True, False, DEC_ROWS),
    "dec_wo": (3072, 4096, "residual", False, False, False, DEC_ROWS),
    "dec_w13": (18432, 3072, "silu_mul", False, True, True, DEC_ROWS),
    "dec_w2": (3072, 9216, "residual", False, False, False, DEC_ROWS),
    "lm_head": (8192, 3072, "none", False, True, False, (1, 8, 38)),
    "ada0": (32, 3072, "gelu", False, False, False, (1,)),
    "ada2": (3072, 32, "residual", False, False, False, (1,)),      # onto ones; K = 32: the matvec's half-empty pair
    "odd17_none": (17, 4192, "none", True, False, False, (1, 5, 8, 9, 38)),
    "odd17_gelu": (17, 4192, "gelu", True, True, False, (1, 5, 8, 9, 38)),
    "odd208_res": (208, 4192, "residual", True, True, False, (1, 5, 8, 9, 38)),
    "odd208_gelu": (208, 4192, "gelu", False, False, False, (1, 5, 8, 9, 38)),
    "odd18_silu": (18, 96, "silu_mul", False, True, False, (1, 5, 8, 9, 38)),
}

_worst = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for key in sorted(_worst):
        print(f"\n[linear forms] {key}: worst |y - y64| / bound = {_worst[key]:.3f}")


def kernel_of(mode, n, k, rows):
    if rows <= 8:
        return "matvec_tc" if mode == "tc" else "matvec_simt"
    return "gemm_wgmma" if mode == "tc" and n % 128 == 0 and k % 64 == 0 else "gemm_simt"


_refs = {}


def ref_of(name, n, k):
    """One dequantised weight at a time (the cases run form by form): the large forms' f64 weights are the cost"""
    if name not in _refs:
        while len(_refs) >= 2:
            _refs.pop(next(iter(_refs)))
        kind = "signed" if sum(map(ord, name)) % 2 else "random"
        _refs[name] = LinearRef(weights(kind, n, k, n + k), n, k)
    return _refs[name]


def ada_m_of(rows):
    return PREFILL if rows % PREFILL == 0 else 1


def layer_inputs(n, k, epi, bias, norm, ada, rows, aset, seed, ones_res=False):
    x = acts(aset, rows, k, seed)
    kw = dict(epi=epi, bias=make_bias(n, seed + 1) if bias else None)
    if epi == "residual":
        kw["res"] = np.ones((rows, n), np.float32) if ones_res else make_res(rows, n, seed + 2)
    if norm:
        kw["gamma"] = make_gamma(k, seed + 3)
        if ada:
            m = ada_m_of(rows)
            kw.update(ada=make_ada(-(-rows // m), k, seed + 4), ada_m=m)
    return x, kw


def call(vx, mode, w, x, kw, in_place=False, **extra):
    assert vx.lib().vox_q4_set_matvec_mode(MODES[mode]) == 0
    try:
        n, _ = w.shape()
        cols = n // 2 if kw["epi"] == "silu_mul" else n
        return vx.q4_linear(w, x, kw["epi"], bias=kw.get("bias"), res=kw.get("res"), gamma=kw.get("gamma"), eps=EPS,
                            ada=kw.get("ada"), ada_m=kw.get("ada_m", 1), ldy=cols + PAD, y_rows=x.shape[0] + 1,
                            sentinel=SENTINEL, in_place=in_place, **extra)
    finally:
        vx.lib().vox_q4_set_matvec_mode(0)


def check_padding(out, rows, cols, what):
    pad = out.copy()
    pad[:rows, :cols] = SENTINEL
    bad = np.argwhere(pad.view(np.uint32) != SENTINEL.view(np.uint32))
    assert bad.size == 0, (what, "stray writes at", bad[:4].tolist())


def check_bound(out, y64, bound, key, what):
    assert np.all(np.isfinite(out)), (what, np.argwhere(~np.isfinite(out))[:4].tolist())
    r = ratio(out, y64, bound)
    _worst[key] = max(_worst.get(key, 0.0), float(r.max()))
    worst = np.unravel_index(int(np.argmax(r)), r.shape)
    assert r.max() <= 1.0, (what, worst, float(r.max()), float(out[worst]), float(y64[worst]))


def run_case(vx, ref, w, x, kw, label):
    """Both modes against one f64 reference, with the padding, repeat, in-place and kernel-choice checks"""
    n, k = ref.n, ref.k
    rows = x.shape[0]
    cols = n // 2 if kw["epi"] == "silu_mul" else n
    y64, bound = ref.forward(x, **kw)
    outs = {}
    for mode in MODES:
        kern = kernel_of(mode, n, k, rows)
        what = (label, mode, kern, rows)
        out = call(vx, mode, w, x, kw)
        check_padding(out, rows, cols, what)
        again = call(vx, mode, w, x, kw)
        assert np.array_equal(out.view(np.uint32), again.view(np.uint32)), (what, "not reproducible")
        if kw["epi"] == "residual":
            inp = call(vx, mode, w, x, kw, in_place=True)
            check_padding(inp, rows, cols, what)
            assert np.array_equal(inp[:rows, :cols].view(np.uint32), out[:rows, :cols].view(np.uint32)), \
                (what, "in place differs")
        key = f"{kern:11s} {kw['epi']:8s} {'norm+ada' if 'ada' in kw else 'norm' if 'gamma' in kw else '-'}"
        check_bound(out[:rows, :cols], y64, bound, key, what)
        outs[mode] = out[:rows, :cols]
    # outputs the product can show in: rows of x not all zero and, for a residual, not lost below the rounding of res
    live = np.repeat(np.any(x != 0, axis=1)[:, None], cols, 1)
    if kw["epi"] == "residual":
        base = kw["res"].astype(np.float64) + (0.0 if kw["bias"] is None else kw["bias"].astype(np.float64))
        live &= np.abs(y64 - base) > 2.0 ** -20 * np.abs(y64)
    if np.count_nonzero(live) >= 64 and kernel_of("tc", n, k, rows) != kernel_of("simt", n, k, rows):
        assert not np.array_equal(outs["tc"][live].view(np.uint32), outs["simt"][live].view(np.uint32)), \
            (label, rows, "tc and simt gave bitwise the same result")


def _cases():
    out = []
    i = 0
    for name, (n, k, epi, bias, norm, ada, rows_set) in FORMS.items():
        for rows in rows_set:
            sets = [a for a in ACT_SETS if norm_allowed(a) or not norm]
            if epi == "silu_mul":
                sets = [a for a in sets if a != "rows_1e30"]
            out.append(pytest.param(name, rows, sets[i % len(sets)], id=f"{name}-{rows}"))
            i += 1
    return out


@pytest.mark.parametrize("name,rows,aset", _cases())
def test_form_at_production_shape(vx, name, rows, aset):
    n, k, epi, bias, norm, ada, _ = FORMS[name]
    ref = ref_of(name, n, k)
    w = vx.Q4Tensor.from_q4_bytes(ref.raw, (n, k))
    x, kw = layer_inputs(n, k, epi, bias, norm, ada, rows, aset, 7 * rows + k, ones_res=name == "ada2")
    run_case(vx, ref, w, x, kw, f"{name} {aset}")


CROSS_N, CROSS_K = 256, 3072


@pytest.fixture(scope="module")
def cross_ref():
    return LinearRef(weights("signed", CROSS_N, CROSS_K, 21), CROSS_N, CROSS_K)


@pytest.mark.parametrize("rows", [5, 38])
@pytest.mark.parametrize("aset", ACT_SETS)
def test_every_set_and_form(vx, cross_ref, aset, rows):
    """N = 256, K = 3072: every activation set with every epilogue, without a norm, with one and with one and ADA, at
    5 rows (both matvecs) and 38 (both GEMMs)"""
    w = vx.Q4Tensor.from_q4_bytes(cross_ref.raw, (CROSS_N, CROSS_K))
    for epi in ("none", "residual", "silu_mul", "gelu"):
        for norm, ada in ((False, False), (True, False), (True, True)):
            if (norm and not norm_allowed(aset)) or (epi == "silu_mul" and aset == "rows_1e30"):
                continue
            x, kw = layer_inputs(CROSS_N, CROSS_K, epi, epi != "silu_mul", norm, ada, rows, aset, 3 * rows)
            run_case(vx, cross_ref, w, x, kw, f"cross {aset} {epi} norm={norm} ada={ada}")


# ------------------------------------------------------------------------------------- the sum-of-squares hand-off


@pytest.mark.parametrize("rows", [1, 2, 5, 8])
@pytest.mark.parametrize("n_res", [3072, 17, 208])
def test_sum_of_squares_handoff(vx, rows, n_res):
    """A residual call (dec wo: N = 3072, K = 4096; or N = 17 / 208, K = 4192, a partial last tile) writes ssq_out: each
    [ceil(N/16)][rows] partial is the sum of squares of the returned f32 y over its 16 rows (relative 2^-19).  A
    SiLU*up call with norm and ADA (dec w13 at K = N of the first call) then reads it as ssq_in on that y, and meets the
    bound, as does the same call without ssq_in (launch_rmsnorm)."""
    k_res = 4096 if n_res == 3072 else 4192
    r1 = ref_of(f"handoff_wo_{n_res}", n_res, k_res)
    w1 = vx.Q4Tensor.from_q4_bytes(r1.raw, (n_res, k_res))
    x, kw = layer_inputs(n_res, k_res, "residual", False, False, False, rows, "gauss", rows)
    y, parts = call(vx, "tc", w1, x, kw, want_ssq_out=True)
    y = y[:rows, :n_res]
    y64, bound = r1.forward(x, **kw)
    check_bound(y, y64, bound, "matvec_tc  residual ssq_out", ("handoff wo", n_res, rows))
    n_parts = -(-n_res // 16)
    assert parts.shape == (n_parts, rows)
    yp = np.zeros((rows, n_parts * 16))
    yp[:, :n_res] = y.astype(np.float64)
    want = (yp ** 2).reshape(rows, n_parts, 16).sum(2).T
    rel = np.abs(parts.astype(np.float64) - want) / np.maximum(want, 1e-300)
    assert rel.max() <= 2.0 ** -19, (n_res, rows, np.unravel_index(int(np.argmax(rel)), rel.shape), rel.max())

    if n_res != 3072:                                   # 17 and 208 are no K of a Q4 weight: partials only
        return
    n13 = 18432
    r2 = ref_of("dec_w13", n13, n_res)
    w2 = vx.Q4Tensor.from_q4_bytes(r2.raw, (n13, n_res))
    _, kw2 = layer_inputs(n13, n_res, "silu_mul", False, True, True, rows, "gauss", 11 * rows)
    y64, bound = r2.forward(y, **kw2)
    fused = call(vx, "tc", w2, y, kw2, ssq_in=parts)
    plain = call(vx, "tc", w2, y, kw2)
    for label, out in (("ssq_in", fused), ("rmsnorm", plain)):
        check_padding(out, rows, n13 // 2, ("handoff w13", label, rows))
        check_bound(out[:rows, :n13 // 2], y64, bound, f"matvec_tc  silu_mul norm+ada {label}",
                    ("handoff w13", label, n_res, rows))


# ------------------------------------------------------------------------------------------------------ refusals


def test_refusals(vx):
    """vox_q4_linear refuses, with VOX_EINVAL and a reason, every argument combination no kernel can honour"""
    n, k = 256, 128
    w = vx.Q4Tensor.from_q4_bytes(weights("random", n, k, 1), (n, k))
    w_odd = vx.Q4Tensor.from_q4_bytes(weights("random", 17, k, 2), (17, k))
    dev = vx.DeviceBuffer
    x = dev.from_numpy(np.ones((16, k), np.float32))
    y = dev.from_numpy(np.zeros((17, n + PAD), np.float32))
    g = dev.from_numpy(np.ones(k, np.float32))
    b = dev.from_numpy(np.ones(n, np.float32))
    ada_v = dev.from_numpy(np.ones(k, np.float32))
    ada = dev.from_numpy(np.array([ada_v.ptr.value], np.uint64))
    ssq_in = dev.from_numpy(np.ones((k // 16, 2), np.float32))
    ssq_out = dev.from_numpy(np.ones((n // 16, 2), np.float32))
    lib = vx.lib()

    def rc(rows=1, ldy=n, bias=None, res=None, epi=0, gamma=None, ada_p=None, ada_m=1, ssq_in=None, ssq_out=None,
           weight=w, mode=0):
        assert lib.vox_q4_set_matvec_mode(mode) == 0
        try:
            code = lib.vox_q4_linear(weight._h, x.ptr, y.ptr, rows, ldy, bias, res, epi, gamma, EPS, ada_p, ada_m,
                                     ssq_in, ssq_out, None)
            assert lib.vox_dev_sync(0) == 0
            return code, lib.vox_last_error().decode()
        finally:
            lib.vox_q4_set_matvec_mode(0)

    assert rc()[0] == 0
    assert rc(rows=16, gamma=g.ptr, ada_p=ada.ptr, ada_m=16)[0] == 0
    assert rc(rows=2, epi=1, res=y.ptr, gamma=g.ptr, ssq_in=ssq_in.ptr, ssq_out=ssq_out.ptr)[0] == 0
    refused = {
        "rows < 1": dict(rows=0),
        "epi 4": dict(epi=4),
        "epi -1": dict(epi=-1),
        "residual without res": dict(epi=1),
        "res with another epi": dict(res=y.ptr, epi=3),
        "SiLU*up, odd N": dict(epi=2, weight=w_odd, ldy=17),
        "SiLU*up, ldy < N/2": dict(epi=2, ldy=n // 2 - 1),
        "SiLU*up with a bias": dict(epi=2, ldy=n // 2, bias=b.ptr),
        "ldy < N": dict(ldy=n - 1),
        "residual, ldy < N": dict(epi=1, res=y.ptr, ldy=n - 1),
        "ADA without gamma": dict(ada_p=ada.ptr),
        "ada_m < 1": dict(gamma=g.ptr, ada_p=ada.ptr, ada_m=0),
        "ssq_in without gamma": dict(ssq_in=ssq_in.ptr),
        "ssq_out without residual": dict(ssq_out=ssq_out.ptr),
        "ssq_in at 9 rows": dict(rows=9, gamma=g.ptr, ssq_in=ssq_in.ptr),
        "ssq_out at 9 rows": dict(rows=9, epi=1, res=y.ptr, ssq_out=ssq_out.ptr),
        "ssq_in, SIMT matvec": dict(gamma=g.ptr, ssq_in=ssq_in.ptr, mode=1),
        "ssq_out, SIMT matvec": dict(epi=1, res=y.ptr, ssq_out=ssq_out.ptr, mode=3),
    }
    for why, args in refused.items():
        code, msg = rc(**args)
        assert code == 1, (why, code, msg)
        assert msg.startswith("q4_linear:"), (why, msg)
    assert rc()[0] == 0                                 # a refusal leaves the handle usable
