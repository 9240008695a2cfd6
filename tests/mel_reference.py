"""Float64 reference of the log-mel front end (kernels.cu K1: mel_kernel, peak_max_kernel, scale_pad_kernel) with a
derived error bound, and a numpy emulation of the kernel's f32 arithmetic, for tests/test_mel_front_end_ref.py (CPU)
and tests/test_mel_front_end_gpu.py.

Reference.  The frames of the reflect-padded signal (torch.stft center=True, mel.rs:190-205, short signals included)
times the kernel's own f32 Hann window, in float64; np.fft.rfft in float64; power; the kernel's own f32 filterbank
(both widened: they are fixed inputs, checked against the oracle by test_model_gpu.py); log10(max(., 1e-10)), the clamp
at 1.5 - 8 and (x + 4) / 4.

Bound (`reference(...)["lo"], ["hi"]`): an interval per output that the kernel's f32 result must lie in.  With
u = 2^-24 and v_j = w_j x_j the frame's windowed samples, A_f = sum_j |v_j|:
  * each DFT bin's real and imaginary part is off by at most d = (400 + C_TW) u A_f: 400 roundings of the fma
    accumulation (every partial sum is at most A_f), the f32 window product (u A_f) and the twiddle table, whose
    sincospif(2 i / 400) is within 1 ulp (2u) of the value at the rounded argument, itself at most 2 pi u off in angle;
    C_TW = 16 covers these 2 pi + 3 with room;
  * |dP_k| <= 2 |X_k| sqrt(2) d + 2 d^2 + 3u (P_k + ...) for the power re^2 + im^2 of the perturbed bin;
  * the filterbank sum of a row with L bins adds gamma(L) sum fb (P + dP), gamma(L) = L u / (1 - L u);
  * the output lies in [L(acc - dacc), L(acc + dacc)], L the clamped, scaled log10, widened by 2 ulps of log10f and
    half an ulp of the final add (the / 4 is exact).
  Subnormal roundings add an absolute 2^-149 per operation.  No special case is needed for the clamp or the 1e-10
  floor: silent or near-floor outputs get wide intervals (or none: both ends clamp to the same value), loud ones tight.
Second tier: outputs whose interval is narrower than TIER2_WIDTH must be within TIER2_E of the f64 value.  TIER2_E
comes from `emulate`, the kernel's arithmetic restated in numpy f32 (test_mel_front_end_ref.py states the margin).

Device normalise and pad (peak_max_kernel + scale_pad_kernel): `normalize_pad` restates the rule -- scale =
0.95f / max|x| in f32, or 1 when max < 1e-10, one f32 multiply per sample, then pad_audio's zeros.
"""
from __future__ import annotations

import numpy as np

from oracle import mel as omel

F32 = np.float32
U = 2.0 ** -24
TINY = 2.0 ** -149          # absolute error of one subnormal rounding
N_FFT, HOP, N_FREQ, N_MELS, PAD = 400, 160, 201, 128, 200
MEL_FR = 8                  # frames per CTA of mel_kernel
C_TW = 16.0
FLOOR = (-6.5 + 4.0) / 4.0  # the clamped output of a silent frame
TIER2_WIDTH = 1e-3
TIER2_E = 4e-6


def num_frames(n: int) -> int:
    return n // HOP


def reflect_index(src: np.ndarray, n: int, mode: str = "reflect") -> np.ndarray:
    """Signal index of padded position src (may be < 0 or >= n): torch's `reflect` with the clamps of mel.rs:190-205
    for signals shorter than the pad.  mode="symmetric" is numpy's edge-repeating reflection, a planted fault;
    mode="no_clamp" drops the clamps (out-of-range indices are returned as they are)."""
    src = np.asarray(src, np.int64)
    out = src.copy()
    lo, hi = src < 0, src >= n
    if mode == "symmetric":
        out[lo] = -src[lo] - 1
        out[hi] = 2 * n - 1 - src[hi]
    else:
        out[lo] = -src[lo]
        out[hi] = 2 * n - 2 - src[hi]
    if mode != "no_clamp":
        out[lo] = np.minimum(out[lo], max(n - 1, 0))
        out[hi] = np.maximum(out[hi], 0)
    return out


def frame_samples(x: np.ndarray, hop: int = HOP, shift: int = 0, mode: str = "reflect", shift_from: int = 0) -> np.ndarray:
    """[F][400] f32 samples of the frames of x (no window).  shift: frames >= shift_from read `shift` samples later
    (planted faults); an index outside the signal reads 0."""
    x = np.asarray(x, F32)
    n = x.size
    F = num_frames(n)
    t = np.arange(F)[:, None]
    src = t * hop - PAD + np.arange(N_FFT)[None, :] + np.where(t >= shift_from, shift, 0)
    idx = reflect_index(src.reshape(-1), n, mode).reshape(src.shape)
    ok = (idx >= 0) & (idx < n)
    return np.where(ok, x[np.clip(idx, 0, max(n - 1, 0))] if n else F32(0), F32(0)).astype(F32)


def scaled_log(a: np.ndarray) -> np.ndarray:
    """L: the clamped, scaled log10 of filterbank sums (float64)."""
    v = np.log10(np.maximum(a, 1e-10))
    return (np.maximum(v, -6.5) + 4.0) / 4.0


def tables():
    """The oracle's f32 Hann window and filterbank (equal to the kernel's: test_model_gpu.py)."""
    return omel.hann_window(N_FFT), omel.create_mel_filterbank()


def _row_lengths(fb: np.ndarray) -> np.ndarray:
    nz = fb != 0
    first = np.argmax(nz, axis=1)
    last = N_FREQ - 1 - np.argmax(nz[:, ::-1], axis=1)
    return np.where(nz.any(axis=1), last - first + 1, 0)


def reference(x: np.ndarray, window: np.ndarray | None = None, fb: np.ndarray | None = None) -> dict:
    """float64 log-mel [F][128] of signal x and its error interval: {"out", "lo", "hi", "width"}."""
    if window is None or fb is None:
        window, fb = tables()
    w64 = np.asarray(window, F32).astype(np.float64)
    fb64 = np.asarray(fb, F32).astype(np.float64)
    v = frame_samples(x).astype(np.float64) * w64[None, :]
    X = np.fft.rfft(v, axis=1)
    P = X.real ** 2 + X.imag ** 2
    absX = np.sqrt(P)
    A = np.abs(v).sum(axis=1, keepdims=True)
    d = (N_FFT + C_TW) * U * A * (1 + 1e-6) + N_FFT * 2 * TINY
    e = np.sqrt(2.0) * d                                # |complex error| of one bin
    dP0 = 2 * absX * e + e * e
    dP = dP0 + 3 * U * (P + dP0) + 4 * TINY
    L = _row_lengths(fb64)[None, :]
    gamma = L * U / (1 - L * U)
    acc = P @ fb64.T
    dacc = dP @ fb64.T + gamma * ((P + dP) @ fb64.T) + (L + 1) * TINY
    out = scaled_log(acc)
    lo, hi = scaled_log(np.maximum(acc - dacc, 0.0)), scaled_log(acc + dacc)
    # 2 ulps of log10f and half an ulp of the add (both at |log10| >= 8 at least), doubled; / 4 is exact
    lg = np.maximum(np.abs(np.log10(np.maximum(acc + dacc, 1e-10))), 8.0).astype(F32)
    eta = 2 * (2 * np.spacing(lg) + 0.5 * np.spacing(lg + F32(4))).astype(np.float64) / 4
    return {"out": out, "lo": lo - eta, "hi": hi + eta, "width": hi - lo + 2 * eta}


def check(got: np.ndarray, ref: dict, e: float = TIER2_E) -> dict:
    """Both tiers for a [F][128] result: {"inside": all in the interval, "tier2": narrow outputs within e, "worst",
    "worst_narrow", "width_median", "narrow_frac", "outside": count}."""
    got = np.asarray(got, np.float64)
    out = {"outside": 0, "inside": True, "tier2": True, "worst": 0.0, "worst_narrow": 0.0, "width_median": 0.0,
           "narrow_frac": 1.0}
    if got.size == 0:
        return out
    bad = (got < ref["lo"]) | (got > ref["hi"]) | ~np.isfinite(got)
    err = np.abs(got - ref["out"])
    narrow = ref["width"] < TIER2_WIDTH
    out.update(outside=int(bad.sum()), inside=not bad.any(), worst=float(np.nan_to_num(err, nan=np.inf).max()),
               width_median=float(np.median(ref["width"])), narrow_frac=float(narrow.mean()))
    if narrow.any():
        wn = float(np.nan_to_num(err[narrow], nan=np.inf).max())
        out.update(worst_narrow=wn, tier2=wn <= e)
    return out


# ---------------------------------------------------------------------------------------------- kernel emulation
# Two mistakes cannot change any output and so are planted in a form that can:
#  * the twiddle index k j + 1 in both tables turns every bin by the same phase, which the power does not see; the
#    planted fault shifts the cosine index only;
#  * bin 200 (Nyquist) has filterbank weight 0 in every row (test_mel_front_end_ref.py pins this), so losing it changes
#    nothing; the planted fault loses the top two bins, 199 being the highest with weight.
FAULTS = ("hop_161", "window_shift", "symmetric_reflect", "no_short_clamp", "twiddle_plus_one", "no_top_bins",
          "fb_late", "cta_frame7_zero", "slide_base_4", "power_re_only", "drop_last_term")


def _fma(a, b, c):
    """f32 fma (a*b is exact in float64; one rounding to f32 up to a rare double rounding)."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def emulate(x: np.ndarray, window: np.ndarray | None = None, fb: np.ndarray | None = None, fault: str | None = None,
            frame0: int = 0) -> np.ndarray:
    """mel_kernel's arithmetic in numpy f32 -> [F][128]: the f32 window product, the twiddle table sincospif(2 i / 400)
    (correctly rounded at the rounded argument) indexed k j mod 400, fma accumulation in j order, re^2 + im^2 with one
    fma, the filterbank as an fma chain in ascending bin order, log10f, clamp, (v + 4) / 4.  `fault`: one of FAULTS,
    each a mistake the kernel could make (frame0: the first frame of the launch, for the per-CTA fault)."""
    if window is None or fb is None:
        window, fb = tables()
    window = np.asarray(window, F32)
    fb = np.asarray(fb, F32)
    hop = 161 if fault == "hop_161" else HOP
    mode = {"symmetric_reflect": "symmetric", "no_short_clamp": "no_clamp"}.get(fault, "reflect")
    shift = {"window_shift": 1, "slide_base_4": 4}.get(fault, 0)
    shift_from = 8 if fault == "slide_base_4" else 0    # as if the buffer base were wrong from the second CTA on
    n = np.asarray(x).size
    F = num_frames(n)
    sp = frame_samples(x, hop, shift, mode, shift_from)
    v = (sp * window[None, :]).astype(F32)
    if fault == "cta_frame7_zero":
        v[(np.arange(F) - frame0) % MEL_FR == MEL_FR - 1] = 0
    i = np.arange(N_FFT)
    arg = (F32(2.0) * i.astype(F32) / F32(N_FFT)).astype(F32).astype(np.float64)
    ct, st = np.cos(np.pi * arg).astype(F32), np.sin(np.pi * arg).astype(F32)
    k = np.arange(N_FREQ)
    re = np.zeros((F, N_FREQ), F32)
    im = np.zeros((F, N_FREQ), F32)
    terms = N_FFT - 1 if fault == "drop_last_term" else N_FFT
    for j in range(terms):
        idx = (k * j) % N_FFT
        vj = v[:, j:j + 1]
        re = _fma(vj, ct[(idx + 1) % N_FFT if fault == "twiddle_plus_one" else idx][None, :], re)
        im = _fma(-vj, st[idx][None, :], im)
    if fault == "power_re_only":
        pw = (re * re).astype(F32)
    else:
        pw = _fma(re, re, (im * im).astype(F32))
    if fault == "no_top_bins":
        pw[:, N_FREQ - 2:] = 0
    if fault == "fb_late":
        fb = np.concatenate([np.zeros((N_MELS, 1), F32), fb[:, :-1]], axis=1)
    acc = np.zeros((F, N_MELS), F32)
    for j in range(N_FREQ):
        acc = _fma(fb[None, :, j], pw[:, j:j + 1], acc)
    lg = np.log10(np.maximum(acc, F32(1e-10)).astype(np.float64)).astype(F32)
    lg = np.maximum(lg, F32(1.5) - F32(8.0))
    return ((lg + F32(4.0)) / F32(4.0)).astype(F32)


# ---------------------------------------------------------------------------------------------- normalise and pad
def normalize_pad(x: np.ndarray, normalize: bool = True) -> np.ndarray:
    """The device rule of peak_max_kernel + scale_pad_kernel followed by pad_audio: [padded] f32."""
    x = np.asarray(x, F32)
    if normalize and x.size:
        mx = F32(np.max(np.abs(x)))
        if not mx < F32(1e-10):
            x = (x * (F32(0.95) / mx)).astype(F32)
    return omel.pad_audio(x)


# ---------------------------------------------------------------------------------------------- test signals
def signal(name: str, n: int, seed: int = 0) -> np.ndarray:
    """The GPU test's signals, n samples of f32."""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    if name == "silence":
        s = np.zeros(n)
    elif name == "dc":
        s = np.full(n, 0.5)
    elif name == "nyquist":
        s = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    elif name == "impulses":   # at CTA-span boundaries: 1280 k - 200 + {0, 1, 1519}
        s = np.zeros(n)
        for kk in range(0, n // 1280 + 2):
            for o in (0, 1, 1519):
                p = 1280 * kk - 200 + o
                if 0 <= p < n:
                    s[p] = 0.8
    elif name == "chirp":      # 50 Hz -> 7950 Hz over the signal
        T = max(n, 1) / 16000.0
        s = 0.7 * np.sin(2 * np.pi * (50 * t / 16000 + (7900 / (2 * T)) * (t / 16000) ** 2))
    elif name == "speech":
        s = omel.peak_normalize(omel.speechlike(n / 16000 + 0.01, seed=1234 + seed)[:n]).astype(np.float64)
    elif name == "hdr":        # a loud sine and quiet noise: the loud bins' rounding reaches the quiet ones
        s = 0.9 * np.sin(2 * np.pi * 1000.5 * t / 16000) + 1e-4 * rng.standard_normal(n)
    elif name == "noise":
        s = rng.uniform(-1, 1, n)
    elif name == "subnormal":
        s = rng.choice([-1.0, 1.0], n) * rng.uniform(1e-45, 1e-38, n)
    elif name == "loud":       # not normalised
        s = 1e3 * omel.peak_normalize(omel.speechlike(n / 16000 + 0.01, seed=99 + seed)[:n]).astype(np.float64)
    else:
        raise KeyError(name)
    return s.astype(F32)


SIGNALS = ("silence", "dc", "nyquist", "impulses", "chirp", "speech", "hdr", "noise", "subnormal", "loud")
EDGE_LENGTHS = (0, 1, 159, 160, 199, 200, 201, 359, 360, 361)
# frame counts 7, 8, 9, 15, 16, 17 (a CTA's 8 frames, one short, one over) at every residue of n mod 4
FRAME_LENGTHS = tuple(160 * f + r for f in (7, 8, 9, 15, 16, 17) for r in (0, 1, 2, 3))
