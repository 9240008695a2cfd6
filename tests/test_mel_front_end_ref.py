"""CPU checks of the float64 log-mel reference and its error bound (tests/mel_reference.py), which
tests/test_mel_front_end_gpu.py holds the kernel to.

  * The reference's framing equals oracle.mel.reflect_pad's at every short length, and its f32 counterparts -- the
    oracle's f32 FFT and the emulation of the kernel's direct DFT -- lie inside the interval of every output.
  * TIER2_E: on every signal the emulation stays within TIER2_E / 4 of the f64 value wherever the interval is
    narrower than TIER2_WIDTH (the largest seen is about 7e-7).
  * The bound is not vacuous: most outputs of noise, and a good share of speech-like audio, get an interval narrower
    than TIER2_WIDTH.
  * Each planted fault (mel_reference.FAULTS), applied to the emulation, fails one tier on at least one signal of the
    GPU test's set.  drop_last_term (the last window sample is ~6e-5) is seen by the second tier only.
  * The device normalise-and-pad rule equals oracle.mel.peak_normalize + pad_audio bit for bit.
"""
import numpy as np
import pytest

import mel_reference as mr
from oracle import mel as omel

LENGTHS = (160, 199, 160 * 17 + 3, 32000)   # one frame with both pads clamped, one CTA of 17 frames, 2 s
CASES = [(s, n) for s in mr.SIGNALS for n in LENGTHS]


@pytest.fixture(scope="module")
def refs():
    return {c: mr.reference(mr.signal(*c)) for c in CASES}


def test_framing_matches_oracle_reflect_pad():
    rng = np.random.default_rng(5)
    for n in list(range(160, 460)) + [1000, 4003]:
        x = rng.standard_normal(n).astype(np.float32)
        p = omel.reflect_pad(x)
        F = n // 160
        exp = p[np.arange(F)[:, None] * 160 + np.arange(400)[None, :]]
        assert np.array_equal(mr.frame_samples(x), exp), n


def test_f32_oracle_and_emulation_inside_the_bound(refs):
    o = omel.MelSpectrogram()
    worst = 0.0
    for c in CASES:
        x = mr.signal(*c)
        ref = refs[c]
        co = mr.check(o.compute_log(x), ref, e=np.inf)
        ce = mr.check(mr.emulate(x), ref, e=mr.TIER2_E / 4)
        print(f"{c[0]:10s} n={c[1]:6d}: f32 FFT outside {co['outside']}, emulation outside {ce['outside']}, "
              f"emulation worst narrow {ce['worst_narrow']:.2e}, median width {ce['width_median']:.1e}, "
              f"narrow {ce['narrow_frac']:.2f}")
        assert co["inside"], (c, co)
        assert ce["inside"] and ce["tier2"], (c, ce)
        worst = max(worst, ce["worst_narrow"])
    print(f"largest emulation error on narrow outputs {worst:.2e} (TIER2_E {mr.TIER2_E:.0e})")


def test_bound_is_not_vacuous(refs):
    noise = mr.check(mr.emulate(mr.signal("noise", 32000)), refs[("noise", 32000)])
    speech = mr.check(mr.emulate(mr.signal("speech", 32000)), refs[("speech", 32000)])
    print(f"narrow fraction: noise {noise['narrow_frac']:.2f}, speech {speech['narrow_frac']:.2f}; median width: "
          f"noise {noise['width_median']:.1e}, speech {speech['width_median']:.1e}")
    assert noise["narrow_frac"] >= 0.9
    assert speech["narrow_frac"] >= 0.3 and speech["width_median"] < 5e-3


def test_nyquist_bin_has_no_filterbank_weight():
    _, fb = mr.tables()
    assert np.all(fb[:, 200] == 0) and fb[:, 199].max() > 0


@pytest.mark.parametrize("fault", mr.FAULTS)
def test_planted_fault_is_caught(fault, refs):
    caught = []
    for c in CASES:
        r = mr.check(mr.emulate(mr.signal(*c), fault=fault), refs[c])
        if not (r["inside"] and r["tier2"]):
            caught.append((c, r["outside"], r["worst_narrow"]))
    print(f"{fault}: fails {len(caught)} of {len(CASES)} signals, e.g. {caught[:2]}")
    assert caught, fault


def test_device_normalize_pad_rule_matches_oracle():
    rng = np.random.default_rng(2)
    cases = [rng.standard_normal(n).astype(np.float32) * 0.3 for n in (1, 7, 1280, 4003, 16000, 16001)]
    tail = rng.uniform(-0.5, 0.5, 4003).astype(np.float32)
    tail[-1] = 0.75                       # the peak at the last sample, on a tail that is not a multiple of 4
    neg = rng.uniform(-0.5, 0.5, 4000).astype(np.float32)
    neg[1234] = -2.5                      # a negative peak
    cases += [tail, neg, np.zeros(4000, np.float32), np.full(4001, 3e-11, np.float32),
              (rng.standard_normal(999) * 1e3).astype(np.float32)]
    for x in cases:
        assert np.array_equal(mr.normalize_pad(x), omel.pad_audio(omel.peak_normalize(x)))
        assert np.array_equal(mr.normalize_pad(x, normalize=False), omel.pad_audio(x))
