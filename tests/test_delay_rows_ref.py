"""CPU side of per-stream transcription delays (vox_session_set_delays, vox_stream_set_delay).

  * detectability: on the decoder-geometry model (window 40), feeding a stream another delay's ADA scale moves its
    logits by at least 10x the GPU tests' bound (LOGIT_REL_BOUND) at every position tests/test_delay_rows_gpu.py
    compares, for every pair of delays those tests put in one batch -- so a row that reads a neighbour's ADA vector
    cannot pass them;
  * ABI: both entry points report VOX_ECUDA without a device, and their ctypes prototypes match the header.
"""
import ctypes
import itertools
import os
import re

import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the delays (tokens of 80 ms) of the GPU tests' mixed batches: stream i runs at DELAYS[i]
DELAYS = (0.5, 1.0, 2.75, 4.25, 6.0, 8.5, 12.0, 15.75, 20.5, 25.25, 30.0)
SECONDS = 8.0   # per stream: positions 37 (the prefill's last row) .. S4 - 1 are compared


def delay_mel(i, seconds=SECONDS):
    return omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(seconds, 700 + i)))


def test_other_delays_ada_exceeds_logit_bound():
    data = geometry_model_bytes(40)
    o64 = OracleModel(data, dtype=torch.float64)
    mel = delay_mel(0)
    emb = OracleModel(data).encode_audio(mel)
    ids = np.random.default_rng(2).integers(0, o64.cfg.vocab, emb.shape[0])
    ids[:PREFIX_LEN] = [1] + [32] * (PREFIX_LEN - 1)
    logits = {d: o64.forward_streaming(None, ids.tolist(), omel.time_embedding(d, o64.cfg.dec_dim), audio_embeds=emb)
              .numpy()[PREFIX_LEN - 1:] for d in DELAYS}
    worst = None
    for a, b in itertools.combinations(DELAYS, 2):
        for own, other in ((a, b), (b, a)):
            bound = LOGIT_REL_BOUND * np.maximum(1.0, np.abs(logits[own]).max(-1))
            ratio = (np.abs(logits[other] - logits[own]).max(-1) / bound).min()
            worst = ratio if worst is None else min(worst, ratio)
            assert ratio >= 10, (own, other, ratio)
    print(f"\n[delay detectability] {len(DELAYS)} delays, {len(logits[DELAYS[0]])} positions: the closest pair moves the "
          f"logits by {worst:.0f}x the bound")


def _prototype(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "voxtral.h")).read(), flags=re.S)
    m = re.search(r"int32_t\s+" + name + r"\s*\(([^)]*)\)", src)
    return [a.strip() for a in m.group(1).split(",")]


def test_prototypes_match_header(vx):
    from voxtral_mini_realtime_rs_b200 import api
    P = ctypes.c_void_p
    want = {
        "vox_session_set_delays": (["vox_session *s", "const float *delays", "int32_t b"], [P, P, ctypes.c_int32]),
        "vox_stream_set_delay": (["vox_stream_pool *p", "int32_t session", "float delay_tokens"],
                                 [P, ctypes.c_int32, ctypes.c_float]),
    }
    for name, (args, ctypes_args) in want.items():
        assert _prototype(name) == args, name
        restype, argtypes = api._SIGS[name]
        assert restype is ctypes.c_int32 and argtypes == ctypes_args, name


def test_entry_points_report_no_device(vx, have_gpu):
    if have_gpu:
        pytest.skip("GPU present")
    lib = vx.lib()
    d = (ctypes.c_float * 2)(1.0, 6.0)
    assert lib.vox_session_set_delays(None, d, 2) == 4          # VOX_ECUDA
    assert lib.vox_stream_set_delay(None, 0, 6.0) == 4
    assert lib.vox_stream_set_delay(None, -1, float("nan")) == 4  # before the arguments are checked
