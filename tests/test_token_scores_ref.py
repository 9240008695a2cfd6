"""CPU side of token confidences (vox_session_set_top_k, vox_session_token_scores, vox_stream_poll_scored).

  * the bound: tests/test_token_scores_gpu.py accepts a log-probability within SCORE_REL_BOUND * max(1, max |f64 logit|)
    of log_softmax of the float64 reference.  logsumexp is 1-Lipschitz in the max norm, so logits within LOGIT_REL_BOUND
    (the decode tests' bound) give log-probabilities within twice that;
  * detectability: on the decoder-geometry model (window 40), along a teacher-forced sequence of two streams:
      - the scores of the neighbouring output position move the top-1 log-probability by at least 10x that bound at
        every position;
      - a neighbouring row's or step's logsumexp moves it by 10x the bound at some positions only (this model's
        logsumexp varies little: median 5x), but by at least 50x OWN_LOGITS_TOL at 90 % of the positions -- the
        tolerance at which the GPU tests compare the kernel with a float64 reduction of the GPU's own logits, row by
        row and step by step.
    So a mis-indexed buffer cannot pass them;
  * ABI: the entry points refuse null handles (VOX_EINVAL), and their ctypes prototypes match the header.
"""
import ctypes
import os
import re

import numpy as np
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes
from test_delay_rows_ref import ROOT, _prototype, delay_mel

# per emitted token: |GPU log-probability - f64 log_softmax| <= SCORE_REL_BOUND * max(1, max |f64 logit|)
SCORE_REL_BOUND = 2 * LOGIT_REL_BOUND
# the kernel alone: |GPU log-probability - float64 log_softmax of the GPU's own logits| <= OWN_LOGITS_TOL
OWN_LOGITS_TOL = 1e-5
MAX_TOP_K = 8   # VOX_MAX_TOP_K, include/voxtral.h


def log_softmax64(logits) -> np.ndarray:
    x = np.asarray(logits, np.float64)
    m = x.max(-1, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(-1, keepdims=True)))


def score_bound(ref_logits) -> np.ndarray:
    """Per row: the largest accepted |log-probability error|."""
    return SCORE_REL_BOUND * np.maximum(1.0, np.abs(np.asarray(ref_logits, np.float64)).max(-1))


def ref_topk(logits, k):
    """(ids, log-probabilities) [..., k] in float64: descending logit, the lower id first on equal logits."""
    x = np.asarray(logits, np.float64)
    order = np.lexsort((np.broadcast_to(np.arange(x.shape[-1]), x.shape), -x), axis=-1)[..., :k]
    return order.astype(np.int32), np.take_along_axis(log_softmax64(x), order, -1)


def test_ref_topk_orders_ties_by_id():
    ids, lp = ref_topk(np.array([[0.0, 2.0, 1.0, 2.0, 2.0]]), 4)
    assert ids.tolist() == [[1, 3, 4, 2]]
    assert np.all(np.diff(lp) <= 0)


def test_misindexed_scores_exceed_bound():
    data = geometry_model_bytes(40)
    o64 = OracleModel(data, dtype=torch.float64)
    o32 = OracleModel(data)
    t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
    rows = []
    for i in range(2):   # two streams of one batch
        emb = o32.encode_audio(delay_mel(i))
        ids = np.random.default_rng(10 + i).integers(0, o64.cfg.vocab, emb.shape[0])
        ids[:PREFIX_LEN] = [1] + [32] * (PREFIX_LEN - 1)
        rows.append(o64.forward_streaming(None, ids.tolist(), t_embed, audio_embeds=emb).numpy()[PREFIX_LEN - 1:])
    n = min(len(r) for r in rows)
    logits = np.stack([r[:n] for r in rows])             # [2][positions][vocab]: the prefill's last row, then each step
    x = logits.max(-1)
    lse = x - log_softmax64(logits).max(-1)               # logsumexp per (row, position)
    top1 = x - lse                                        # the top-1 log-probability
    bound = score_bound(logits)
    step_bound = np.minimum(bound[:, 1:], bound[:, :-1])
    moved = {   # |wrong - right top-1 log-probability|, with the bound of the row it is compared at
        "neighbouring row's logsumexp": (np.abs(lse[::-1] - lse), bound),
        "neighbouring step's logsumexp": (np.abs(lse[:, 1:] - lse[:, :-1]), step_bound),
        "off-by-one output position": (np.abs(top1[:, 1:] - top1[:, :-1]), step_bound),
    }
    for what, (d, b) in moved.items():
        r = d / b
        print(f"\n[score detectability] {what}: {r.size} positions, moves the top-1 log-probability by "
              f"{r.min():.2f} .. {r.max():.0f}x the f64 bound (median {np.median(r):.1f}x), and by >= "
              f"{np.percentile(d, 10) / OWN_LOGITS_TOL:.0f}x the own-logits tolerance at 90 % of them")
        assert r.max() >= 10, what                                  # the f64 comparison fails on it
        assert np.percentile(d, 10) >= 50 * OWN_LOGITS_TOL, what    # so does the own-logits one, nearly everywhere
    # a shifted position reads another token's scores altogether
    assert (moved["off-by-one output position"][0] / step_bound).min() >= 10


def test_prototypes_match_header(vx):
    from voxtral_mini_realtime_rs_b200 import api
    P, I, S = ctypes.c_void_p, ctypes.c_int32, ctypes.c_size_t
    PI, PS = ctypes.POINTER(ctypes.c_int32), ctypes.POINTER(ctypes.c_size_t)
    want = {
        "vox_session_set_top_k": (["vox_session *s", "int32_t k"], [P, I]),
        "vox_session_token_scores": (["vox_session *s", "int32_t *top_ids", "float *top_logprobs", "size_t cap",
                                      "int32_t *b", "int32_t *n", "int32_t *k"], [P, P, P, S, PI, PI, PI]),
        "vox_stream_pool_set_top_k": (["vox_stream_pool *p", "int32_t k"], [P, I]),
        "vox_stream_poll_scored": (["vox_stream_pool *p", "int32_t session", "int32_t *ids", "int32_t *top_ids",
                                    "float *top_logprobs", "size_t cap", "size_t *n", "int32_t *done"],
                                   [P, I, P, P, P, S, PS, PI]),
    }
    for name, (args, ctypes_args) in want.items():
        assert _prototype(name) == args, name
        restype, argtypes = api._SIGS[name]
        assert restype is ctypes.c_int32 and argtypes == ctypes_args, name
    hdr = open(os.path.join(ROOT, "include", "voxtral.h")).read()
    assert re.search(r"#define VOX_MAX_TOP_K (\d+)", hdr).group(1) == str(MAX_TOP_K)


def test_null_handles_are_refused(vx):
    lib = vx.lib()
    n = ctypes.c_size_t()
    assert lib.vox_session_set_top_k(None, 1) == 1            # VOX_EINVAL: no session
    assert lib.vox_session_token_scores(None, None, None, 0, None, None, None) == 1
    assert lib.vox_stream_pool_set_top_k(None, 1) == 1
    assert lib.vox_stream_poll_scored(None, 0, None, None, None, 0, ctypes.byref(n), None) == 1
