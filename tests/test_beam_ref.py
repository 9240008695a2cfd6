"""CPU side of beam search (vox_session_set_beam, vox_session_nbest): the reference selection rule of
tests/beam_reference.py, and the ABI of the new entry points."""
import ctypes
import itertools
import os
import re

import numpy as np
import torch

from beam_reference import beam_search, log_softmax64, oracle_beam
from oracle import mel as omel
from oracle.model import OracleModel
from test_delay_rows_ref import ROOT, _prototype

MAX_BEAM = 8   # VOX_MAX_BEAM, include/voxtral.h


def toy_search(table, n, W):
    """Beam search over a logit table that depends on the previous token: table[prev][t] (prev = -1 row for the first)."""
    lp = log_softmax64(table)
    return beam_search(lp[0], lambda states, toks: (lp[np.array(toks) + 1], [None] * len(toks)), n, W)


def exhaustive(table, n):
    lp = log_softmax64(table)
    out = []
    for seq in itertools.product(range(table.shape[1]), repeat=n):
        prev = [-1] + list(seq[:-1])
        out.append((sum(lp[p + 1][t] for p, t in zip(prev, seq)), seq))
    return out


def test_wide_beam_is_exhaustive():
    rng = np.random.default_rng(0)
    table = rng.normal(size=(3, 2))   # rows: first position, after token 0, after token 1
    n, W = 3, MAX_BEAM                # 2^3 sequences: the beam keeps them all
    ids, scores, _ = toy_search(table, n, W)
    ref = sorted(exhaustive(table, n), key=lambda e: -e[0])
    assert [tuple(r) for r in ids] == [seq for _, seq in ref]
    assert np.allclose(scores, [s for s, _ in ref], rtol=0, atol=1e-12)
    assert np.all(np.diff(scores) <= 0)


def test_tie_order_is_parent_rank_then_token_id():
    table = np.zeros((4, 3))   # every token equally likely: all scores tie
    ids, scores, _ = toy_search(table, 2, 4)
    # candidates (parent rank, id): ranks 0..2 after position 0 hold ids 0, 1, 2; then (0,0) (0,1) (0,2) (1,0)
    assert ids.tolist() == [[0, 0], [0, 1], [0, 2], [1, 0]]
    assert np.all(scores == scores[0])


def test_narrow_beam_keeps_the_best_candidates():
    table = np.log(np.array([[0.5, 0.3, 0.2], [0.1, 0.1, 0.8], [0.9, 0.05, 0.05], [0.4, 0.4, 0.2]]))
    ids, scores, margins = toy_search(table, 2, 2)
    # position 0: 0 (0.5), 1 (0.3); position 1: 0->2 (0.40), 1->0 (0.27) beat 0->0 / 0->1 (0.05)
    assert ids.tolist() == [[0, 2], [1, 0]]
    assert np.allclose(np.exp(scores), [0.40, 0.27])
    assert len(margins) == 2 and all(len(m) == 2 for m in margins)


def test_width_one_is_greedy_and_wider_scores_no_worse(tiny_gguf):
    o = OracleModel(tiny_gguf, dtype=torch.float64)
    mel = omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(4.0, 60)))
    emb = o.encode_audio(mel)
    t = omel.time_embedding(6.0, o.cfg.dec_dim)
    greedy = o.transcribe_streaming(None, t, audio_embeds=emb)
    ids1, s1 = oracle_beam(o, emb, t, 1)
    assert ids1[0].tolist() == list(greedy)
    ids4, s4 = oracle_beam(o, emb, t, 4)
    print(f"\n[beam ref] tiny model, {ids4.shape[1]} positions: greedy {s1[0]:.4f}, W=4 best {s4[0]:.4f}, "
          f"{int((ids4[0] != ids1[0]).sum())} positions differ")
    assert s4[0] >= s1[0] - 1e-9
    assert np.all(np.diff(s4) <= 0)
    assert len({tuple(r) for r in ids4}) == 4


def test_prototypes_match_header(vx):
    from voxtral_mini_realtime_rs_b200 import api
    P, I, S = ctypes.c_void_p, ctypes.c_int32, ctypes.c_size_t
    PI = ctypes.POINTER(ctypes.c_int32)
    want = {
        "vox_session_set_beam": (["vox_session *s", "int32_t width"], [P, I]),
        "vox_session_nbest": (["vox_session *s", "int32_t *ids", "double *scores", "size_t cap", "int32_t *b",
                               "int32_t *w", "int32_t *n"], [P, P, P, S, PI, PI, PI]),
    }
    for name, (args, ctypes_args) in want.items():
        assert _prototype(name) == args, name
        restype, argtypes = api._SIGS[name]
        assert restype is ctypes.c_int32 and argtypes == ctypes_args, name
    hdr = open(os.path.join(ROOT, "include", "voxtral.h")).read()
    assert re.search(r"#define VOX_MAX_BEAM (\d+)", hdr).group(1) == str(MAX_BEAM)


def test_null_handles_are_refused(vx):
    lib = vx.lib()
    assert lib.vox_session_set_beam(None, 2) == 1   # VOX_EINVAL: no session
    assert lib.vox_session_nbest(None, None, None, 0, None, None, None) == 1
