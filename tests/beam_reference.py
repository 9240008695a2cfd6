"""Reference beam search with the selection rule of vox_session_set_beam (include/voxtral.h).

After the prefill the beam list holds the prefix alone, with score 0.  At each emitted position every live beam j offers
its W most likely tokens (descending log-probability, the lower id first on ties); a candidate scores cum[j] + lp.  The
new list is the W best candidates by score descending, then parent rank j ascending, then token id ascending.
"""
import numpy as np
import torch

from oracle.model import PREFIX_LEN, OracleModel


def log_softmax64(logits) -> np.ndarray:
    x = np.asarray(logits, np.float64)
    m = x.max(-1, keepdims=True)
    return x - (m + np.log(np.exp(x - m).sum(-1, keepdims=True)))


def topk_ids(lp, k):
    """The k best ids of a row: descending value, the lower id first on ties."""
    return np.lexsort((np.arange(lp.size), -lp))[:k]


def select(cum, lps, W):
    """One selection.  cum [n_live], lps [n_live][V] -> (parents, tokens, scores) of the W best, in rank order, and the
    margins: the score gaps between neighbouring entries of the W + 1 best candidates."""
    cands = []
    for j, (c, lp) in enumerate(zip(cum, lps)):
        for t in topk_ids(lp, W + 1):
            cands.append((-(c + float(lp[t])), j, int(t)))
    cands.sort()
    best = cands[:W]
    scores = [-c[0] for c in cands[:W + 1]]
    return [c[1] for c in best], [c[2] for c in best], scores[:W], -np.diff(scores)


def beam_search(first_lp, step_lp, n, W):
    """Generic driver: first_lp [V] is the prefix's distribution; step_lp(parent_states, tokens) -> (lps [W][V], states)
    runs one step for the new beams.  Returns ids [W][n], scores [W] in rank order, and the margins of every position."""
    hyps, cum, states = [[]], [0.0], [None]
    lps = [first_lp]
    margins = []
    for i in range(n):
        par, tok, sc, mg = select(cum, lps, W)
        margins.append(mg)
        hyps = [hyps[j] + [t] for j, t in zip(par, tok)]
        cum = sc
        if i + 1 < n:
            lps, states = step_lp([states[j] for j in par], tok)
    return np.array(hyps, np.int32), np.array(cum), margins


def oracle_beam(o: OracleModel, audio_embeds, t_embed, W, record=None):
    """Beam search on the oracle decoder for one stream: one KV cache per beam, the beams of a step batched through
    decoder_forward_batched.  record (optional dict) receives the logits of every evaluated row per position."""
    audio = torch.as_tensor(audio_embeds).to(o.dtype)
    n = audio.shape[0] - PREFIX_LEN
    ada = o.ada_scales(t_embed)
    prefix = [1] + [32] * (PREFIX_LEN - 1)
    cache = o.new_cache()
    h = o.decoder_forward_with_cache(audio[:PREFIX_LEN] + o.embed_tokens(prefix), ada, cache)
    logits0 = o.lm_head(h[-1:]).numpy()
    rows = [logits0]
    pos = [PREFIX_LEN]

    def step(caches, toks):
        caches = [[dict(layer) for layer in c] for c in caches]   # a child shares its parent's history
        p = pos[0]
        x = audio[p:p + 1].repeat(len(toks), 1) + o.embed_tokens(toks)
        hid = o.decoder_forward_batched(x, ada, caches)
        lg = o.lm_head(hid).numpy()
        rows.append(lg)
        pos[0] += 1
        return log_softmax64(lg), caches

    ids, scores, margins = beam_search(log_softmax64(logits0)[0], lambda st, tk: step([cache if s is None else s for s in st], tk),
                                       n, W)
    if record is not None:
        record["logits"] = rows
        record["margins"] = margins
    return ids, scores
