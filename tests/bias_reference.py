"""Phrase boosting (vox_session_set_bias, include/voxtral.h) in plain Python / numpy: the rule the device applies.

A stream's list is phrases p_i (1..16 token ids >= FIRST_TEXT_ID) with boosts b_i > 0.  Its history h is the text ids
(>= FIRST_TEXT_ID) it has emitted since the history was last cleared.  Candidate t gets

    boost(t) = max { b_i : 0 <= j < len_i, the last j ids of h equal p_i[0..j), p_i[j] = t }   (0 when none)

and the emitted id is the argmax of float32(logit(t) + boost(t)), the lowest id winning a tie.
"""
import numpy as np

FIRST_TEXT_ID = 1000
MAX_PHRASES = 256
MAX_LEN = 16
HIST = MAX_LEN - 1   # the longest prefix a phrase can have matched before its last id


def boosts(phrases, betas, hist):
    """{t: boost(t)} by brute force over (phrase, j); hist is the stream's history (a list, oldest first)."""
    out = {}
    for p, b in zip(phrases, betas):
        for j in range(min(len(p) - 1, len(hist)) + 1):
            if list(hist[len(hist) - j:]) == list(p[:j]):
                t = p[j]
                out[t] = max(out.get(t, 0.0), float(b))
    return out


def biased_argmax(logits, offered):
    """The greedy rule on the whole boosted vector: argmax of float32(logit + boost), lowest id first on ties (for rows
    without NaN, which the tests use)."""
    v = np.asarray(logits, np.float32).copy()
    for t, b in offered.items():
        v[t] = np.float32(v[t] + np.float32(b))
    v[np.isnan(v)] = -np.inf
    return int(np.argmax(v))   # the first maximum; an all -inf row gives 0, as on the device


def candidate_argmax(logits, a, offered):
    """The kernel's rule: the greedy id a at its own value against the offered ids only, same order."""
    logits = np.asarray(logits, np.float32)
    la = float(logits[a])
    best, bi = (-np.inf if np.isnan(la) else la), a
    for t, b in offered.items():
        x = float(np.float32(logits[t] + np.float32(b)))
        if x > best or (x == best and t < bi):
            best, bi = x, t
    return bi


def greedy(logits):
    return biased_argmax(logits, {})


def push(hist, t, cap=None):
    """The history after emitting t: text ids join it (the last `cap` kept when cap is given), others leave it as is."""
    if t < FIRST_TEXT_ID:
        return list(hist)
    h = list(hist) + [int(t)]
    return h[-cap:] if cap else h


class Stream:
    """One stream's list and history, stepped along emitted positions."""

    def __init__(self, phrases=(), betas=()):
        self.set(phrases, betas)

    def set(self, phrases, betas):
        self.phrases = [list(map(int, p)) for p in phrases]
        self.betas = [float(b) for b in betas]
        self.hist = []

    def emit(self, logits):
        """The id this stream emits from these logits (greedy when its list is empty), with the history advanced."""
        if not self.phrases:
            return greedy(logits)
        t = candidate_argmax(logits, greedy(logits), boosts(self.phrases, self.betas, self.hist))
        self.hist = push(self.hist, t, HIST)
        return t


def flat(phrases):
    """(ids, lens) in vox_session_set_bias's packing."""
    return [t for p in phrases for t in p], [len(p) for p in phrases]
