"""CPU checks of the phrase-boosting rule (tests/bias_reference.py), the restatement the GPU test holds the device to.

- The brute-force boost over (phrase, j) equals an independently written Aho-Corasick automaton on random phrase sets
  with overlapping phrases, shared prefixes, repeated ids and phrases of length 1 and 16.
- A history capped at its last 15 text ids gives the boosts of the full history.
- The kernel's shortcut -- the greedy id against the offered ids only -- equals the lowest-id argmax of the fully boosted
  vector, on random f32 logits with planted ties.
- Ids below 1000 never change the history.
"""
from collections import deque

import numpy as np
import pytest

import bias_reference as br


class AhoCorasick:
    """Trie of the phrases with failure links.  After reading the history, the node is its longest suffix that is a
    phrase prefix; the offered ids are the trie edges out of that node and every node on its failure chain (the shorter
    suffixes that are prefixes, down to the root).  An edge's boost is the largest boost of the phrases through it."""

    def __init__(self, phrases, betas):
        self.goto = [{}]
        self.depth = [0]
        self.edge_boost = [{}]   # node -> {id: largest boost of a phrase continuing with id there}
        for p, b in zip(phrases, betas):
            node = 0
            for t in p:
                eb = self.edge_boost[node]
                eb[t] = max(eb.get(t, 0.0), float(b))
                if t not in self.goto[node]:
                    self.goto[node][t] = len(self.goto)
                    self.goto.append({})
                    self.depth.append(self.depth[node] + 1)
                    self.edge_boost.append({})
                node = self.goto[node][t]
        self.fail = [0] * len(self.goto)
        q = deque(self.goto[0].values())
        while q:
            u = q.popleft()
            for t, v in self.goto[u].items():
                f = self.fail[u]
                while f and t not in self.goto[f]:
                    f = self.fail[f]
                self.fail[v] = self.goto[f][t] if t in self.goto[f] and self.goto[f][t] != v else 0
                q.append(v)

    def step(self, node, t):
        while node and t not in self.goto[node]:
            node = self.fail[node]
        return self.goto[node].get(t, 0)

    def boosts(self, hist):
        node = 0
        for t in hist:
            node = self.step(node, t)
        out = {}
        while True:
            for t, b in self.edge_boost[node].items():
                out[t] = max(out.get(t, 0.0), b)
            if node == 0:
                return out
            node = self.fail[node]


def random_phrases(rng, n, alphabet, lengths=(1, 16)):
    """n phrases over a small alphabet of text ids (so phrases overlap, share prefixes and repeat ids), with lengths
    1 and 16 always present."""
    ids = br.FIRST_TEXT_ID + rng.choice(5000, size=alphabet, replace=False)
    phrases = []
    for i in range(n):
        L = lengths[i] if i < len(lengths) else int(rng.integers(1, br.MAX_LEN + 1))
        phrases.append([int(x) for x in rng.choice(ids, size=L)])
    # shared prefixes and a phrase that is a prefix of another
    for i in range(min(4, n - 1)):
        k = int(rng.integers(1, len(phrases[i]) + 1))
        phrases.append(phrases[i][:k] + [int(x) for x in rng.choice(ids, size=int(rng.integers(0, 4)))])
    phrases = [p[:br.MAX_LEN] for p in phrases]
    betas = rng.uniform(0.1, 8.0, size=len(phrases)).astype(np.float32)
    return phrases, betas, ids


def history_near(rng, phrases, ids, n):
    """A history built mostly from phrase pieces (so prefixes match), with stray ids in between."""
    h = []
    while len(h) < n:
        if rng.random() < 0.7:
            p = phrases[int(rng.integers(len(phrases)))]
            h += p[:int(rng.integers(0, len(p) + 1))]
        else:
            h.append(int(rng.choice(ids)))
    return h[:n]


@pytest.mark.parametrize("seed", range(12))
def test_brute_force_equals_aho_corasick(seed):
    rng = np.random.default_rng(seed)
    alphabet = [2, 3, 5, 12][seed % 4]
    n = [1, 3, 40, 256][seed % 4]
    phrases, betas, ids = random_phrases(rng, n, alphabet)
    ac = AhoCorasick(phrases, betas)
    for _ in range(60):
        h = history_near(rng, phrases, ids, int(rng.integers(0, 40)))
        assert br.boosts(phrases, betas, h) == ac.boosts(h), (phrases, h)


def test_repeated_ids_and_self_overlap():
    """Phrases whose prefixes are their own suffixes: every partial match is offered at once."""
    a, b = 1001, 1002
    phrases, betas = [[a, a, a, b], [a, b, a, b], [b]], [3.0, 2.0, 0.5]
    ac = AhoCorasick(phrases, betas)
    for h, want in [([], {a: 3.0, b: 0.5}), ([a], {a: 3.0, b: 2.0}), ([a, a], {a: 3.0, b: 2.0}),
                    ([a, a, a], {a: 3.0, b: 3.0}), ([a, b, a], {a: 3.0, b: 2.0}), ([b, b], {a: 3.0, b: 0.5})]:
        assert br.boosts(phrases, betas, h) == want, h
        assert ac.boosts(h) == want, h


@pytest.mark.parametrize("seed", range(6))
def test_history_capped_at_15_gives_the_same_boosts(seed):
    rng = np.random.default_rng(100 + seed)
    phrases, betas, ids = random_phrases(rng, 64, 3 + seed)
    h, capped = [], []
    for t in history_near(rng, phrases, ids, 400):
        h = br.push(h, t)
        capped = br.push(capped, t, br.HIST)
        assert len(capped) <= br.HIST
        assert br.boosts(phrases, betas, h) == br.boosts(phrases, betas, capped)


def test_special_ids_never_enter_the_history():
    rng = np.random.default_rng(7)
    phrases, betas, ids = random_phrases(rng, 16, 4)
    h = [int(x) for x in rng.choice(ids, size=10)]
    for t in [0, 1, 2, 32, 33, 999, 500]:
        assert br.push(h, t) == h
        assert br.push(h, t, br.HIST) == h[-br.HIST:]
    s = br.Stream(phrases, betas)
    s.hist = list(h)
    logits = np.full(int(max(ids)) + 1, -5.0, np.float32)
    logits[32] = 1e6   # a [STREAMING_PAD] that no boost can beat
    assert s.emit(logits) == 32 and s.hist == h


@pytest.mark.parametrize("seed", range(10))
def test_candidate_argmax_equals_full_biased_argmax(seed):
    """Random f32 logits with planted ties: equal logits, equal boosted values, a boosted id tying the greedy one (from
    either side of it), boosts too small to move a value (float32 rounding), and boosts of ids below the greedy one."""
    rng = np.random.default_rng(200 + seed)
    phrases, betas, ids = random_phrases(rng, 48, 6)
    ids = np.array(sorted(set(t for p in phrases for t in p)))
    V = int(ids.max()) + 50
    n_diff = 0
    for trial in range(200):
        logits = rng.normal(0, 3, V).astype(np.float32)
        if trial % 3 == 0:   # a coarse grid: many equal logits
            logits = np.round(logits * 2) / 2
        h = history_near(rng, phrases, list(ids), int(rng.integers(0, 20)))
        off = br.boosts(phrases, betas, h)
        a = br.greedy(logits)
        kind = trial % 5
        cand = sorted(off)
        if cand and kind == 1:   # an offered id at exactly the greedy value after its boost
            t = cand[int(rng.integers(len(cand)))]
            if t != a:
                logits[t] = np.float32(logits[a] - np.float32(off[t]))
                if np.float32(logits[t] + np.float32(off[t])) != logits[a]:
                    logits[t] = np.nextafter(logits[t], np.float32(np.inf))
        elif cand and kind == 2:   # two offered ids at equal boosted values
            t, u = cand[0], cand[-1]
            logits[u] = np.float32(logits[t] + np.float32(off[t]) - np.float32(off[u]))
        elif cand and kind == 3:   # a huge logit: the boost is lost in float32 rounding
            t = cand[0]
            logits[t] = logits[a] = np.float32(3e9)
        elif kind == 4:   # the greedy id tied by an unboosted id above and below
            m = logits.max()
            lo = int(rng.integers(0, 500))
            logits[lo] = m
            logits[V - 1] = m
        a = br.greedy(logits)
        full = br.biased_argmax(logits, off)
        assert br.candidate_argmax(logits, a, off) == full, (seed, trial)
        n_diff += full != a
    assert n_diff > 20   # the boosts do change decisions here


def test_stream_clears_history_on_set():
    s = br.Stream([[1001, 1002]], [50.0])
    logits = np.zeros(1100, np.float32)
    logits[1002] = 0.5   # offered only once 1001 is in the history
    assert s.emit(logits) == 1001 and s.hist == [1001]
    assert s.emit(logits) == 1002 and s.hist == [1001, 1002]
    s.set([[1003]], [1.0])
    assert s.hist == []
