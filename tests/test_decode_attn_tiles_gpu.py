"""The persistent decode kernel's attention phase over many K/V tiles, against a float64 reference, at the production
decoder geometry (synth.decoder_geometry_config: G = 4 query heads per kv head, head dim 128).

The attention phase (decode_mega.cu, MG_ATTN) walks each key chunk in tiles of KT keys with an online softmax; KT and the
chunk count NC follow the rows of the launch (tests/test_decode_attn_tiles_ref.TILING).  Streams of 150 s of
speechlike audio give 984 positions, so at window 8192 every chunk of position 900 and later holds 3 tiles or more at
every batch size.  Window 383 gives 384 keys: chunks end in a full tile at B = 1, 3, 4 and 8.  Window 400 gives 401 keys:
chunks end in a short tail of 5 (B = 1, 3, 4), 9 (B = 8), 37 (B = 2) or 38 keys (B = 5).

Every stream is teacher-forced along the GPU's own greedy ids (as tests/test_decode_geometry_gpu.py does) and every
step's logits are compared with OracleModel(dtype=float64) fed the GPU's audio embeddings:
max |dlogit| <= LOGIT_REL_BOUND * max(1, max |ref|).  Paths: the persistent kernel at B = 1, 2, 3, 5, 8 (one launch per
step) and B = 11 at window 8192 (8 + 3 rows, two launches), and the per-op cross-checks mega_off (B = 1, 3) and tc_off
(B = 1).  debug("mega_attn") reports the tiling of each launch of the last step; the test asserts the tile counts it
claims from it, so a change of KT or NC fails here instead of quietly testing less.

The ring instantiation: an unbounded StreamingPool on the window-400 model with 1, 3 and 8 sessions of the same audio.
Its KV ring of 30 pages (480 positions) wraps once within the 984 positions.  Each emitted token's top-k
log-probabilities are compared with log_softmax of the f64 reference run on that session's own embeddings and ids,
within score_bound (tests/test_token_scores_ref.py).

tests/test_decode_attn_tiles_ref.py pins that the reference's schedule equals the kernel's and that the kernel mistakes
this test is meant to catch move the logits far past the bound at these windows and positions.
"""
import time

import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_attn_tiles_ref import RING_POSITIONS, TILING, chunk_tiles
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes
from test_token_scores_ref import MAX_TOP_K, log_softmax64, score_bound

pytestmark = pytest.mark.gpu

WINDOWS = (8192, 383, 400)
SECONDS = 150.0            # 15 746 mel frames -> 984 positions: the prefill's last row (37) + 946 decode steps
MEL_FRAMES = 15800         # S_max = frames / 4 stays within the encoder's 4096-row RoPE table
PREFIX = [1] + [32] * (PREFIX_LEN - 1)
RING_PAGES = RING_POSITIONS // 16


def _audio(i):
    return omel.peak_normalize(omel.speechlike(SECONDS, 700 + i))


def _f64_logits(o64, emb, seq):
    """f64 reference logits of positions 37 .. len(seq) - 1 of one stream, as float32 (plus max |logit| per row in f64):
    the f32 rounding is ~1e-7 relative, far below the bound."""
    t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
    ref = o64.forward_streaming(None, list(seq), t_embed, audio_embeds=torch.from_numpy(emb)).numpy()[PREFIX_LEN - 1:]
    return ref.astype(np.float32), np.abs(ref).max(-1)


class LongStreams:
    """One window: the GPU model, the streams' mels, teacher ids and the f64 reference logits of positions 37..S4-1."""

    def __init__(self, vx, window):
        self.window = window
        self.n = 11 if window == 8192 else 8
        self.data = geometry_model_bytes(window)
        self.model = vx.Q4ModelLoader.from_bytes(self.data).load(0, max_batch=self.n, max_mel_frames=MEL_FRAMES)
        self.vocab = self.model.info["vocab"]
        self.mels = np.concatenate([omel.mel_tensor_from_audio(_audio(i)) for i in range(self.n)])
        emb = self.model.encode_audio(self.mels)                  # [N, S4, D]
        self.S4 = emb.shape[1]
        free = self.model.transcribe_streaming(self.mels)         # greedy ids of positions 37..S4-2
        self.seqs = np.concatenate([np.tile(PREFIX, (self.n, 1)), free], 1).astype(np.int32)
        t0 = time.time()
        self.o64 = OracleModel(self.data, dtype=torch.float64)
        refs = [_f64_logits(self.o64, emb[i], self.seqs[i]) for i in range(self.n)]
        self.ref = np.stack([r[0] for r in refs])                 # [N, S4 - 37, V]
        self.ref_max = np.stack([r[1] for r in refs])
        print(f"\n[attention tiles] window {window}: f64 reference of {self.n} streams x {self.S4} positions in "
              f"{time.time() - t0:.0f} s")

    def teacher_forced(self, B):
        """Streams 0..B-1 teacher-forced; checks every step on the fly.  Returns (largest relative logit error, launches
        per decode step, debug("mega_attn") of the last step)."""
        m = self.model
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        toks = m.prefill(self.seqs[:B, :PREFIX_LEN])
        worst, launches = self._check_row(0, B, toks), []
        for p in range(PREFIX_LEN, self.S4):
            n0 = m.launch_count()
            toks = m.decode_step(tok=self.seqs[:B, p])
            launches.append(m.launch_count() - n0)
            worst = max(worst, self._check_row(p - PREFIX_LEN + 1, B, toks))
        return worst, np.array(launches), m.debug("mega_attn")

    def _check_row(self, r, B, toks):
        logits = self.model.debug("logits").reshape(B, self.vocab).astype(np.float64)
        err = np.abs(logits - self.ref[:B, r]).max(-1) / np.maximum(1.0, self.ref_max[:B, r])
        pos = PREFIX_LEN - 1 + r
        assert err.max() <= LOGIT_REL_BOUND, (self.window, B, pos, int(np.argmax(err)), err.max())
        # the device argmax (cross-CTA on the persistent path) == argmax of the logits it read
        assert np.array_equal(np.asarray(toks).reshape(-1)[:B], logits.argmax(-1)), (self.window, B, pos)
        return float(err.max())


@pytest.fixture(scope="module", params=WINDOWS, ids=lambda w: f"window{w}")
def long_streams(request, vx):
    g = LongStreams(vx, request.param)
    yield g
    g.model.close()


def _tiling_claims(window, B, S4, launches):
    """Checks the readout of the last step (position S4 - 1) against TILING and the tile counts this module claims;
    returns a description per launch."""
    assert launches is not None and launches.size % 4 == 0, launches
    groups = launches.reshape(-1, 4).astype(int)
    assert groups[:, 0].tolist() == [min(8, B - b0) for b0 in range(0, B, 8)], groups
    out = []
    for rows, MT, KT, NC in groups.tolist():
        assert (KT, NC) == TILING[rows], ("attention tiling changed: update TILING and the pins", rows, KT, NC)
        tiles = [t for t in chunk_tiles(S4 - 1, window, NC, KT) if t]
        if window == 8192:
            assert min(map(len, tiles)) >= 3, (rows, tiles)
        elif window == 383 and rows in (1, 3, 4, 8):
            assert all(t[-1] == KT for t in tiles), (rows, tiles)              # full final tiles
        elif window == 400:
            assert any(len(t) > 1 and t[-1] < KT for t in tiles), (rows, tiles)   # a short tail after full tiles
        out.append(f"{rows} rows: KT {KT}, NC {NC}, tiles per chunk {[len(t) for t in tiles]}, last tiles "
                   f"{[t[-1] for t in tiles]}")
    return "; ".join(out)


@pytest.mark.parametrize("B", [1, 2, 3, 5, 8, 11])
def test_persistent_kernel_long_vs_f64_reference(long_streams, B):
    g = long_streams
    if B > g.n:
        pytest.skip("11 streams only at window 8192")
    g.model.debug("mega_auto")
    worst, launches, tiling = g.teacher_forced(B)
    print(f"\n[attention tiles] window {g.window:5d} mega B={B:2d}: max |dlogit| / max(1, max|ref|) = {worst:.2e} over "
          f"{g.S4 - PREFIX_LEN + 1} steps; {_tiling_claims(g.window, B, g.S4, tiling)}")
    # no silent fall-back to per-op launches: exactly one persistent launch per group of 8 rows, every step
    assert np.all(launches == (B + 7) // 8), (B, np.unique(launches))


@pytest.mark.parametrize("path,B", [("mega_off", 1), ("mega_off", 3), ("tc_off", 1)])
def test_per_op_paths_long_vs_f64_reference(long_streams, path, B):
    g = long_streams
    g.model.debug(path)
    try:
        worst, launches, tiling = g.teacher_forced(B)
    finally:
        g.model.debug("tc_on" if path == "tc_off" else "mega_auto")
    print(f"\n[attention tiles] window {g.window:5d} {path} B={B}: max |dlogit| / max(1, max|ref|) = {worst:.2e}")
    assert tiling is None                                                    # no persistent launch in the last step
    assert np.all(launches > 2 * g.model.info["dec_layers"])                # per-op launches, not the persistent kernel


def _pool_run(vx, model, audios):
    """Unbounded pool, every session opened at tick 0 and fed 2 s per tick: (ids, top ids, top log-probabilities, audio
    embeddings, session infos, largest KV page count) per session."""
    pool = vx.StreamingPool(model, max_sessions=len(audios), max_seconds=None)
    try:
        pool.set_top_k(MAX_TOP_K)
        n = len(audios)
        sids = [pool.open() for _ in range(n)]
        fed, finished = [0] * n, [False] * n
        ids, tops, lps, embs = ([[] for _ in range(n)] for _ in range(4))
        max_pages = 0
        for _ in range(10000):
            for i in range(n):
                if fed[i] < audios[i].size:
                    pool.push(sids[i], audios[i][fed[i]:fed[i] + 32000])
                    fed[i] += 32000
                elif not finished[i]:
                    pool.finish(sids[i])
                    finished[i] = True
            pool.tick()
            done_all = True
            for i in range(n):
                got, done, t, l = pool.poll(sids[i], scores=True)
                ids[i] += got
                tops[i].append(t)
                lps[i].append(l)
                info = pool.session_info(sids[i])
                have = sum(e.shape[0] for e in embs[i])
                if info["audio_embeds"] > have:     # the buffers slide: collect the embeddings as they appear
                    embs[i].append(pool.audio_embeds(sids[i], first=have, n=info["audio_embeds"] - have))
                max_pages = max(max_pages, info["kv_pages"])
                done_all = done_all and done
            if done_all:
                break
        infos = [pool.session_info(s) for s in sids]
        return ids, [np.concatenate(t) for t in tops], [np.concatenate(l) for l in lps], \
            [np.concatenate(e) for e in embs], infos, max_pages
    finally:
        pool.close()


@pytest.fixture(scope="module")
def ring_refs():
    """f64 reference log-probabilities (stored as f32) and score bounds per (embeddings, ids) of a pooled session:
    sessions of the same audio in the 1-, 3- and 8-session pools share one reference when their embeddings and ids are
    identical."""
    return {}


@pytest.mark.parametrize("n_sessions", [1, 3, 8])
def test_ring_instantiation_scores_vs_f64_reference(vx, long_streams, ring_refs, n_sessions):
    g = long_streams
    if g.window != 400:
        pytest.skip("the ring instantiation runs on the window-400 model")
    audios = [_audio(i) for i in range(n_sessions)]
    t0 = time.time()
    ids, tops, lps, embs, infos, max_pages = _pool_run(vx, g.model, audios)
    t_pool, t_ref, worst = time.time() - t0, 0.0, 0.0
    assert max_pages == RING_PAGES
    for i in range(n_sessions):
        n = len(ids[i])
        assert n > 900 and tops[i].shape == (n, MAX_TOP_K), (i, n, tops[i].shape)
        assert infos[i]["decoder_positions"] > RING_POSITIONS                # the KV ring wrapped
        assert infos[i]["first_audio_embed"] > 0                             # and the embedding buffer slid
        assert embs[i].shape[0] >= PREFIX_LEN - 1 + n, (embs[i].shape, n)
        assert tops[i][:, 0].tolist() == ids[i]
        seq = PREFIX + ids[i][:-1]                                           # the session's own ids, teacher-forced
        emb = np.ascontiguousarray(embs[i][:len(seq)])
        key = (emb.tobytes(), tuple(seq))
        if key not in ring_refs:
            t1 = time.time()
            ref, _ = _f64_logits(g.o64, emb, seq)
            ref = ref.astype(np.float64)
            ring_refs[key] = (log_softmax64(ref).astype(np.float32), score_bound(ref))   # f32: ~1e-6 of ~2e-4
            t_ref += time.time() - t1
        lsm, bound = ring_refs[key]
        err = np.abs(lps[i] - np.take_along_axis(lsm, tops[i], -1)).max(-1) / bound
        worst = max(worst, float(err.max()))
        assert err.max() <= 1.0, (n_sessions, i, int(np.argmax(err)) + PREFIX_LEN - 1, err.max())
    print(f"\n[attention tiles] ring, window 400, {n_sessions} sessions x {infos[0]['decoder_positions']} positions: "
          f"max |dlogprob| = {worst:.2f} x bound; pool {t_pool:.0f} s, new f64 references {t_ref:.0f} s")
