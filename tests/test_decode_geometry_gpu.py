"""The decode step at the production decoder geometry against a float64 reference, with the sliding window biting.

Model: synth.decoder_geometry_config -- the full model's decoder layer (3072, 32:8 x 128 heads, FFN 9216) at 2 layers,
vocabulary 32768 (2048 lm_head tiles), the tiny encoder -- at decoder windows 8192 (never bites), 40 (bites from
position 41 on) and 8 (bites everywhere: 9 keys, so with 4 key chunks of ceil(9/4) = 3 keys the last chunk is empty).

Every stream is teacher-forced (vox_prefill + vox_decode_step(tok=...)) along the ids the model itself produced, and the
logits of the prefill and of every decode step are compared with oracle.model.OracleModel(dtype=float64) at the same
position, fed the GPU's own audio embeddings (the encoder has its own tests):
max |dlogit| <= LOGIT_REL_BOUND * max(1, max |ref|) per step.  tests/test_decode_geometry_ref.py pins that the
reference at window W +- 1 differs from the one at W by far more than that bound at every decode position where the
window bites.

Paths (a 132-SM H100; key chunks per (stream, kv head) NC = min(4, 132 // (8 * rows in the launch))):
  persistent kernel, B = 1, 2, 3, 4, 5, 8 -> token capacities 1, 2, 4, 4, 8, 8; NC 4, 4, 4, 4, 3, 2; wo (64 block pairs)
    and w2 (144) split into K slices from B = 5 on;
  B = 11 -> two launches per step (8 rows, NC 2; then a ragged group of 3 rows on the 8-token instantiation, NC 4);
  mega_off -> per-op launches with the fused single-token attention (decode_attn.cu), B = 1, 3;
  tc_off -> SIMT matvecs and the SIMT attention kernel, B = 1;
  the prefill (38 rows per stream) runs the prefill attention kernel; its last row is compared too.
NC = 1 is not reached at this geometry on 132 SMs.  Each persistent-path step must be exactly one launch per group of 8
rows.  transcribe_streaming (CUDA-graph replay of the step, and eager) is compared at its last step.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes, rel_err
from test_golden_gpu import NEAR_TIE, assert_ids_match

pytestmark = pytest.mark.gpu

WINDOWS = (8192, 40, 8)
SECONDS = 19.5           # 168 positions: the prefill's last row (37) + 130 decode steps
N_STREAMS = 11
MEL_FRAMES = 2700
PREFIX = [1] + [32] * (PREFIX_LEN - 1)


def _mel(i, seconds=SECONDS):
    return omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(seconds, 500 + i)))


class Geometry:
    """One window: the GPU model, the streams' mels, teacher ids and the f64 reference logits of positions 37..S4-1."""

    def __init__(self, vx, window, data=None):
        self.window = window
        self.data = geometry_model_bytes(window) if data is None else data
        self.model = vx.Q4ModelLoader.from_bytes(self.data).load(0, max_batch=N_STREAMS, max_mel_frames=MEL_FRAMES)
        self.vocab = self.model.info["vocab"]
        self.mels = np.concatenate([_mel(i) for i in range(N_STREAMS)])
        emb = self.model.encode_audio(self.mels)                  # [N, S4, D]
        self.S4 = emb.shape[1]
        free = self.model.transcribe_streaming(self.mels)         # greedy ids of positions 37..S4-2 (graph replay)
        self.graph_logits = self.model.debug("logits").reshape(N_STREAMS, self.vocab).copy()   # position S4-2
        self.free = free
        self.seqs = np.concatenate([np.tile(PREFIX, (N_STREAMS, 1)), free], 1).astype(np.int32)   # input token per position
        o64 = OracleModel(self.data, dtype=torch.float64)
        t_embed = omel.time_embedding(6.0, o64.cfg.dec_dim)
        self.ref = np.stack([
            o64.forward_streaming(None, self.seqs[i].tolist(), t_embed, audio_embeds=torch.from_numpy(emb[i]))
            .numpy()[PREFIX_LEN - 1:] for i in range(N_STREAMS)])   # [N, S4 - 37, V] f64

    def teacher_forced(self, B):
        """Streams 0..B-1 teacher-forced: (logits [B, S4-37, V], device argmax per row, launches per decode step)."""
        m = self.model
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        toks = [m.prefill(self.seqs[:B, :PREFIX_LEN])]
        rows = [m.debug("logits").reshape(B, self.vocab).copy()]
        launches = []
        for p in range(PREFIX_LEN, self.S4):
            n0 = m.launch_count()
            toks.append(m.decode_step(tok=self.seqs[:B, p]))
            launches.append(m.launch_count() - n0)
            rows.append(m.debug("logits").reshape(B, self.vocab).copy())
        return np.stack(rows, 1), np.stack(toks, 1), np.array(launches)

    def check(self, what, B, logits, toks=None):
        """Per-step bound against the f64 reference; prints and returns the largest relative error."""
        ref = self.ref[:B] if logits.ndim == 3 else self.ref[:B, -2]
        err = rel_err(logits, ref)
        worst = np.unravel_index(int(np.argmax(err)), err.shape)
        print(f"\n[decode geometry] window {self.window:5d} {what:>9s} B={B:2d}: max |dlogit| / max(1, max|ref|) = "
              f"{err.max():.2e} over {err.size} rows")
        assert err.max() <= LOGIT_REL_BOUND, (what, B, self.window, worst, err.max())
        if toks is not None:   # the device argmax (cross-CTA on the persistent path) == argmax of the logits it read
            assert np.array_equal(toks, logits.argmax(-1)), (what, B)
        return err.max()


@pytest.fixture(scope="module", params=WINDOWS, ids=lambda w: f"window{w}")
def geom(request, vx):
    g = Geometry(vx, request.param)
    yield g
    g.model.close()


@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 8, 11])
def test_persistent_kernel_vs_f64_reference(geom, B):
    geom.model.debug("mega_auto")
    logits, toks, launches = geom.teacher_forced(B)
    geom.check("mega", B, logits, toks)
    # no silent fall-back to per-op launches: exactly one persistent launch per group of 8 rows, every step
    assert np.all(launches == (B + 7) // 8), (B, np.unique(launches))


@pytest.mark.parametrize("path,B", [("mega_off", 1), ("mega_off", 3), ("tc_off", 1)])
def test_per_op_paths_vs_f64_reference(geom, path, B):
    geom.model.debug(path)
    try:
        logits, toks, launches = geom.teacher_forced(B)
    finally:
        geom.model.debug("tc_on" if path == "tc_off" else "mega_auto")
    geom.check(path, B, logits, toks)
    assert np.all(launches > 2 * geom.model.info["dec_layers"])   # per-op launches, not the persistent kernel


def test_graph_replay_and_eager_transcribe_vs_f64_reference(geom):
    """transcribe_streaming replays one captured decode step as a CUDA graph; graph_off launches it eagerly.  Both give
    the ids the teacher forcing followed, and their last step's logits (position S4-2) meet the bound."""
    geom.check("graph", N_STREAMS, geom.graph_logits)
    m = geom.model
    m.debug("graph_off")
    try:
        ids = m.transcribe_streaming(geom.mels)
        last = m.debug("logits").reshape(N_STREAMS, geom.vocab).copy()
    finally:
        m.debug("graph_on")
    assert np.array_equal(ids, geom.free)
    geom.check("eager", N_STREAMS, last)
    # the teacher ids are the GPU's own greedy ids: against the f64 reference they may differ only at near-ties
    for i in range(N_STREAMS):
        r = geom.ref[i, :-1]
        top2 = np.sort(r, -1)[:, -2:]
        bad = np.nonzero(r.argmax(-1) != geom.free[i])[0]
        for j in bad:
            assert top2[j, 1] - top2[j, 0] < NEAR_TIE and r[j, geom.free[i, j]] == top2[j, 0], (i, j)


def test_streaming_pool_sessions_of_different_ages(vx, geom):
    """Three live sessions of different lengths opened at different ticks share one pool: one decoder step carries rows
    at different positions (paged KV).  Each session's ids == the f32 oracle's offline ids (near-tie rule)."""
    o32 = OracleModel(geom.data)
    t_embed = omel.time_embedding(6.0, o32.cfg.dec_dim)
    audios = [omel.peak_normalize(omel.speechlike(s, 600 + i)) for i, s in enumerate((5.0, 7.5, 6.0))]
    golds = []
    for a in audios:
        info = {}
        toks = o32.transcribe_streaming(omel.mel_tensor_from_audio(a), t_embed, info=info)
        golds.append({"tokens": np.array(toks), "margins": np.array(info["margins"]), "second": np.array(info["second"])})
    pool = vx.StreamingPool(geom.model, max_sessions=3, max_seconds=10.0)
    try:
        start = [0, 6, 14]
        sids, fed, got, finished = [None] * 3, [0] * 3, [[], [], []], [False] * 3
        max_rows = 0
        for tick in range(400):
            for i in range(3):
                if tick == start[i]:
                    sids[i] = pool.open()
                if sids[i] is None or finished[i]:
                    continue
                if fed[i] < audios[i].size:
                    pool.push(sids[i], audios[i][fed[i]:fed[i] + 1280])
                    fed[i] += 1280
                else:
                    pool.finish(sids[i])
                    finished[i] = True
            st = pool.tick()
            max_rows = max(max_rows, st["decode_rows"] // max(1, st["decode_steps"]))
            done_all = True
            for i in range(3):
                if sids[i] is None:
                    done_all = False
                    continue
                ids, done = pool.poll(sids[i])
                got[i] += ids
                done_all = done_all and done
            if done_all:
                break
        for i in range(3):
            assert len(got[i]) == len(golds[i]["tokens"]), i
            assert_ids_match(np.array(got[i], np.int32), golds[i], f"window {geom.window} pooled session {i}", geom.model,
                             audio=audios[i])
        assert max_rows >= 3          # the three sessions really shared decoder steps
    finally:
        pool.close()


@pytest.mark.slow
def test_full_size_decode_step_is_one_persistent_launch(vx, full_gguf):
    """The full-size model takes the persistent decode-step kernel for B = 1, 3, 8: one launch per step."""
    m = vx.Q4ModelLoader.from_file(full_gguf).load(0, max_batch=8, max_mel_frames=1400)
    try:
        mels = np.concatenate([_mel(i, 6.0) for i in range(8)])
        for B in (1, 3, 8):
            m.encode_audio(mels[:B])
            m.reset_cache()
            m.prefill(np.tile(PREFIX, (B, 1)).astype(np.int32))
            for _ in range(4):
                n0 = m.launch_count()
                m.decode_step(batch=B)
                assert m.launch_count() - n0 == 1, B
    finally:
        m.close()
