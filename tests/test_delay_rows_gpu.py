"""Streams at different transcription delays in one batched decode step (vox_session_set_delays, vox_stream_set_delay).

The delay only changes the ADA scale on the FFN-norm input of every decoder layer.  Rows at different delays read their
own stream's ADA vectors inside the kernels (persistent kernel, tensor-core matvec, wgmma operand split, RMSNorm), so
the step still sweeps the weights once.  Model: the decoder-geometry model (synth.decoder_geometry_config) at decoder
windows 40 and 8192, 11 streams, stream i at DELAYS[i].  Every stream is teacher-forced along the GPU's own greedy ids
and each row's logits are compared with OracleModel(dtype=float64) at that row's delay (the prefill's last row and every
decode step), with the bound LOGIT_REL_BOUND.  tests/test_delay_rows_ref.py pins that another delay's ADA vector moves
the logits by far more than that bound.
"""
import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_decode_geometry_ref import LOGIT_REL_BOUND, geometry_model_bytes, rel_err
from test_delay_rows_ref import DELAYS, delay_mel
from test_golden_gpu import assert_ids_match

pytestmark = pytest.mark.gpu

N = len(DELAYS)
MEL_FRAMES = 2000
PREFIX = [1] + [32] * (PREFIX_LEN - 1)
VOX_EINVAL = 1   # include/voxtral.h


class Mixed:
    """One window: the model, the streams' mels, teacher ids under mixed delays and the f64 reference per stream."""

    def __init__(self, vx, window):
        self.window = window
        self.data = geometry_model_bytes(window)
        self.model = m = vx.Q4ModelLoader.from_bytes(self.data).load(0, max_batch=N, max_mel_frames=MEL_FRAMES)
        self.vocab = m.info["vocab"]
        self.mels = np.concatenate([delay_mel(i) for i in range(N)])
        m.set_delays(DELAYS)
        emb = m.encode_audio(self.mels)
        self.S4 = emb.shape[1]
        free = m.transcribe_streaming(self.mels)
        self.seqs = np.concatenate([np.tile(PREFIX, (N, 1)), free], 1).astype(np.int32)
        o64 = OracleModel(self.data, dtype=torch.float64)
        self.ref = np.stack([
            o64.forward_streaming(None, self.seqs[i].tolist(), omel.time_embedding(DELAYS[i], o64.cfg.dec_dim),
                                  audio_embeds=torch.from_numpy(emb[i])).numpy()[PREFIX_LEN - 1:] for i in range(N)])

    def teacher_forced(self, B, steps=None):
        m = self.model
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        toks = [m.prefill(self.seqs[:B, :PREFIX_LEN])]
        rows = [m.debug("logits").reshape(B, self.vocab).copy()]
        launches = []
        for p in range(PREFIX_LEN, self.S4 if steps is None else PREFIX_LEN + steps):
            n0 = m.launch_count()
            toks.append(m.decode_step(tok=self.seqs[:B, p]))
            launches.append(m.launch_count() - n0)
            rows.append(m.debug("logits").reshape(B, self.vocab).copy())
        return np.stack(rows, 1), np.stack(toks, 1), np.array(launches)

    def check(self, what, B, logits, toks=None):
        ref = self.ref[:B, :logits.shape[1]]
        err = rel_err(logits, ref)
        print(f"\n[mixed delays] window {self.window:5d} {what:>9s} B={B:2d}: max |dlogit| / max(1, max|ref|) = "
              f"{err.max():.2e} over {err.size} rows")
        assert err.max() <= LOGIT_REL_BOUND, (what, B, self.window, np.unravel_index(int(np.argmax(err)), err.shape))
        if toks is not None:
            assert np.array_equal(toks, logits.argmax(-1)), (what, B)


@pytest.fixture(scope="module", params=(40, 8192), ids=lambda w: f"window{w}")
def mixed(request, vx):
    g = Mixed(vx, request.param)
    g.model.set_delays(DELAYS)
    yield g
    g.model.close()


@pytest.mark.parametrize("B", [2, 3, 5, 8, 11])
def test_persistent_kernel_mixed_delays(mixed, B):
    mixed.model.debug("mega_auto")
    logits, toks, launches = mixed.teacher_forced(B)
    mixed.check("mega", B, logits, toks)
    assert np.all(launches == (B + 7) // 8), (B, np.unique(launches))   # one weight sweep per group of 8 rows


@pytest.mark.parametrize("path,B", [("mega_off", 3), ("mega_off", 11), ("tc_off", 3)])
def test_per_op_paths_mixed_delays(mixed, path, B):
    """mega_off at 3 rows: the tensor-core matvec's per-row staging; at 11 rows the decode rows take the wgmma GEMM (per-row
    operand split).  tc_off: the per-row RMSNorm ahead of the SIMT matvec."""
    mixed.model.debug(path)
    try:
        logits, toks, launches = mixed.teacher_forced(B)
    finally:
        mixed.model.debug("tc_on" if path == "tc_off" else "mega_auto")
    mixed.check(path, B, logits, toks)
    assert np.all(launches > 2 * mixed.model.info["dec_layers"])


@pytest.mark.parametrize("gemm", ["gemm_tc", "gemm_simt"])
def test_prefill_mixed_delays(mixed, gemm):
    """The 11 x 38-row prefill: per-row wgmma operand split, or per-row RMSNorm ahead of the SIMT GEMM."""
    mixed.model.debug(gemm)
    try:
        logits, toks, _ = mixed.teacher_forced(N, steps=0)
    finally:
        mixed.model.debug("gemm_tc")
    mixed.check(f"prefill {gemm[5:]}", N, logits, toks)


@pytest.mark.parametrize("path", ["mega_auto", "mega_off"])
def test_one_delay_via_set_delays_equals_set_delay(mixed, path):
    """set_delays([d] * B) after another delay: bitwise the logits, ids and launch counts of set_delay(d)."""
    m, B, d = mixed.model, 5, 12.0
    m.debug(path)
    try:
        m.set_delay(d)
        a = mixed.teacher_forced(B, steps=6)
        m.set_delay(30.0)                    # every stream's set now holds delay 30 ...
        mixed.teacher_forced(B, steps=1)
        m.set_delays([d] * B)                # ... and is rewritten with delay 12
        b = mixed.teacher_forced(B, steps=6)
    finally:
        m.debug("mega_auto")
        m.set_delays(DELAYS)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_graph_replay_follows_delay_changes(mixed):
    """transcribe_streaming replays a captured decode step.  Between consecutive graph transcriptions at the same B and
    length, set_delay -> set_delays -> set_delays (other values) -> set_delay only rewrite the streams' ADA sets, which
    the replayed step reads in place.  Each stream's ids equal the eager transcription and the B = 1 transcription at that
    stream's delay, both run afterwards without graphs."""
    m, B = mixed.model, 4
    mels = mixed.mels[:B]
    o32 = OracleModel(mixed.data)
    golds = {}

    def gold(i, delay):   # the f32 oracle's ids with their top-2 margins (the near-tie rule of assert_ids_match)
        if (i, delay) not in golds:
            info = {}
            toks = o32.transcribe_streaming(mels[i:i + 1], omel.time_embedding(delay, o32.cfg.dec_dim), info=info)
            golds[i, delay] = {"tokens": np.array(toks), "margins": np.array(info["margins"]),
                               "second": np.array(info["second"])}
        return golds[i, delay]

    phases = [[6.0] * B, [0.5, 6.0, 12.0, 30.0], [30.0, 2.75, 0.5, 12.0], [12.0] * B]

    def apply(per):
        m.set_delay(per[0]) if len(set(per)) == 1 else m.set_delays(per)

    try:
        graph = []
        for per in phases:                   # graph replay only, back to back at B = 4
            apply(per)
            graph.append(m.transcribe_streaming(mels))
        m.debug("graph_off")
        for per, g in zip(phases, graph):
            apply(per)
            assert np.array_equal(g, m.transcribe_streaming(mels)), per
            for i in range(B):
                m.set_delay(per[i])   # (assert_ids_match teacher-forces a near-tie's remainder at B = 1)
                one = np.asarray(m.transcribe_streaming(mels[i:i + 1]), np.int32)
                what = f"window {mixed.window} delays {per} stream {i}"
                assert_ids_match(g[i], gold(i, per[i]), what + " (batched, graph)", m, mel=mels[i:i + 1])
                assert_ids_match(one, gold(i, per[i]), what + " (B = 1)", m, mel=mels[i:i + 1])
    finally:
        m.debug("graph_on")
        m.set_delays(DELAYS)


def _run_pool(vx, model, audios, delays, opens, unbounded):
    pool = vx.StreamingPool(model, max_sessions=len(audios), max_seconds=None if unbounded else 12.0)
    n = len(audios)
    sids, fed, finished, ids = [None] * n, [0] * n, [False] * n, [[] for _ in range(n)]
    max_rows = 0
    try:
        for tick in range(2000):
            for i in range(n):
                if tick == opens[i]:
                    sids[i] = pool.open(delay=delays[i])
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
            for i in range(n):
                if sids[i] is None:
                    done_all = False
                    continue
                got, done = pool.poll(sids[i])
                ids[i] += got
                done_all = done_all and done
            if done_all:
                break
        return pool, sids, ids, max_rows
    except Exception:
        pool.close()
        raise


def _offline(model, audio, delay):
    model.set_delay(delay)
    return model.transcribe_pcm(audio, peak_normalize=False)[0].tolist()


@pytest.mark.parametrize("unbounded", [False, True], ids=["bounded", "unbounded"])
@pytest.mark.parametrize("mega", [True, False], ids=["mega", "mega_off"])
def test_streaming_pool_mixed_delays(vx, mixed, monkeypatch, unbounded, mega):
    """Sessions at delays 1, 6 and 30 opened at different ticks, then 11 sessions at mixed delays (two row groups per
    step).  Each session's ids == transcribe_pcm of its audio at its delay.  A reused slot runs at 6 again."""
    if mixed.window != 40:
        pytest.skip("one window is enough for the pool's bookkeeping")
    if not mega:
        monkeypatch.setenv("VOX_MEGA", "0")   # the pool's session reads it when it is created
    m = mixed.model
    try:
        audios = [omel.peak_normalize(omel.speechlike(s, 800 + i)) for i, s in enumerate((5.0, 7.5, 6.0))]
        pool, sids, ids, _ = _run_pool(vx, m, audios, [1.0, 6.0, 30.0], [0, 6, 14], unbounded)
        try:
            for i, a in enumerate(audios):
                assert ids[i] == _offline(m, a, [1.0, 6.0, 30.0][i]), i
            # errors (VOX_EINVAL): after the prefill, an unknown session
            for bad in ((sids[0], 2.0), (N + 5, 2.0)):
                with pytest.raises(vx.VoxtralError) as e:
                    pool.set_delay(*bad)
                assert e.value.code == VOX_EINVAL, bad
            # a session reusing the delay-30 slot (the only free one) runs at the default 6; NaN is refused
            pool.close_session(sids[2])
            reuse = pool.open()
            assert reuse == sids[2]
            with pytest.raises(vx.VoxtralError) as e:
                pool.set_delay(reuse, float("nan"))
            assert e.value.code == VOX_EINVAL
            a = omel.peak_normalize(omel.speechlike(5.0, 900))
            for k in range(0, a.size, 16000):
                pool.push(reuse, a[k:k + 16000])
                pool.tick()
            pool.finish(reuse)
            got = []
            for _ in range(50):
                pool.tick()
                part, done = pool.poll(reuse)
                got += part
                if done:
                    break
            assert got == _offline(m, a, 6.0)
        finally:
            pool.close()
        audios = [omel.peak_normalize(omel.speechlike(4.0 + 0.25 * i, 850 + i)) for i in range(N)]
        opens = [0] * 8 + [2, 3, 5]
        pool, sids, ids, max_rows = _run_pool(vx, m, audios, list(DELAYS), opens, unbounded)
        pool.close()
        assert max_rows > 8   # two row groups in one step
        for i, a in enumerate(audios):
            assert ids[i] == _offline(m, a, DELAYS[i]), i
    finally:
        m.set_delays(DELAYS)


@pytest.mark.slow
def test_full_size_eight_delays_one_launch_per_step(vx, full_gguf):
    """The full-size model, 8 pool sessions at 8 delays: ids == offline per session, one persistent launch per step."""
    m = vx.Q4ModelLoader.from_file(full_gguf).load(0, max_batch=8, max_mel_frames=1400)
    try:
        delays = DELAYS[:8]
        audios = [omel.peak_normalize(omel.speechlike(6.0, 950 + i)) for i in range(8)]
        # the decode step of 8 rows at 8 delays is one persistent-kernel launch
        m.set_delays(delays)
        m.encode_audio(np.concatenate([omel.mel_tensor_from_audio(a) for a in audios]))
        m.reset_cache()
        m.prefill(np.tile(PREFIX, (8, 1)).astype(np.int32))
        for _ in range(4):
            n0 = m.launch_count()
            m.decode_step(batch=8)
            assert m.launch_count() - n0 == 1
        pool = vx.StreamingPool(m, max_sessions=8, max_seconds=10.0)
        try:
            sids = [pool.open(delay=d) for d in delays]
            for a, s in zip(audios, sids):
                pool.push(s, a)
                pool.finish(s)
            st = pool.tick()
            ids = [pool.poll(s)[0] for s in sids]
            assert st["decode_rows"] == 8 * st["decode_steps"]   # all 8 sessions share every step
        finally:
            pool.close()
        for i, a in enumerate(audios):
            assert ids[i] == _offline(m, a, delays[i]), i
    finally:
        m.close()
