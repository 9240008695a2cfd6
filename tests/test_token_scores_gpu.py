"""Token confidences: the top-k ids and log-probabilities of every emitted token (vox_session_set_top_k,
vox_session_token_scores, vox_stream_pool_set_top_k, vox_stream_poll_scored).

Model: the decoder-geometry model (synth.decoder_geometry_config, vocab 32768) at decoder windows 40 and 8192, 11 streams
at the mixed delays of test_delay_rows_ref.DELAYS, teacher-forced along the GPU's own greedy ids as in
tests/test_delay_rows_gpu.py.  Each returned log-probability is compared with log_softmax of OracleModel(dtype=float64)
at SCORE_REL_BOUND (tests/test_token_scores_ref.py pins that a mis-indexed row, step or position exceeds it), and with a
float64 reduction of the GPU's own logits at 1e-5 (the kernel alone).  Scores on or off never change the ids or the
logits, and cost exactly one launch per prefill and decode step.
"""
import ctypes

import numpy as np
import pytest

from oracle import mel as omel
from oracle.model import PREFIX_LEN
from test_delay_rows_gpu import Mixed, N, PREFIX, VOX_EINVAL
from test_delay_rows_ref import DELAYS, SECONDS
from test_token_scores_ref import MAX_TOP_K, OWN_LOGITS_TOL, log_softmax64, ref_topk, score_bound

pytestmark = pytest.mark.gpu

VOX_ECAPACITY = 7   # include/voxtral.h


def check_own_logits(logits, top_ids, top_lp, what):
    """The kernel alone: ids bitwise the float64 top-k of the GPU's own logits (ties by ascending id), log-probabilities
    within 1e-5 of log_softmax over them."""
    k = top_ids.shape[-1]
    ids, lp = ref_topk(logits, k)
    assert np.array_equal(top_ids, ids), what
    err = np.abs(top_lp.astype(np.float64) - lp).max()
    assert err <= OWN_LOGITS_TOL, (what, err)
    return err


def check_order(top_ids, top_lp, toks, what):
    assert np.array_equal(top_ids[..., 0], toks), what            # rank 0 is the emitted greedy id
    assert np.all(top_lp <= 0), what
    assert np.all(np.diff(top_lp, axis=-1) <= 0), what


class Scored(Mixed):
    def teacher_forced(self, B, steps=None, k=MAX_TOP_K):
        """logits [B][T][V], greedy ids [B][T], scores [B][T][k] x 2 of the prefill's last row and each decode step, and
        the launches of every decode step."""
        m = self.model
        m.set_top_k(k)
        m.encode_audio(self.mels[:B])
        m.reset_cache()
        toks = [m.prefill(self.seqs[:B, :PREFIX_LEN])]
        rows = [m.debug("logits").reshape(B, self.vocab).copy()]
        scores = [m.token_scores()] if k else []
        launches = []
        for p in range(PREFIX_LEN, self.S4 if steps is None else PREFIX_LEN + steps):
            n0 = m.launch_count()
            toks.append(m.decode_step(tok=self.seqs[:B, p]))
            launches.append(m.launch_count() - n0)
            rows.append(m.debug("logits").reshape(B, self.vocab).copy())
            if k:
                scores.append(m.token_scores())
        ids = np.concatenate([s[0] for s in scores], 1) if k else None
        lp = np.concatenate([s[1] for s in scores], 1) if k else None
        return np.stack(rows, 1), np.stack(toks, 1), ids, lp, np.array(launches)

    def check_f64(self, what, B, logits, toks, top_ids, top_lp):
        ref = self.ref[:B, :logits.shape[1]]
        check_order(top_ids, top_lp, toks, what)
        own = check_own_logits(logits, top_ids, top_lp, what)
        lsm = log_softmax64(ref)
        bound = score_bound(ref)
        err = np.abs(top_lp - np.take_along_axis(lsm, top_ids, -1)).max(-1) / bound
        print(f"\n[token scores] window {self.window:5d} {what:>9s} B={B:2d}: max |dlogprob| = {err.max():.2f} x bound "
              f"vs f64, {own:.1e} vs own logits, over {err.size} rows")
        assert err.max() <= 1.0, (what, B, np.unravel_index(int(np.argmax(err)), err.shape))
        # the ids of ranks whose f64 neighbours are separated by more than twice the bound are the f64 ranking's
        k = top_ids.shape[-1]
        rid, rlp = ref_topk(ref, k + 1)
        gap = -np.diff(rlp, axis=-1) > 2 * bound[..., None]
        sure = gap[..., :k] & np.concatenate([np.ones_like(gap[..., :1]), gap[..., :k - 1]], -1)
        assert np.array_equal(top_ids[sure], rid[..., :k][sure]), (what, B)
        assert sure[..., 0].mean() > 0.5


@pytest.fixture(scope="module", params=(40, 8192), ids=lambda w: f"window{w}")
def scored(request, vx):
    g = Scored(vx, request.param)
    g.model.set_delays(DELAYS)
    yield g
    g.model.close()


@pytest.mark.parametrize("B", [1, 3, 8, 11])
def test_persistent_kernel_scores(scored, B):
    m = scored.model
    m.debug("mega_auto")
    logits, toks, top_ids, top_lp, launches = scored.teacher_forced(B)
    scored.check_f64("mega", B, logits, toks, top_ids, top_lp)
    assert np.all(launches == (B + 7) // 8 + 1), (B, np.unique(launches))   # one score launch for every group
    off_logits, off_toks, _, _, off_launches = scored.teacher_forced(B, k=0)
    assert np.all(off_launches == (B + 7) // 8), (B, np.unique(off_launches))
    assert np.array_equal(off_logits, logits) and np.array_equal(off_toks, toks)   # bitwise: scores change nothing
    again = scored.teacher_forced(B)
    assert np.array_equal(again[2], top_ids) and np.array_equal(again[3], top_lp)   # bitwise reproducible


@pytest.mark.parametrize("path,B", [("mega_off", 3), ("mega_off", 11), ("tc_off", 3)])
def test_per_op_path_scores(scored, path, B):
    m = scored.model
    m.debug(path)
    try:
        logits, toks, top_ids, top_lp, _ = scored.teacher_forced(B)
        off_logits, off_toks, _, _, _ = scored.teacher_forced(B, k=0)
    finally:
        m.debug("tc_on" if path == "tc_off" else "mega_auto")
    scored.check_f64(path, B, logits, toks, top_ids, top_lp)
    assert np.array_equal(off_logits, logits) and np.array_equal(off_toks, toks)


def test_smaller_k_is_a_prefix(scored):
    m = scored.model
    _, _, i8, l8, _ = scored.teacher_forced(3, steps=5)
    _, _, i3, l3, _ = scored.teacher_forced(3, steps=5, k=3)
    assert i3.shape[-1] == 3
    assert np.array_equal(i3, i8[..., :3]) and np.array_equal(l3, l8[..., :3])
    m.set_top_k(0)


def _replay(m, ids):
    """Teacher-forced prefill + decode steps over the embeddings the last transcribe left resident: the scores of its
    positions, [B][n][k]."""
    B, n = ids.shape
    m.reset_cache()
    m.prefill(np.tile(PREFIX, (B, 1)).astype(np.int32))
    parts = [m.token_scores()]
    for j in range(n - 1):
        m.decode_step(tok=ids[:, j])
        parts.append(m.token_scores())
    return np.concatenate([p[0] for p in parts], 1), np.concatenate([p[1] for p in parts], 1)


@pytest.mark.parametrize("B", [1, 3, 8, 11])
def test_transcribe_scores_graph_and_offline(scored, B):
    """transcribe_streaming and transcribe_pcm replay a captured step.  With scores on and off the ids are bitwise
    equal; on, token_scores() has n_out positions that are bitwise those of a teacher-forced prefill / decode_step run
    over the same embeddings, and every prefill and decode step costs exactly one more launch (the captured step
    includes the score launch: k changed, so the graph was re-captured)."""
    if scored.window != 40:
        pytest.skip("the graph bookkeeping does not depend on the window")
    m = scored.model
    audio = np.stack([omel.peak_normalize(omel.speechlike(SECONDS, 700 + i)) for i in range(B)])
    runs = {"streaming": lambda: np.asarray(m.transcribe_streaming(scored.mels[:B])).reshape(B, -1),
            "pcm": lambda: m.transcribe_pcm(audio, peak_normalize=False)}
    try:
        for name, run in runs.items():
            got = {}
            for k in (0, MAX_TOP_K, 0, MAX_TOP_K):
                m.set_top_k(k)
                n0 = m.launch_count()
                ids = run()
                got.setdefault(k, []).append((ids, m.launch_count() - n0, m.token_scores() if k else None))
            (i0, n_off, _), (i1, _, _) = got[0]
            (j0, n_on, s0), (j1, _, s1) = got[MAX_TOP_K]
            assert np.array_equal(i0, j0) and np.array_equal(i0, i1) and np.array_equal(i0, j1), name
            n_out = i0.shape[1]
            assert n_on - n_off == n_out, (name, n_on, n_off, n_out)      # prefill + (n_out - 1) decode steps
            top_ids, top_lp = s0
            assert top_ids.shape == (B, n_out, MAX_TOP_K), name
            check_order(top_ids, top_lp, i0, name)
            assert np.array_equal(s1[0], top_ids) and np.array_equal(s1[1], top_lp), name   # repeatable
            r_ids, r_lp = _replay(m, i0)
            assert np.array_equal(r_ids, top_ids) and np.array_equal(r_lp, top_lp), name
    finally:
        m.set_top_k(0)


def test_errors(vx, scored):
    m = scored.model
    lib = vx.lib()
    for k in (-1, MAX_TOP_K + 1):
        with pytest.raises(vx.VoxtralError) as e:
            m.set_top_k(k)
        assert e.value.code == VOX_EINVAL, k
    m.set_top_k(0)
    m.transcribe_streaming(scored.mels[:2])
    with pytest.raises(vx.VoxtralError) as e:     # the last run had scores off
        m.token_scores()
    assert e.value.code == VOX_EINVAL
    m.set_top_k(4)
    try:
        ids = m.transcribe_streaming(scored.mels[:2])
        need = ids.size * 4
        buf_i, buf_l = np.empty(need, np.int32), np.empty(need, np.float32)
        b, n, k = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
        ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        assert lib.vox_session_token_scores(m._s, ptr(buf_i), ptr(buf_l), need - 1, ctypes.byref(b), ctypes.byref(n),
                                            ctypes.byref(k)) == VOX_ECAPACITY
        assert lib.vox_session_token_scores(m._s, ptr(buf_i), ptr(buf_l), need, ctypes.byref(b), ctypes.byref(n),
                                            ctypes.byref(k)) == 0
        assert (b.value, n.value, k.value) == (2, ids.shape[1], 4)
    finally:
        m.set_top_k(0)


def tiny_reduction(vx, tiny_gguf, mega):
    """vocab 512: fewer logits per row than CTAs x threads, so most threads and lanes hold empty lists."""
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=3, max_mel_frames=2000)
    try:
        if not mega:
            m.debug("mega_off")
        mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(4.0, 60 + i))) for i in range(3)])
        m.encode_audio(mels)
        m.reset_cache()
        m.set_top_k(MAX_TOP_K)
        toks = m.prefill(np.tile(PREFIX, (3, 1)).astype(np.int32))
        for step in range(12):
            logits = m.debug("logits").reshape(3, -1)
            assert logits.shape[1] == 512
            top_ids, top_lp = m.token_scores()
            check_order(top_ids[:, 0], top_lp[:, 0], toks, f"tiny step {step}")
            check_own_logits(logits, top_ids[:, 0], top_lp[:, 0], f"tiny step {step}")
            toks = m.decode_step(batch=3)
    finally:
        m.close()


@pytest.mark.parametrize("mega", [True, False], ids=["mega", "mega_off"])
def test_tiny_model_reduction(vx, tiny_gguf, mega):
    tiny_reduction(vx, tiny_gguf, mega)


def _pool_run(vx, model, audios, opens, unbounded):
    pool = vx.StreamingPool(model, max_sessions=len(audios), max_seconds=None if unbounded else 12.0)
    try:
        pool.set_top_k(MAX_TOP_K)
        n = len(audios)
        sids, fed, finished = [None] * n, [0] * n, [False] * n
        ids, tops, lps = [[] for _ in range(n)], [[] for _ in range(n)], [[] for _ in range(n)]
        for tick in range(2000):
            for i in range(n):
                if tick == opens[i]:
                    sids[i] = pool.open()
                    with pytest.raises(vx.VoxtralError) as e:   # k is pool-wide: not while a session is open
                        pool.set_top_k(2)
                    assert e.value.code == VOX_EINVAL
                if sids[i] is None or finished[i]:
                    continue
                if fed[i] < audios[i].size:
                    pool.push(sids[i], audios[i][fed[i]:fed[i] + 1280])
                    fed[i] += 1280
                else:
                    pool.finish(sids[i])
                    finished[i] = True
            pool.tick()
            done_all = True
            for i in range(n):
                if sids[i] is None:
                    done_all = False
                    continue
                got, done, t, l = pool.poll(sids[i], scores=True)
                assert t.shape == (len(got), MAX_TOP_K)
                ids[i] += got
                tops[i].append(t)
                lps[i].append(l)
                done_all = done_all and done
            if done_all:
                break
        return ids, [np.concatenate(t) for t in tops], [np.concatenate(l) for l in lps]
    finally:
        pool.close()


@pytest.mark.parametrize("unbounded", [False, True], ids=["bounded", "unbounded"])
@pytest.mark.parametrize("mega", [True, False], ids=["mega", "mega_off"])
def test_streaming_pool_scores(vx, scored, monkeypatch, unbounded, mega):
    """Sessions opened at different ticks (up to 11 rows per step): each session's ids are its offline ids, and its
    scores are those of the offline transcription of the same audio within the f64 bound."""
    if scored.window != 40:
        pytest.skip("one window is enough for the pool's bookkeeping")
    if not mega:
        monkeypatch.setenv("VOX_MEGA", "0")   # the pool's session reads it when it is created
    m = scored.model
    audios = [omel.peak_normalize(omel.speechlike(4.0 + 0.25 * i, 850 + i)) for i in range(N)]
    opens = [0] * 8 + [2, 3, 5]
    ids, tops, lps = _pool_run(vx, m, audios, opens, unbounded)
    bound = score_bound(scored.ref).max()
    m.set_delay(6.0)
    m.set_top_k(MAX_TOP_K)
    try:
        for i, a in enumerate(audios):
            off = m.transcribe_pcm(a, peak_normalize=False)[0]
            o_ids, o_lp = (x[0] for x in m.token_scores())
            assert ids[i] == off.tolist(), i
            assert tops[i].shape == o_ids.shape, i
            assert np.array_equal(tops[i][:, 0], off), i
            same = tops[i] == o_ids
            assert same[:, 0].all()
            assert np.abs(lps[i][same] - o_lp[same]).max() <= 2 * bound, i   # both within the f64 bound
    finally:
        m.set_top_k(0)
        m.set_delays(DELAYS)


@pytest.mark.slow
def test_full_size_scores(vx, full_gguf):
    """The production model (vocab 131072), 8 streams on the persistent kernel: ids with scores on are the ids with
    scores off, rank 0 is the emitted id, and the kernel matches a float64 reduction of the GPU's own logits."""
    m = vx.Q4ModelLoader.from_file(full_gguf).load(0, max_batch=8, max_mel_frames=1400)
    try:
        audios = np.stack([omel.peak_normalize(omel.speechlike(6.0, 950 + i)) for i in range(8)])
        off = m.transcribe_pcm(audios, peak_normalize=False)
        m.set_top_k(MAX_TOP_K)
        on = m.transcribe_pcm(audios, peak_normalize=False)
        assert np.array_equal(off, on)
        top_ids, top_lp = m.token_scores()
        check_order(top_ids, top_lp, on, "full size")
        m.reset_cache()
        toks = m.prefill(np.tile(PREFIX, (8, 1)).astype(np.int32))
        for step in range(6):
            n0 = m.launch_count()
            if step:
                toks = m.decode_step(batch=8)
                assert m.launch_count() - n0 == 2    # the persistent kernel + the score launch
            s_ids, s_lp = m.token_scores()
            logits = m.debug("logits").reshape(8, -1)
            assert logits.shape[1] == 131072
            check_order(s_ids[:, 0], s_lp[:, 0], toks, f"full size step {step}")
            check_own_logits(logits, s_ids[:, 0], s_lp[:, 0], f"full size step {step}")
    finally:
        m.close()
