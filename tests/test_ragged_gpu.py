"""vox_transcribe_pcm_ragged: streams of different lengths in one call, and transcribe_long (long recordings as rows of
ragged calls).

  * Equal lengths are vox_transcribe_pcm bit for bit: ids, token scores (k = 3) and n-best (W = 2), b = 1, 3, 8, 11.
  * Mixed lengths: each stream's ids equal that stream's own vox_transcribe_pcm under the near-tie / teacher-forcing
    rule (test_golden_gpu.assert_ids_match; the packed GEMMs run at another M), at b = 5 and 11 (rows retire across the
    8-row groups of the persistent kernel), with S % 4 != 0 and a stream at exactly max_mel_frames, on the default
    paths and under mega_off, enc_attn_simt, gemm_simt and tc_off.  With pad_audio's 76 + 17 tokens of padding even a
    one-sample stream has S4 = 47, so n_out = 0 and 1 cannot be reached from PCM; the host arithmetic of those edges is
    pinned in test_ragged_ref.py.
  * The ragged encoder at the production encoder geometry (window 750 biting inside the longer streams) against the f64
    reference run on each stream alone: packed encoder output and audio embeddings, tensor-core and SIMT attention.
  * Rows retire: persistent-kernel launches per step = ceil(live rows / 8), and max n_out - 1 steps.
  * Per-stream delays, token scores and beams (W = 2, 4) compose.
  * After a ragged call, vox_prefill / vox_decode_step with add_audio read the streams in the caller's order, up to the
    shortest stream's positions.
  * transcribe_long equals per-chunk vox_transcribe_pcm of the host-normalised chunks (overlap 0 and > 0).
  * Bad arguments are refused before device work and leave the session usable; a ragged call leaves the cache empty.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import mel as omel
from oracle.model import PREFIX_LEN, OracleModel
from test_encoder_geometry_ref import EMBED_REL_BOUND, encoder_geometry_bytes, rel_err
from test_golden_gpu import NEAR_TIE, assert_ids_match
from voxtral_mini_realtime_rs_b200 import synth

pytestmark = pytest.mark.gpu

MAX_BATCH = 22
MAX_MEL = 1400


@pytest.fixture(scope="module")
def tiny(vx, tiny_gguf):
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=MAX_BATCH, max_mel_frames=MAX_MEL)
    yield m
    m.close()


def _audio(seconds, seed):
    return synth.speechlike(seconds, seed=seed).astype(np.float32)


def _stream(n, seed):
    """n samples of speech-like audio."""
    a = _audio(max(n, 16000) / 16000.0 + 0.1, seed)[:n]
    assert a.size == n
    return a


def _longest_samples(vx, max_mel):
    """The most samples whose padded mel still fits max_mel frames."""
    lo, hi = 1, max_mel * 160
    frames = lambda n: vx.lib().vox_mel_num_frames(vx.lib().vox_pad_audio_len(n, None))
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if frames(mid) <= max_mel:
            lo = mid
        else:
            hi = mid - 1
    assert frames(lo) == max_mel
    return lo


def _mixed_lengths(vx, b):
    """b lengths in samples, all different: a few samples, S % 4 != 0 ones, and one at exactly MAX_MEL mel frames."""
    base = [1, 16000 + 160 * 3, 52000, 21000 + 160 * 7, 36000 + 160, 9000, 44000, 27000, 31000 + 160 * 5, 5000, 60000]
    lens = base[:b - 1] + [_longest_samples(vx, MAX_MEL)]
    assert len(set(lens)) == b
    return lens


def _single_gold(m, audio, k=2, normalize=True):
    """Ids of the stream's own vox_transcribe_pcm, with its top-2 margins for the near-tie rule."""
    m.set_top_k(k)
    ids = m.transcribe_pcm(audio, peak_normalize=normalize)[0]
    top, lp = m.token_scores()
    m.set_top_k(0)
    return {"tokens": ids, "margins": (lp[0, :, 0] - lp[0, :, 1]).astype(np.float64), "second": top[0, :, 1],
            "top": top[0], "lp": lp[0]}


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b", [1, 3, 8, 11])
def test_equal_lengths_bitwise(tiny, b):
    audios = [_audio(3.0, 100 + i) for i in range(b)]
    arr = np.stack(audios)
    try:
        tiny.set_top_k(3)
        ref = tiny.transcribe_pcm(arr)
        ref_top, ref_lp = tiny.token_scores()
        got = tiny.transcribe_pcm_ragged(audios)
        sc = tiny.token_scores_ragged()
        for i in range(b):
            np.testing.assert_array_equal(got[i], ref[i])
            np.testing.assert_array_equal(sc[i][0], ref_top[i])
            np.testing.assert_array_equal(sc[i][1].view(np.uint32), ref_lp[i].view(np.uint32))
        tiny.set_top_k(0)
        tiny.set_beam(2)
        ref = tiny.transcribe_pcm(arr)
        ref_ids, ref_scores = tiny.nbest()
        got = tiny.transcribe_pcm_ragged(audios)
        nb = tiny.nbest_ragged()
        for i in range(b):
            np.testing.assert_array_equal(got[i], ref[i])
            np.testing.assert_array_equal(nb[i][0], ref_ids[i])
            np.testing.assert_array_equal(nb[i][1], ref_scores[i])
    finally:
        tiny.set_top_k(0)
        tiny.set_beam(1)
    print(f"\n[ragged] b={b} equal lengths: ids, k=3 scores and W=2 n-best bitwise equal to vox_transcribe_pcm")


@pytest.mark.parametrize("path", ["default", "mega_off", "enc_attn_simt", "gemm_simt", "tc_off"])
@pytest.mark.parametrize("b", [5, 11])
def test_mixed_lengths_match_single_stream(vx, tiny, b, path):
    lens = _mixed_lengths(vx, b)
    audios = [_stream(n, 200 + i) for i, n in enumerate(lens)]
    assert [a.size for a in audios] == lens
    golds = [_single_gold(tiny, a) for a in audios]
    on, off = {"default": (None, None), "mega_off": ("mega_off", "mega_on"), "enc_attn_simt": ("enc_attn_simt", "enc_attn_tc"),
               "gemm_simt": ("gemm_simt", "gemm_tc"), "tc_off": ("tc_off", "tc_on")}[path]
    if on:
        tiny.debug(on)
    try:
        got = tiny.transcribe_pcm_ragged(audios)
    finally:
        if off:
            tiny.debug(off)
    for i, a in enumerate(audios):
        assert got[i].shape == golds[i]["tokens"].shape == (vx.stream_n_out(lens[i]),)
        assert_ids_match(got[i], golds[i], f"b={b} {path} stream {i} ({lens[i]} samples)", tiny, audio=a)


def test_rows_retire(vx, tiny):
    lens = _mixed_lengths(vx, 11)
    audios = [_stream(n, 300 + i) for i, n in enumerate(lens)]
    n_out = [vx.stream_n_out(n) for n in lens]
    before = tiny.debug("mega_epoch")[0]
    tm = vx.Timings()
    tiny.transcribe_pcm_ragged(audios, timings=tm)
    launches = tiny.debug("mega_epoch")[0] - before
    expect = sum(-(-sum(1 for n in n_out if n > t) // 8) for t in range(1, max(n_out)))
    print(f"\n[ragged] n_out {sorted(n_out, reverse=True)}: {launches:.0f} persistent-kernel launches over "
          f"{max(n_out) - 1} steps (b x steps / 8 rounded up per step would be {(max(n_out) - 1) * 2})")
    assert launches == expect
    assert tm.decode_tokens == max(n_out)
    assert tiny.cache_len() == 0


def test_mixed_delays(vx, tiny):
    lens = _mixed_lengths(vx, 5)
    audios = [_stream(n, 400 + i) for i, n in enumerate(lens)]
    delays = [6.0, 2.0, 9.0, 6.0, 4.0]
    golds = []
    try:
        for a, d in zip(audios, delays):
            tiny.set_delay(d)
            golds.append(_single_gold(tiny, a))
        tiny.set_delays(delays)
        got = tiny.transcribe_pcm_ragged(audios)
    finally:
        tiny.set_delay(6.0)
    for i, a in enumerate(audios):
        # teacher forcing runs stream 0's delay: compare the free-running ids only, a near-tie ends the comparison
        g, x = golds[i], got[i]
        diff = np.nonzero(x != g["tokens"])[0]
        if diff.size:
            j = int(diff[0])
            assert g["margins"][j] < NEAR_TIE and x[j] == g["second"][j], (i, j)
        print(f"\n[ragged] delay {delays[i]}: stream {i} {diff[0] if diff.size else x.size}/{x.size} ids equal")


def test_token_scores_compose(vx, tiny):
    lens = _mixed_lengths(vx, 5)
    audios = [_stream(n, 500 + i) for i, n in enumerate(lens)]
    golds = [_single_gold(tiny, a, k=4) for a in audios]
    tiny.set_top_k(4)
    try:
        got = tiny.transcribe_pcm_ragged(audios)
        sc = tiny.token_scores_ragged()
    finally:
        tiny.set_top_k(0)
    for i in range(len(audios)):
        g = golds[i]
        top, lp = sc[i]
        assert top.shape == lp.shape == (g["tokens"].size, 4)
        np.testing.assert_array_equal(top[:, 0], got[i])
        diff = np.nonzero(got[i] != g["tokens"])[0]
        upto = int(diff[0]) if diff.size else got[i].size
        if diff.size:
            assert g["margins"][upto] < NEAR_TIE and got[i][upto] == g["second"][upto]
        err = float(np.abs(lp[:upto, 0] - g["lp"][:upto, 0]).max()) if upto else 0.0
        print(f"\n[ragged] scores stream {i}: {upto}/{got[i].size} positions compared, max |d logprob| {err:.2e}")
        assert err < NEAR_TIE


@pytest.mark.parametrize("W", [2, 4])
def test_beams_compose(vx, tiny, W):
    lens = _mixed_lengths(vx, 5)[:4] if W == 4 else _mixed_lengths(vx, 5)
    audios = [_stream(n, 600 + i) for i, n in enumerate(lens)]
    tiny.set_beam(W)
    try:
        single = []
        for a in audios:
            tiny.transcribe_pcm(a)
            ids, scores = tiny.nbest()
            single.append((ids[0], scores[0]))
        tiny.transcribe_pcm_ragged(audios)
        nb = tiny.nbest_ragged()
    finally:
        tiny.set_beam(1)
    for i in range(len(audios)):
        assert nb[i][0].shape == single[i][0].shape == (W, vx.stream_n_out(lens[i]))
        np.testing.assert_allclose(nb[i][1], single[i][1], rtol=1e-4, atol=1e-3)
        np.testing.assert_array_equal(nb[i][0], single[i][0])
    print(f"\n[ragged] W={W}: every stream's n-best equals its single-stream beam call")


def test_add_audio_after_ragged_call_reads_caller_order(vx, tiny):
    """Streams given shortest first, so the caller's order is the reverse of the sorted decoder rows.  A prefill and
    decode steps teacher-forced along the ragged ids, with add_audio, read stream i's embeddings in row i: they give
    stream i's ragged ids (near-tie runner-ups allowed), up to the shortest stream's positions, and refuse the next."""
    lens = [9000, 21000 + 160 * 7, 44000]
    audios = [_stream(n, 1000 + i) for i, n in enumerate(lens)]
    b = len(audios)
    tiny.set_top_k(2)
    try:
        ids = tiny.transcribe_pcm_ragged(audios)
        sc = tiny.token_scores_ragged()
    finally:
        tiny.set_top_k(0)
    assert ids[0].size < ids[1].size < ids[2].size
    n = ids[0].size   # the shortest stream's S4 is PREFIX_LEN + n
    try:
        got = [tiny.prefill(np.tile([1] + [32] * (PREFIX_LEN - 1), (b, 1)), add_audio=True)]
        for t in range(1, n + 1):   # position PREFIX_LEN + n - 1 has audio too; its id is the one no call emits
            got.append(tiny.decode_step(tok=[x[t - 1] for x in ids], add_audio=True))
        assert tiny.cache_len() == PREFIX_LEN + n
        with pytest.raises(vx.VoxtralError) as e:
            tiny.decode_step(tok=[x[n - 1] for x in ids], add_audio=True)
        assert e.value.code == 1
    finally:
        tiny.reset_cache()
    got = np.stack(got[:n], 1)
    for i in range(b):
        top, lp = sc[i]
        for j in np.nonzero(got[i] != ids[i][:n])[0]:
            assert lp[j, 0] - lp[j, 1] < NEAR_TIE and got[i][j] == top[j, 1], (i, j)
        print(f"\n[ragged] add_audio after a ragged call: stream {i} {int((got[i] == ids[i][:n]).sum())}/{n} ids equal")


# ---------------------------------------------------------------------------------------------------------------------
def _gpu_mel(vx, audio):
    return vx.MelSpectrogram.voxtral(0).compute_log(vx.pad_audio(audio)).T[None]


@pytest.mark.parametrize("attn", ["enc_attn_tc", "enc_attn_simt"])
def test_ragged_encoder_packed_embeds_vs_f64(vx, attn):
    """Window 750: streams of 30, 16 and 7 s (S = 938, 588, 363 encoder frames): the window bites inside the first."""
    data = encoder_geometry_bytes(750)
    m = vx.Q4ModelLoader.from_bytes(data).load(0, max_batch=3, max_mel_frames=4000)
    o64 = OracleModel(data, dtype=torch.float64)
    try:
        audios = [vx.peak_normalize(_audio(s, 700 + i)) for i, s in enumerate((30.0, 16.0, 7.0))]
        m.debug(attn)
        try:
            m.transcribe_pcm_ragged(audios, peak_normalize=False)
        finally:
            m.debug("enc_attn_tc")
        d, D = o64.cfg.enc_dim, o64.cfg.dec_dim
        enc = m.debug("enc_out").reshape(-1, d)
        emb = m.debug("audio_embeds").reshape(-1, D)   # stream after stream, in the caller's order
        r0 = e0 = 0
        for i, a in enumerate(audios):
            mel = _gpu_mel(vx, a)
            cap = {}
            ref_emb = o64.encode_audio(mel, cap).numpy()
            ref_enc = cap["enc_out"].numpy()
            S = ref_enc.shape[0]
            got_enc = enc[r0:r0 + S]
            r0 += S
            got_emb = emb[e0:e0 + ref_emb.shape[0]]
            e0 += ref_emb.shape[0]
            e1, e2 = rel_err(got_enc, ref_enc), rel_err(got_emb, ref_emb)
            print(f"\n[ragged encoder] {attn} stream {i} S={S}: enc_out {e1:.2e}, embeds {e2:.2e} (bound {EMBED_REL_BOUND:.0e})")
            assert S > 750 or i > 0
            assert e1 <= EMBED_REL_BOUND and e2 <= EMBED_REL_BOUND
        assert r0 == enc.shape[0] and e0 == emb.shape[0]
    finally:
        m.close()


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("overlap,seconds", [(0, 16.5), (40, 15.0)])
def test_transcribe_long(vx, tiny_gguf, overlap, seconds):
    """3 s chunks, two per call: six chunks, the last call a full chunk beside a shorter one (a ragged call)."""
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=2, max_mel_frames=1100)
    try:
        rec = _audio(seconds, 800) * 0.3
        rec[int(11.5 * 16000)] = 0.9          # the peak is in a later chunk
        ids, plan = m.transcribe_long(rec, max_mel_frames=300, overlap_frames=overlap)
        assert len(plan) == 6 and len(ids) == len(plan)
        assert plan[-1][1] - plan[-1][0] < plan[-2][1] - plan[-2][0]
        norm = vx.peak_normalize(rec)
        for (a, b, idx, _), got in zip(plan, ids):
            chunk = norm[a:b]
            gold = _single_gold(m, chunk, normalize=False)
            assert got.shape == gold["tokens"].shape
            assert_ids_match(got, gold, f"overlap {overlap} chunk {idx}", m, mel=_gpu_mel(vx, chunk))
        print(f"\n[ragged] transcribe_long overlap {overlap}: {len(plan)} chunks in 3 calls match per-chunk "
              f"vox_transcribe_pcm")
    finally:
        m.close()


def _raw(vx, m, samples, lens, b, cap):
    """vox_transcribe_pcm_ragged with the arguments as given (the wrapper sizes them right)."""
    out = np.zeros(max(cap, 1), np.int32)
    no = np.zeros(max(b, 1), np.int32)
    ln = np.array(lens, np.uint64)
    return vx.lib().vox_transcribe_pcm_ragged(m._s, samples.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), b, 1,
                                              out.ctypes.data_as(C.c_void_p), cap, no.ctypes.data_as(C.c_void_p), None)


def test_errors_and_cache(vx, tiny):
    a = _audio(4.0, 900)
    baseline = tiny.transcribe_pcm(a)[0]
    x = np.concatenate([a, a[:30000]])
    n1, n2 = vx.stream_n_out(a.size), vx.stream_n_out(30000)
    cases = [
        (x, [a.size, 30000], 0, n1 + n2, 1),                    # b < 1
        (np.zeros(MAX_BATCH + 1, np.float32), [1] * (MAX_BATCH + 1), MAX_BATCH + 1, 1000, 1),   # b > max_batch
        (x, [a.size, 0], 2, n1 + n2, 1),                        # an empty stream
        (np.zeros(MAX_MEL * 160, np.float32), [MAX_MEL * 160], 1, 1000, 1),   # more mel frames than the session takes
        (x, [a.size, 30000], 2, n1 + n2 - 1, 7),                # out_ids one short: VOX_ECAPACITY
    ]
    for samples, lens, b, cap, code in cases:
        assert _raw(vx, tiny, samples, lens, b, cap) == code, (lens, b, cap)
    tiny.set_beam(4)
    try:
        streams = [a[:20000 + 1000 * i] for i in range(6)]          # 6 x 4 rows > 22
        with pytest.raises(vx.VoxtralError) as e:
            tiny.transcribe_pcm_ragged(streams)
        assert e.value.code == 1
    finally:
        tiny.set_beam(1)
    np.testing.assert_array_equal(tiny.transcribe_pcm(a)[0], baseline)
    tiny.transcribe_pcm_ragged([a, a[:30000]])
    assert tiny.cache_len() == 0
    nxt = tiny.prefill(np.array([[1] + [32] * 37], np.int32), add_audio=False)
    assert nxt.shape == (1,) and tiny.cache_len() == 38
    tiny.reset_cache()
    np.testing.assert_array_equal(tiny.transcribe_pcm(a)[0], baseline)
