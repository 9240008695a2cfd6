"""The audio front end (kernels.cu K1) on the GPU against the float64 reference of tests/mel_reference.py, and every
call path's mel against the offline mel, bit for bit.

  * mel_kernel through vox_mel_compute_log at the edge lengths (0, 1, 159 .. 361), at 7, 8, 9, 15, 16 and 17 frames
    with n % 4 at every residue, 2 s and 30 s, on every signal of mel_reference.SIGNALS: every output inside its
    interval, outputs with an interval narrower than TIER2_WIDTH within TIER2_E.  Per signal the worst |GPU - f64|,
    the median interval width and the fraction of outputs under the tier-2 width are printed.
  * vox_mel_compute_log_dev from device pointers offset by 0 .. 4 floats (float4 span staging off and on), layouts 0
    and 1: layout 0 equals the host entry's result bit for bit, layout 1 is its transpose, a repeat is bitwise equal.
  * peak_max_kernel + scale_pad_kernel through vox_transcribe_pcm (B = 3), _dev (offset pointer) and _ragged: the
    "pcm_pad" debug read equals mel_reference.normalize_pad of every stream bit for bit, and "mel" equals the offline
    vox_mel_compute_log of that padded signal bit for bit.
  * The stream pool's incremental mel, read with vox_stream_mel_range after every tick, equals the offline mel of
    pad_audio(x) bit for bit: pieces of cycling sizes, a bounded pool with two sessions at different phases and an
    unbounded pool over 72 s whose buffers slide; evicted frames give VOX_ECAPACITY.
"""
import ctypes as C

import numpy as np
import pytest

import mel_reference as mr
from oracle import mel as omel

pytestmark = pytest.mark.gpu

PIECES = (1, 159, 160, 161, 1279, 1280, 4001, 16000)


@pytest.fixture(scope="module")
def ms(vx):
    return vx.MelSpectrogram(0)


@pytest.fixture(scope="module")
def tables(ms):
    return ms.window(), ms.mel_basis()


@pytest.fixture(scope="module")
def model(vx, tiny_gguf):
    m = vx.Q4ModelLoader.from_file(tiny_gguf).load(0, max_batch=4, max_mel_frames=1500)
    yield m
    m.close()


@pytest.fixture
def make_pool(vx, model):
    """StreamingPool factory whose pools are freed when the test ends, while `model` is still open (a pool reads its
    model when it is freed; left to the garbage collector, that could happen after the model was closed)."""
    pools = []

    def make(**kw):
        pools.append(vx.StreamingPool(model, **kw))
        return pools[-1]
    yield make
    for p in pools:
        p.close()


def _check_signal(ms, tables, x):
    got = ms.compute_log(x)
    assert got.shape == (mr.num_frames(x.size), 128)
    return mr.check(got, mr.reference(x, *tables))


def test_kernel_against_f64(ms, tables):
    lengths = mr.EDGE_LENGTHS + mr.FRAME_LENGTHS + (32000,)
    for name in mr.SIGNALS:
        worst, worst_n, widths, narrow, outputs = 0.0, 0.0, [], 0.0, 0
        runs = [(n, mr.signal(name, n)) for n in lengths]
        if name in ("speech", "noise", "impulses"):
            runs.append((480000, mr.signal(name, 480000)))
        for n, x in runs:
            r = _check_signal(ms, tables, x)
            assert r["inside"], (name, n, r)
            assert r["tier2"], (name, n, r)
            k = mr.num_frames(n) * 128
            worst, worst_n = max(worst, r["worst"]), max(worst_n, r["worst_narrow"])
            if k:
                widths.append(r["width_median"])
                narrow += r["narrow_frac"] * k
                outputs += k
        print(f"{name:10s}: worst |GPU - f64| {worst:.2e}, worst on narrow outputs {worst_n:.2e}, median width "
              f"{np.median(widths):.1e}, under {mr.TIER2_WIDTH:.0e}: {narrow / max(outputs, 1):.2f}")


def test_repeat_is_bitwise_equal(ms):
    x = mr.signal("speech", 160 * 17 + 3)
    assert np.array_equal(ms.compute_log(x), ms.compute_log(x))
    assert np.all(ms.compute_log(mr.signal("silence", 16000)) == np.float32(mr.FLOOR))


def test_dev_entry_offsets_and_layouts(vx, ms):
    lib = vx.lib()
    for n in (160, 199, 361, 160 * 8 + 1, 160 * 9 + 2, 160 * 16 + 3, 160 * 17, 32000):
        x = mr.signal("noise", n, seed=n)
        host = ms.compute_log(x)
        F = host.shape[0]
        for off in range(5):
            buf = np.zeros(n + 8, np.float32)
            buf[off:off + n] = x
            src = vx.DeviceBuffer.from_numpy(buf)
            dst = vx.DeviceBuffer(max(F * 128 * 4, 16))
            outs = []
            for layout in (0, 1, 0):
                vx.api._check(lib.vox_mel_compute_log_dev(ms._h, C.c_void_p(src.ptr.value + 4 * off), n, dst.ptr, layout,
                                                          None))
                vx.api._check(lib.vox_dev_sync(0))
                outs.append(dst.to_numpy(np.float32, (F * 128,)))
            assert np.array_equal(outs[0].reshape(F, 128), host), (n, off)
            assert np.array_equal(outs[1].reshape(128, F), host.T), (n, off)
            assert np.array_equal(outs[2], outs[0]), (n, off)
            src.free()
            dst.free()


def _front_end_matches(model, ms, streams, normalize=True):
    pcm = model.debug("pcm_pad")
    mel = model.debug("mel")
    p0 = m0 = 0
    for x in streams:
        exp = mr.normalize_pad(x, normalize)
        got = pcm[p0:p0 + exp.size]
        assert np.array_equal(got, exp), (x.size, np.flatnonzero(got != exp)[:8])
        offline = ms.compute_log(exp)
        assert np.array_equal(mel[m0:m0 + offline.size].reshape(offline.shape), offline), x.size
        p0 += exp.size
        m0 += offline.size
    assert pcm.size == p0 and mel.size == m0


def test_device_normalize_pad_and_mel_batched(model, ms):
    rng = np.random.default_rng(11)
    for n in (16000, 16003):
        a = rng.uniform(-0.4, 0.4, n).astype(np.float32)
        tail = rng.uniform(-0.4, 0.4, n).astype(np.float32)
        tail[-1] = 0.6                               # the peak at the last sample (a scalar tail when n % 4 != 0)
        neg = rng.uniform(-0.4, 0.4, n).astype(np.float32)
        neg[n // 3] = -1.7                           # a negative peak
        zero = np.zeros(n, np.float32)
        tiny = np.full(n, 5e-11, np.float32)         # peak below 1e-10: not scaled
        for group in ((a, tail, neg), (zero, tiny, a)):
            for normalize in (True, False):
                model.transcribe_pcm(np.stack(group), peak_normalize=normalize)
                _front_end_matches(model, ms, group, normalize)


def test_device_normalize_pad_and_mel_dev_offset(vx, model, ms):
    n, b = 16001, 3
    x = np.stack([mr.signal("speech", n, seed=s) * np.float32(0.3 + s) for s in range(b)])
    buf = np.zeros(b * n + 4, np.float32)
    buf[1:1 + b * n] = x.reshape(-1)
    dev = vx.DeviceBuffer.from_numpy(buf)

    class Offset:   # the device pointer one float into the allocation: no float4 path anywhere
        ptr = C.c_void_p(dev.ptr.value + 4)
    model.transcribe_pcm_dev(Offset, b, n)
    _front_end_matches(model, ms, list(x))
    dev.free()


def test_device_normalize_pad_and_mel_ragged(model, ms):
    rng = np.random.default_rng(4)
    streams = [rng.uniform(-0.3, 0.3, n).astype(np.float32) for n in (7, 16001, 4003, 48000)]
    streams[2][-1] = -0.9
    model.transcribe_pcm_ragged(streams)
    _front_end_matches(model, ms, streams)
    model.transcribe_pcm_ragged(streams, peak_normalize=False)
    _front_end_matches(model, ms, streams, normalize=False)


def test_mel_read_after_uploaded_mel(vx, model):
    mel = omel.mel_tensor_from_audio(mr.signal("speech", 8000))
    model.encode_audio(mel)
    assert np.array_equal(model.debug("mel").reshape(mel.shape), mel)
    with pytest.raises(vx.VoxtralError) as e:
        model.debug("pcm_pad")
    assert e.value.code == 3


def _stream(pool, sessions):
    """Pushes each session's audio in cycling piece sizes (session i starting i pieces into the cycle and after
    `start` pushes of the others), ticks after every round and collects [previous mel_frames, mel_frames) of every
    session.  sessions: [(audio, start_round)] -> per session the collected frames."""
    ids = [None] * len(sessions)
    pos = [0] * len(sessions)
    got = [[] for _ in sessions]
    done_mel = [0] * len(sessions)
    finished = [False] * len(sessions)
    rnd = 0
    while not all(finished):
        for i, (x, start) in enumerate(sessions):
            if rnd < start or finished[i]:
                continue
            if ids[i] is None:
                ids[i] = pool.open()
            k = PIECES[(rnd - start + i) % len(PIECES)]
            piece = x[pos[i]:pos[i] + k]
            pos[i] += piece.size
            if piece.size:
                pool.push(ids[i], piece)
            if pos[i] >= x.size:
                pool.finish(ids[i])
                finished[i] = True
        pool.tick()
        for i in range(len(sessions)):
            if ids[i] is None:
                continue
            m = pool.session_info(ids[i])["mel_frames"]
            if m > done_mel[i]:
                got[i].append(pool.mel_range(ids[i], done_mel[i], m - done_mel[i]))
                done_mel[i] = m
        rnd += 1
    return ids, [np.concatenate(g) for g in got]


def test_stream_pool_mel_bounded(vx, make_pool, ms):
    a, b = mr.signal("speech", 5 * 16000 + 3, seed=1), mr.signal("chirp", 4 * 16000 + 1)
    pool = make_pool(max_sessions=2, max_seconds=8)
    ids, got = _stream(pool, [(a, 0), (b, 3)])
    for x, g, sid in zip((a, b), got, ids):
        assert np.array_equal(g, ms.compute_log(omel.pad_audio(x)))
        assert pool.session_info(sid)["mel_frames"] == g.shape[0]
        with pytest.raises(vx.VoxtralError) as e:
            pool.mel_range(sid, g.shape[0] - 1, 2)
        assert e.value.code == 1


def test_stream_pool_mel_unbounded_slides(vx, make_pool, ms):
    x = mr.signal("speech", 72 * 16000 + 2, seed=3)
    pool = make_pool(max_sessions=1, max_seconds=None)
    ids, got = _stream(pool, [(x, 0)])
    exp = ms.compute_log(omel.pad_audio(x))
    assert got[0].shape == exp.shape
    # 30 s of padded audio resident: the mel buffer slid at least twice over this session
    assert exp.shape[0] > 2 * vx.lib().vox_mel_num_frames(vx.lib().vox_pad_audio_len(30 * 16000, None))
    bad = np.flatnonzero(np.any(got[0] != exp, axis=1))
    assert bad.size == 0, bad[:8]
    with pytest.raises(vx.VoxtralError) as e:
        pool.mel_range(ids[0], 0, 1)
    assert e.value.code == 7
