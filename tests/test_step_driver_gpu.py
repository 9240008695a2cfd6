"""The session's decode-step driver: what a replayed CUDA graph of the step reads, and the persistent kernel's epoch count.

Model: the production decoder geometry (test_decode_geometry_ref.geometry_model_bytes, window 8192), max_batch 12.

- The captured step reads the op table the host built for its token capacity; an incremental call at another row count
  rebuilds that table in between, so a later replay must find the table of its own capacity again.
- Every host-side choice the captured kernels depend on is in the graph's key: the per-op path at 11 rows (the wgmma
  GEMM) is captured again after gemm_simt.  The streams' length is not: the rows' audio offsets are bound per call, so
  a step captured for one length replays for another.
- The host counts the persistent kernel's launches exactly as the device epoch advances (one per launch, ceil(R / 8)
  per step over R rows), through graph replays, incremental steps, beam calls and reset.
"""
import numpy as np
import pytest

from oracle import mel as omel
from oracle.model import PREFIX_LEN
from test_decode_geometry_ref import geometry_model_bytes

pytestmark = pytest.mark.gpu

N_STREAMS = 11
MEL_FRAMES = 1600
PREFIX = [1] + [32] * (PREFIX_LEN - 1)


@pytest.fixture(scope="module")
def drv(vx):
    m = vx.Q4ModelLoader.from_bytes(geometry_model_bytes(8192)).load(0, max_batch=12, max_mel_frames=MEL_FRAMES)
    mels = np.concatenate([omel.mel_tensor_from_audio(omel.peak_normalize(omel.speechlike(8.0, 700 + i)))
                           for i in range(N_STREAMS)])
    yield m, mels
    m.close()


def _transcribe(m, mels):
    """(ids, last-step logits, launches) of one transcribe_streaming call."""
    n0 = m.launch_count()
    ids = m.transcribe_streaming(mels)
    launches = m.launch_count() - n0
    return np.asarray(ids).reshape(len(mels), -1), m.debug("logits").reshape(len(mels), -1).copy(), launches


def _eager(m, mels):
    m.debug("graph_off")
    try:
        return _transcribe(m, mels)
    finally:
        m.debug("graph_on")


def _assert_same(a, b, what):
    assert a[0].shape[1] > 4, what   # several replayed steps
    assert np.array_equal(a[0], b[0]), what
    assert np.array_equal(a[1], b[1]), what


@pytest.mark.parametrize("capture,incremental", [(8, 4), (4, 8), (1, 8)])
def test_replay_after_incremental_call_at_another_capacity(drv, capture, incremental):
    m, mels = drv
    m.debug("mega_auto")
    first = _transcribe(m, mels[:capture])
    m.reset_cache()
    m.prefill(np.tile(PREFIX, (incremental, 1)).astype(np.int32), add_audio=False)
    for _ in range(3):
        m.decode_step(batch=incremental, add_audio=False)
    again = _transcribe(m, mels[:capture])
    _assert_same(again, first, ("replay", capture, incremental))
    _assert_same(again, _eager(m, mels[:capture]), ("eager", capture, incremental))


def test_q4_path_is_in_the_graph_key(drv):
    m, mels = drv
    m.debug("mega_off")
    try:
        _transcribe(m, mels)            # captures the per-op step at 11 rows on the wgmma GEMM
        m.debug("gemm_simt")
        graph = _transcribe(m, mels)
        eager = _eager(m, mels)
    finally:
        m.debug("gemm_tc")
        m.debug("mega_auto")
    _assert_same(graph, eager, "gemm_simt")
    assert graph[2] == eager[2]


def test_replay_across_stream_lengths(drv):
    """Two transcriptions at 4 rows whose streams differ in length: the second replays the step graph the first captured,
    and gives the ids and last-step logits of an eager run."""
    m, mels = drv
    m.debug("mega_auto")
    full = _transcribe(m, mels[:4])
    short = np.ascontiguousarray(mels[:4, :, :MEL_FRAMES // 2])
    again = _transcribe(m, short)
    assert again[0].shape[1] < full[0].shape[1]
    _assert_same(again, _eager(m, short), "shorter streams")


def _assert_epoch(m, what):
    host, dev = m.debug("mega_epoch")
    assert host == dev, (what, host, dev)
    return host


def test_epoch_count_is_exact(drv):
    m, mels = drv
    m.debug("mega_auto")
    e0 = _assert_epoch(m, "start")
    ids, _, _ = _transcribe(m, mels)
    e1 = _assert_epoch(m, "graph transcription at 11 rows")
    assert e1 - e0 == 2 * (ids.shape[1] - 1)       # two launches per step over 11 rows
    for _ in range(5):
        m.decode_step(batch=N_STREAMS, add_audio=False)
    assert _assert_epoch(m, "decode steps at 11 rows") == e1 + 10
    m.set_beam(4)
    try:
        m.transcribe_streaming(mels[:3])              # 12 rows
    finally:
        m.set_beam(1)
    _assert_epoch(m, "beam call at 3 x 4")
    m.reset_cache()
    _assert_epoch(m, "reset")
