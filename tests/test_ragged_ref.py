"""CPU side of vox_transcribe_pcm_ragged and Q4VoxtralModel.transcribe_long.

  * The wrapper's host sizing (stream_n_out: pad_audio length -> mel frames -> two stride-2 convolutions -> / 4 -> minus
    the 38-token prefix) equals what the oracle's pipeline produces for the same stream, at lengths around every
    rounding edge; frames_n_out at mel lengths where S4 = 37, 38, 39 and S % 4 != 0 equals the oracle conv stem's own
    output length.
  * transcribe_long's orchestration, with the device call replaced by a fake: one peak normalisation over the whole
    recording, the reference ChunkIterator's plan (overlap > 0, a last chunk of a few samples), chunks grouped into calls
    in order with at most max_batch // W per call.
  * join_chunk_texts follows transcribe.rs:256-275: ids >= 1000, decode, trim, drop empty texts, join with a space.
  * The ctypes prototype of vox_transcribe_pcm_ragged matches the header.
"""
import numpy as np
import pytest

import voxtral_mini_realtime_rs_b200 as vx
from oracle import mel as omel
from oracle.model import PREFIX_LEN
from test_delay_rows_ref import _prototype

REDUCE = 4


def _oracle_n_out(n_samples: int) -> int:
    padded = omel.pad_audio(np.zeros(n_samples, np.float32))
    frames = omel.num_frames(padded.size)
    s = frames
    for _ in range(2):                           # conv.rs:47-48, k3 s2 p1
        s = (s + 2 * 1 - 3) // 2 + 1
    return max(0, s // REDUCE - PREFIX_LEN)


@pytest.mark.parametrize("n", [1, 2, 159, 160, 161, 639, 640, 641, 1279, 1280, 1281, 2559, 2560, 2561, 16000, 16001,
                               47999, 48000, 48001, 160000 - 1, 160000, 192000 + 77])
def test_stream_n_out_matches_oracle(n):
    assert vx.stream_n_out(n) == _oracle_n_out(n)


def _oracle_conv_len(frames, tiny_oracle):
    mel = np.zeros((1, 128, frames), np.float32)
    return int(tiny_oracle.conv_stem(mel).shape[0])


@pytest.mark.parametrize("s4", [0, 1, 36, 37, 38, 39, 40])
def test_frames_n_out_edges(tiny_oracle, s4):
    """Mel lengths whose encoder length S gives S4 = s4, with S % 4 = 0 and 3 (shorter than the prefix: no output; 38:
    none; 39: one)."""
    for s_extra in (0, 3):
        S = 4 * s4 + s_extra
        if S < 1:
            continue
        frames = 4 * S - 3                       # the fewest mel frames giving S encoder frames
        assert _oracle_conv_len(frames, tiny_oracle) == S
        assert vx.frames_n_out(frames) == max(0, S // REDUCE - PREFIX_LEN) == max(0, s4 - PREFIX_LEN)


# ---------------------------------------------------------------------------------------------------------------------
class _Fake(vx.Q4VoxtralModel):
    """A Q4VoxtralModel whose device call records its arguments and returns one array per stream."""

    def __init__(self, max_batch, beam=1):
        self.max_batch, self._beam = max_batch, beam
        self.calls = []

    def transcribe_pcm_ragged(self, streams, peak_normalize=True, timings=None):
        self.calls.append(([np.array(s, copy=True) for s in streams], peak_normalize))
        return [np.array([len(self.calls), i], np.int32) for i in range(len(streams))]

    def close(self):
        pass


@pytest.mark.parametrize("max_batch,beam", [(8, 1), (2, 1), (8, 4), (3, 2)])
@pytest.mark.parametrize("overlap", [0, 50])
def test_transcribe_long_orchestration(max_batch, beam, overlap):
    rng = np.random.default_rng(5)
    n = 1200 * 160 * 4 + 7                            # four 1200-frame chunks and a last one of 7 samples (overlap 0)
    rec = (rng.standard_normal(n) * 0.1).astype(np.float32)
    rec[n - 3] = 2.5                                  # the peak is in the last chunk
    m = _Fake(max_batch, beam)
    ids, plan = m.transcribe_long(rec, max_mel_frames=1200, overlap_frames=overlap)
    assert plan == omel.chunk_plan(n, 1200, overlap_frames=overlap)
    if overlap == 0:
        assert plan[-1][1] - plan[-1][0] == 7 and plan[-1][3]
    norm = omel.peak_normalize(rec)                   # once, over the whole recording
    per_call = max_batch // beam
    assert [len(c[0]) for c in m.calls] == [min(per_call, len(plan) - i) for i in range(0, len(plan), per_call)]
    flat = [s for c in m.calls for s in c[0]]
    assert len(flat) == len(plan) and all(c[1] is False for c in m.calls)
    for (a, b, _, _), s in zip(plan, flat):
        np.testing.assert_array_equal(s, norm[a:b])
    assert [tuple(x) for x in ids] == [(1 + i // per_call, i % per_call) for i in range(len(plan))]


def test_transcribe_long_without_normalisation():
    rec = np.linspace(-0.2, 0.2, 5000, dtype=np.float32)
    m = _Fake(4)
    m.transcribe_long(rec, max_mel_frames=10, peak_normalize=False)
    np.testing.assert_array_equal(np.concatenate([s for c in m.calls for s in c[0]]), rec)


class _Tok:
    def decode(self, ids):
        return "".join({1000: " hello", 1001: "world ", 1002: "  ", 1003: "x"}.get(i, "?") for i in ids)


def test_join_chunk_texts():
    chunks = [[1, 32, 1000, 1001], [32, 33], [1002], [999, 1003, 5]]
    # chunk 1: " helloworld " -> "helloworld"; chunk 2: no text ids; chunk 3: blank after trim; chunk 4: "x"
    assert vx.join_chunk_texts(_Tok(), chunks) == "helloworld x"
    assert vx.join_chunk_texts(_Tok(), []) == ""


def test_ragged_prototype():
    p = _prototype("vox_transcribe_pcm_ragged")
    assert "const size_t *lens" in p and "int32_t *n_out" in p
    from voxtral_mini_realtime_rs_b200.api import _SIGS
    assert len(_SIGS["vox_transcribe_pcm_ragged"][1]) == 9
