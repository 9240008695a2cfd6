import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    config.addinivalue_line("markers", "slow: long-running (full-size model)")


@pytest.fixture(scope="session")
def vx():
    """The product package with its in-tree library built (never the oracle)."""
    from voxtral_mini_realtime_rs_b200 import build as vbuild
    import voxtral_mini_realtime_rs_b200 as v
    if not os.path.exists(v.lib_path()):
        vbuild.build()
    v.lib()
    return v


@pytest.fixture(scope="session")
def have_gpu(vx):
    return vx.device_count() > 0


@pytest.fixture(scope="session")
def tiny_gguf(tmp_path_factory):
    from oracle import gguf_synth
    p = str(tmp_path_factory.mktemp("gguf") / "tiny.gguf")
    gguf_synth.write_synthetic_gguf(p, gguf_synth.VoxtralConfig.tiny(), seed=3)
    return p


@pytest.fixture(scope="session")
def full_gguf(tmp_path_factory):
    """The full-size synthetic model (seed 42, 2.5 GB; the weights bench.py runs), written once per session."""
    from voxtral_mini_realtime_rs_b200 import synth
    p = str(tmp_path_factory.mktemp("gguf_full") / "voxtral_synth_s42.gguf")
    synth.write_synthetic_gguf(p, synth.VoxtralConfig(), seed=42)
    return p


@pytest.fixture(scope="session")
def tiny_oracle(tiny_gguf):
    from oracle.model import OracleModel
    return OracleModel(tiny_gguf)


def closed_form_weights(n, k, c=0.0007, a=0.05, fn=np.cos):
    """Reference test input generator (tests.rs:435-438): fn(i*c)*a in f32."""
    i = np.arange(n * k, dtype=np.float32)
    return (fn(i * np.float32(c)).astype(np.float32) * np.float32(a)).astype(np.float32)
