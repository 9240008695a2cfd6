"""The Tekken encoder (tokenizer.cpp) under AddressSanitizer + UBSan, built like test_host_sanitizers.py: random bytes,
random and truncated UTF-8, long runs, two threads on one handle, and vocabularies with byte tokens cut away, a duplicated
token or another pattern (tests/native/tokenizer_encode_driver.cpp)."""
import base64
import json
import os
import shutil
import subprocess

import pytest

import tekken_reference as tr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "voxtral_mini_realtime_rs_b200", "csrc")


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
def test_tokenizer_encode_under_asan_ubsan(tmp_path):
    pytest.importorskip("regex")   # the synthetic vocabulary's trainer pre-tokenizes with it
    exe = tmp_path / "drv"
    cmd = ["g++", "-std=c++17", "-g", "-O1", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
           "-fno-omit-frame-pointer", "-pthread", "-I", CSRC, "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "native", "tokenizer_encode_driver.cpp"), os.path.join(CSRC, "tokenizer.cpp"),
           "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and ("asan" in r.stderr.lower() or "sanitize" in r.stderr.lower()):
        pytest.skip("toolchain without sanitizer runtimes")
    assert r.returncode == 0, r.stderr[-2000:]
    doc = json.loads(tr.synthetic_bpe_tekken_json(tr.BPE_CORPUS, 400))
    cut = json.loads(json.dumps(doc))
    cut["config"]["default_vocab_size"] = 1000 + 128             # bytes 128..255 cut away
    dup = json.loads(json.dumps(doc))
    dup["vocab"].append(dict(dup["vocab"][300], rank=len(dup["vocab"])))
    dup["vocab"][280] = dict(dup["vocab"][300], rank=280)
    dup["vocab"][5] = {"rank": 5, "token_bytes": base64.b64encode(b"e").decode(), "token_str": "e"}   # byte 5 missing
    dup["vocab"].append({"rank": len(dup["vocab"]), "token_bytes": base64.b64encode(b"\x05").decode(), "token_str": None})
    dup["config"]["default_vocab_size"] = 1000 + len(dup["vocab"])
    pat = json.loads(json.dumps(doc))
    pat["config"]["pattern"] = r"\s+|\S+"
    paths = []
    for name, d in (("bpe", doc), ("cut", cut), ("dup", dup), ("pattern", pat)):
        p = tmp_path / f"{name}.json"
        p.write_text(json.dumps(d))
        paths.append(str(p))
    r = subprocess.run([str(exe)] + paths, capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0"))
    assert r.returncode == 0, (r.stdout[-1000:], r.stderr[-3000:])
    assert "done" in r.stdout and "ERROR: AddressSanitizer" not in r.stderr and "runtime error" not in r.stderr
    print(r.stdout)
