#!/usr/bin/env python
"""Prefill GEMM times on the H100: the four decoder GEMMs of one layer at the prefill's shape, and the whole prefill.

Per GEMM (wqkv 6144 x 3072, wo 3072 x 4096, w13 18432 x 3072, w2 3072 x 9216) at M = 38 * B token rows, B = 1, 2, 4, 8:
vox_q4_matmul (the Q4 operator, which takes the same launch_q4_linear path as the session: M > 8 runs split_tiles + the
wgmma GEMM K3), device-timed with CUDA events over `--iters` launches that rotate over four copies of the weight (so the
weights come from HBM, as in a prefill, where every layer's weights are read once), median of `--rounds` rounds.
Rates: the f32-equivalent 2*M*N*K and the 3-product f16 tensor work (3 x that) per second, each beside the 989 TFLOP/s
dense FP16 figure of NVIDIA's H100 SXM data sheet (a data-sheet peak, not a measurement).

Whole prefill: the session's device-timed prefill (vox_timings prefill_ms) of B streams of 16 s on the full-size
synthetic model (seed 42, the weights bench.py runs), median of `--rounds` transcribe calls after one warm-up call.

    python scripts/prefill_bench.py [--rounds 5] [--iters 20] [--gguf PATH] [--out FILE]

--gguf: where the synthetic model is written (reused when it exists: A/B runs of two builds share one file; the build
is picked with VOX_LIB_PATH).  Prints one JSON line with the card's name and power limit; --out also writes it.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEMMS = {"wqkv": (6144, 3072), "wo": (3072, 4096), "w13": (18432, 3072), "w2": (3072, 9216)}
PEAK_F16_TFLOPS = 989.0   # H100 SXM data sheet, dense FP16 / BF16, 700 W card
COPIES = 4


def gemm_times(vx, torch, rounds: int, iters: int, batches) -> dict:
    from voxtral_mini_realtime_rs_b200 import synth
    rng = np.random.default_rng(7)
    out = {}
    for name, (n, k) in GEMMS.items():
        ws = [vx.Q4Tensor.from_q4_bytes(synth.random_q4_blocks(rng, n * k, 1.0 / np.sqrt(k)), (n, k)) for _ in range(COPIES)]
        m_max = 38 * max(batches)
        x = vx.DeviceBuffer.from_numpy(rng.standard_normal((m_max, k)).astype(np.float32))
        y = vx.DeviceBuffer(m_max * n * 4)
        lib = vx.lib()
        for B in batches:
            M = 38 * B

            def run(i):
                rc = lib.vox_q4_matmul(ws[i % COPIES]._h, x.ptr, y.ptr, 1, M, None, None)
                assert rc == 0, f"vox_q4_matmul failed: {rc}"

            for i in range(2 * COPIES):   # warm-up: module load, split buffer growth
                run(i)
            torch.cuda.synchronize()
            ms = []
            for _ in range(rounds):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(iters):
                    run(i)
                e1.record()
                e1.synchronize()
                ms.append(e0.elapsed_time(e1) / iters)
            t = statistics.median(ms)
            flop = 2.0 * M * n * k
            out.setdefault(f"B{B}", {})[name] = {
                "M": M, "ms": round(t, 4), "ms_rounds": [round(v, 4) for v in ms],
                "f32_equiv_tflops": round(flop / t / 1e9, 1),
                "f16_3product_tflops": round(3 * flop / t / 1e9, 1),
                "f16_3product_share_of_datasheet_989": round(3 * flop / t / 1e9 / PEAK_F16_TFLOPS, 3)}
        x.free()
        y.free()
    for B, g in out.items():
        g["layer_ms"] = round(sum(v["ms"] for v in g.values()), 4)
    return out


def prefill_times(vx, gguf: str, rounds: int, batches) -> dict:
    from oracle import mel as omel
    m = vx.Q4ModelLoader.from_file(gguf).load(0, max_batch=max(batches), max_mel_frames=2800)
    audio = [omel.peak_normalize(omel.speechlike(16.0, 40 + i)) for i in range(max(batches))]
    mels = np.concatenate([omel.mel_tensor_from_audio(a) for a in audio])
    out = {}
    for B in batches:
        m.transcribe_streaming(mels[:B])    # warm-up (captures the decode-step graph at this B)
        ms = []
        for _ in range(rounds):
            tm = vx.Timings()
            m.transcribe_streaming(mels[:B], timings=tm)
            ms.append(tm.prefill_ms)
        out[f"B{B}"] = {"ms": round(statistics.median(ms), 3), "ms_rounds": [round(v, 3) for v in ms]}
    m.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--gguf", default=None)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    import voxtral_mini_realtime_rs_b200 as vx
    from voxtral_mini_realtime_rs_b200 import synth

    if vx.device_count() < 1 or not torch.cuda.is_available():
        sys.exit("prefill_bench.py needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    batches = (1, 2, 4, 8)
    res = {"gpu": gpu, "lib": vx.lib_path(), "rounds": args.rounds, "iters": args.iters}
    res["gemm"] = gemm_times(vx, torch, args.rounds, args.iters, batches)
    with tempfile.TemporaryDirectory() as d:
        path = args.gguf or os.path.join(d, "full.gguf")
        if not os.path.exists(path):
            synth.write_synthetic_gguf(path, synth.VoxtralConfig(), seed=42)
        res["prefill"] = prefill_times(vx, path, args.rounds, batches)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
