"""All-CTA phase trace of the persistent decode-step kernel: skew vs fixed cost per phase.

    VOX_MEGA_TRACE_ALL=1 python scripts/mega_trace_all.py [--streams B] [--save trace.npy]

Every CTA stamps (SM clock) op start / first weights ready (or KV walk start) / body done / barrier passed; the CTAs are
aligned on their exit from the first grid barrier (they leave it within one L2 round trip of each other).  Per op class:
  ready50       median CTA: first weight stage consumed (= fragment staging done) / KV walk started
  done10..max   body finished (fastest decile / median / slowest decile / slowest CTA): max - p50 = imbalance + stragglers
  phase         barrier exit to barrier exit (median CTA);  bar-lat = phase - donemax = pure barrier latency
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("VOX_MEGA_TRACE_ALL", "1")
import voxtral_mini_realtime_rs_b200 as vx  # noqa: E402
from voxtral_mini_realtime_rs_b200 import synth  # noqa: E402

GGUF = os.environ.get("VOX_BENCH_GGUF", "/dev/shm/voxtral_synth_s42.gguf")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=8)
    ap.add_argument("--save", metavar="NPY", default=None, help="also write the raw trace [CTA][op][4] here")
    args = ap.parse_args()
    if not os.path.exists(GGUF):
        synth.write_synthetic_gguf(GGUF, synth.VoxtralConfig(), seed=42)
    B = args.streams
    audio = np.stack([synth.speechlike(16.0, seed=1234 + i) for i in range(B)])
    model = vx.Q4ModelLoader.from_file(GGUF).load(0, max_batch=B, max_mel_frames=2400)
    tm = vx.Timings()
    model.debug("mega_on")
    model.transcribe_pcm(audio, timings=tm)
    model.transcribe_pcm(audio, timings=tm)
    tr = model.debug("mega_trace_all")
    n = 1 + 5 * model.info["dec_layers"] + 2         # embed, 5 phases per layer, lm_head, argmax
    tr = tr.reshape(-1, n, 4)                        # one row per CTA: the grid is one CTA per SM of this device
    per_layer = ["qkv", "attn", "wo", "w13", "w2"]
    names = ["embed"] + per_layer * ((n - 3) // len(per_layer)) + ["lm_head", "argmax"]
    step = (tm.decode_ms - tm.prefill_ms) / max(1, tm.decode_tokens - 1)
    print(f"B={B}: step (graph) {step:.3f} ms; flags {os.environ.get('VOX_MEGA_FLAGS', '0')}")
    # SM clocks are not mutually synchronised (and drift): every CTA is measured against ITS OWN exit from the previous
    # grid barrier -- all CTAs leave a barrier within one L2 round trip of each other, so these offsets are comparable.
    agg = {}
    if args.save:
        np.save(args.save, tr)
    for i, nm in enumerate(names):
        start, done, exit_, ready = tr[:, i, 0], tr[:, i, 1], tr[:, i, 2], tr[:, i, 3]
        prev = tr[:, i - 1, 2] if i > 0 else start
        if i == n - 1:
            exit_ = done
        d_done = done - prev           # per CTA: body finished, since the previous barrier
        d_ready = ready - prev
        d_exit = exit_ - prev
        a = agg.setdefault(nm, dict(n=0, ready=0.0, p10=0.0, p50=0.0, p90=0.0, mx=0.0, phase=0.0))
        a["n"] += 1
        a["ready"] += float(np.median(d_ready))
        a["p10"] += float(np.percentile(d_done, 10))
        a["p50"] += float(np.median(d_done))
        a["p90"] += float(np.percentile(d_done, 90))
        a["mx"] += float(d_done.max())
        a["phase"] += float(np.median(d_exit))
    print(f"{'op':8s} {'n':>3s} {'ready50':>7s} {'done10':>7s} {'done50':>7s} {'done90':>7s} {'donemax':>7s} {'phase':>7s} {'bar-lat':>7s} (mean us since the previous barrier) | total")
    tot = 0.0
    for nm, a in agg.items():
        c = a["n"]
        tot += a["phase"]
        print(f"{nm:8s} {c:3d} {a['ready'] / c:7.2f} {a['p10'] / c:7.2f} {a['p50'] / c:7.2f} {a['p90'] / c:7.2f} {a['mx'] / c:7.2f} {a['phase'] / c:7.2f} "
              f"{(a['phase'] - a['mx']) / c:7.2f} | {a['phase']:8.1f}")
    print(f"sum of phases {tot:.1f} us")
    tw = model.debug("mega_trace_w")
    if tw is not None:
        tw = tw.reshape(16, 6, 8)
        print("warp-level trace, CTA 0, op " + os.environ.get("VOX_MEGA_TRACE_W_OP", "lm_head") + " (SM cycles since the first stamp): per group = start, "
              "stage1, stage2, stage3 ready, body done, group barrier passed, epilogue done, (reducers) partials summed")
        for gidx in range(6):
            print(f" group {gidx}")
            for w in range(16):
                print("   w%02d " % w + " ".join(f"{int(v):7d}" for v in tw[w, gidx, :8]))


if __name__ == "__main__":
    main()
