"""Per-chunk latency of the streaming Conformer encoder (TransformerASR.encode_streaming on per-layer device caches).

For each DynChunkTrainConfig and number of concurrent streams it reports, after the caches have filled:
  * stream: the median and range of CUDA-event times of one encode_streaming call (one chunk of every stream);
  * recompute: a masked encode(..., dynchunktrain_config) of the window a cache-less implementation must re-encode for the
    same chunk (num_layers x max(left frames + chunk - 1, conv halo) + chunk frames, rounded up to whole chunks);
  * the host time of the same call without synchronisation (how long the launches take to enqueue);
  * the real-time factor per stream (chunk time / chunk audio, 40 ms per encoder frame).
The model is the LibriSpeech Conformer-Transducer's encoder shape (Conformer-L, RoPE, 12 layers) with seeded weights.
The card's name and power limit are read in the same run.

    python tools/streaming_asr.py [--chunks 40] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def host_enqueue(fn, n):
    """Median host time for fn to return (no synchronisation): when it is close to the device time of fn, the device
    waits on the host's launches."""
    ts = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    torch.cuda.synchronize()
    ts.sort()
    return ts[len(ts) // 2]


def timed(fn, n):
    ts = []
    for _ in range(n):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return {"median_ms": ts[len(ts) // 2], "min_ms": ts[0], "max_ms": ts[-1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=40, help="timed chunks per configuration")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("streaming_asr.py needs a CUDA device")
    import bench
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    dev = torch.device("cuda:0")
    cfg = dict(CONFORMER_LARGE, num_decoder_layers=1)
    tr = bench.build_product_asr(cfg, seeded_asr_state(cfg, 0), dev).transformer
    L, halo = cfg["num_encoder_layers"], (cfg["kernel_size"] - 1) // 2
    rows = []
    gen = torch.Generator().manual_seed(0)
    for cs, lc in ((24, 8), (16, 4)):
        for B in (1, 32):
            dc = DynChunkTrainConfig(cs, lc)
            fill = lc + 2
            src = torch.randn(B, (fill + args.chunks + 10) * cs, 640, generator=gen).to(dev)
            ctx = tr.make_streaming_context(dc)
            k = [0]

            def step():
                tr.encode_streaming(src[:, k[0] * cs:(k[0] + 1) * cs], ctx)
                k[0] += 1
            for _ in range(fill + 3):  # fill the caches and warm every shape
                step()
            st = timed(step, args.chunks)
            st["host_enqueue_ms"] = host_enqueue(step, 5)
            keep = L * max(lc * cs + cs - 1, halo) + cs
            keep = -(-keep // cs) * cs
            win = src[:, :keep].contiguous()
            tr.encode(win, None, dynchunktrain_config=dc)
            rc = timed(lambda: tr.encode(win, None, dynchunktrain_config=dc), max(5, args.chunks // 4))
            chunk_audio_ms = cs * 40.0
            row = {"chunk_size": cs, "left_context_chunks": lc, "streams": B, "stream": st, "recompute_window_frames": keep,
                   "recompute": rc, "rtf_per_stream": st["median_ms"] / chunk_audio_ms,
                   "speedup_vs_recompute": rc["median_ms"] / st["median_ms"]}
            rows.append(row)
            print(f"({cs}, {lc}) x {B:2d} streams: stream {st['median_ms']:.3f} ms [{st['min_ms']:.3f}, {st['max_ms']:.3f}]  "
                  f"host {st['host_enqueue_ms']:.3f} ms  recompute of {keep} frames {rc['median_ms']:.3f} ms  RTF {row['rtf_per_stream']:.4f}  "
                  f"x{row['speedup_vs_recompute']:.1f}", flush=True)
    res = {"card": card(), "model": "conformer_large RoPEMHA 12 layers (encoder only)", "rows": rows}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
