"""Per-chunk time of StreamingASR.transcribe_chunk, from waveform to text, on the transducer fixture's model (12-layer
RoPEMHA Conformer-L, proj_enc, 640 / 512 / 1000 prediction network; tests/streaming_asr_util.build).

For 1 and 32 streams at DynChunkTrainConfig (24, 8) and (16, 4): a stream of --chunks chunks of seeded audio after
--warmup chunks, and per chunk
  * wall: host clock around transcribe_chunk, which ends in the token copy the detokeniser needs (the chunk's only host
    synchronisation), so it is the waveform-to-text time;
  * enqueue: host clock around encode_chunk alone (front end, encoder and proj_enc enqueued, nothing awaited);
  * launches: library kernel launches per chunk (sbk_launch_count; the greedy search kernel included).
Prints one JSON line per setting, with the card name and power limit read in the same run.

    python tools/streaming_asr_e2e.py [--chunks 40] [--warmup 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout.strip().splitlines()[0]
    name, power = (s.strip() for s in q.split(","))
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("streaming_asr_e2e: needs a CUDA device")
    import streaming_asr_util as SU
    from speechbrain_b200._lib import lib
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    asr = SU.build("RoPEMHA")[0]
    name, power = card()
    for B in (1, 32):
        for chunk, left in ((24, 8), (16, 4)):
            cfg = DynChunkTrainConfig(chunk, left)
            n = asr.get_chunk_size_frames(cfg)
            total = args.warmup + args.chunks
            wav = torch.randn(B, total * n, generator=torch.Generator().manual_seed(B * 100 + chunk)).cuda() * 0.1
            ctx = asr.make_streaming_context(cfg)
            wall, enq, launches = [], [], []
            for k in range(total):
                ch = wav[:, k * n:(k + 1) * n]
                torch.cuda.synchronize()
                l0 = lib().sbk_launch_count()
                t0 = time.perf_counter()
                x = asr.encode_chunk(ctx, ch)
                t1 = time.perf_counter()
                asr.decode_chunk(ctx, x)
                t2 = time.perf_counter()
                if k >= args.warmup:
                    wall.append((t2 - t0) * 1e3)
                    enq.append((t1 - t0) * 1e3)
                    launches.append(lib().sbk_launch_count() - l0)
            print(json.dumps(dict(streams=B, chunk_size=chunk, left_context_chunks=left, chunk_samples=n,
                                  chunk_audio_ms=n / 16.0, chunks=args.chunks, wall_ms_median=statistics.median(wall),
                                  wall_ms_max=max(wall), enqueue_ms_median=statistics.median(enq),
                                  launches_per_chunk=sorted(set(launches)), gpu=name, power_limit=power)))


if __name__ == "__main__":
    main()
