"""Timings of the Loquacious Conformers (conformer_activation=torch.nn.GELU) on one GPU, on seeded weights, 10 s utterances.
CUDA events around whole calls after warm-up; each row reports the median and the range (min, max) over --reps calls:

* xlarge (18 layers, d_model 1024, 16 heads): encode (wav -> encoder states, AsrEngine.encode_wav) at 32 x 10 s;
* xlarge encode + 48 greedy steps (AsrEngine.transcribe_greedy_dev) at 32 x 10 s;
* xlarge, the recipe's test search (beam 80, CTC 0.3 with blank 3, temperature 1.15, using_eos_threshold) on 8 x 10 s of
  encoder states: one step = (time of a 24-step search - time of the 1-step search run just before it) / 23, per pair;
* Conformer-L (14 layers, d_model 768, 12 heads) encode at 32 x 10 s with Swish and with GELU on the same weights, the two
  engines called alternately in one run, so the activation's cost is measured rather than assumed.

Prints one JSON object with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def stats(ts):
    ts = sorted(ts)
    return dict(median_ms=round(ts[len(ts) // 2], 3), min_ms=round(ts[0], 3), max_ms=round(ts[-1], 3))


def measure(fns, reps, warmup=3):
    """{name: stats} of the callables in fns, called in turn (alternated) reps times after warmup calls each"""
    for _ in range(warmup):
        for f in fns.values():
            f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():
            ts[k].append(timed(f))
    return {k: stats(v) for k, v in ts.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=11)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("loquacious.py measures on a GPU; none found")
    import loquacious_oracle as LO
    import test_gpu_loquacious as T
    from mirrors import build_mirror, seeded
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_LARGE, LOQUACIOUS_XLARGE
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info()}
    g = torch.Generator().manual_seed(0)
    wav = torch.randn(32, 160000, generator=g).to(dev)
    lens = torch.ones(32, device=dev)
    cfg = LOQUACIOUS_XLARGE
    eng = AsrEngine(cfg, seeded(cfg), device=str(dev))
    out = measure({"xlarge_encode_32x10s": lambda: eng.encode_wav(wav, lens),
                   "xlarge_encode_greedy48_32x10s": lambda: eng.transcribe_greedy_dev(wav, lens, 48, LO.BOS, LO.EOS)},
                  args.reps)
    res.update(out)
    enc, l8 = eng.encode_wav(wav[:8], lens[:8]), lens[:8]
    del eng
    m = build_mirror(cfg, seeded(cfg))
    searchers = {s: T.searcher(m, (s + 0.5) / enc.shape[1]) for s in (1, 24)}
    for b in searchers.values():
        b(enc, l8)
    torch.cuda.synchronize()
    steps = []  # per alternated pair: (24-step search - 1-step search) / 23
    for _ in range(max(5, args.reps // 2)):
        t1, t24 = timed(lambda: searchers[1](enc, l8)), timed(lambda: searchers[24](enc, l8))
        steps.append((t24 - t1) / 23)
    res["xlarge_beam80_ctc_step_8x10s"] = stats(steps)
    del searchers, m
    cfg = LOQUACIOUS_LARGE
    sd = seeded(cfg)
    engs = {a: AsrEngine(dict(cfg, conformer_activation=a), sd, device=str(dev)) for a in ("swish", "gelu")}
    res.update(measure({f"large_{a}_encode_32x10s": (lambda e=e: e.encode_wav(wav, lens)) for a, e in engs.items()},
                       args.reps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
