"""Encoder cost per batch when E batches of 32 x 10 s go through Fbank -> CMVN -> CNN -> Conformer-L as ONE pass of E*32
utterances, for E = 1, 2, 4, 7, 16 (seeded conformer_large.yaml weights, RoPEMHA and RelPosMHAXL).

* CUDA events around whole-pipeline graph replays (poll interval 0, no decode steps), after warm-up, rounds alternated over
  E; reports the median per-batch time of each E and its spread over the rounds;
* one torch.profiler pass per E (a separate run of the same graph): kernel count, summed kernel time and first kernel
  start -> last kernel end, all per batch.

Prints the card name and power limit read in the same run, then one JSON line (``--out DIR`` also writes it and the traces
there).  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, L = 32, 160000


def _time(fn, reps):
    """Median of `reps` event-timed calls (ms)."""
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def _profile(fn, trace):
    """Kernel count, summed kernel time (us) and first start -> last end (us) of one profiled call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        ev = [e for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    t0 = min(e["ts"] for e in ev)
    t1 = max(e["ts"] + e["dur"] for e in ev)
    return len(ev), sum(e["dur"] for e in ev), t1 - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", default="1,2,4,7,16", help="batches per encoder pass (E)")
    ap.add_argument("--rounds", type=int, default=3, help="timing rounds, each over every E")
    ap.add_argument("--reps", type=int, default=8, help="timed calls per round and E")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("group_encode.py needs a CUDA device")
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    Es = [int(x) for x in args.passes.split(",")]
    out_dir = args.out or os.path.join(os.environ.get("TMPDIR", "/tmp"), "group_encode")
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    wav = torch.randn(max(Es) * B, L, generator=g).to(dev)
    lens = torch.linspace(1.0, 0.5, B).repeat(max(Es)).to(dev)
    res = dict(card=card, batch=f"{B} x 10 s", passes=Es)
    for att in ("RoPEMHA", "RelPosMHAXL"):
        cfg = dict(CONFORMER_LARGE, attention_type=att)
        eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device=dev, parts=("fbank", "cnn", "encoder"))
        eng.set_poll_interval(0)  # one graph per call, as the group call replays
        outs = {E: torch.empty(E * B, eng.num_frames(L)[1], cfg["d_model"], device=dev) for E in Es}
        calls = {E: (lambda E=E: eng.encode_wav(wav[:E * B], lens[:E * B], out=outs[E])) for E in Es}
        per = {E: [] for E in Es}
        for r in range(args.rounds):
            for E in (Es if r % 2 == 0 else Es[::-1]):
                calls[E]()  # (re)captures the graph for this shape
                torch.cuda.synchronize()
                per[E].append(_time(calls[E], args.reps) / E)
        rows = {}
        for E in Es:
            n, busy, span = _profile(calls[E], os.path.join(out_dir, f"group_encode_{att}_E{E}.pt.trace.json"))
            xs = sorted(per[E])
            rows[E] = dict(ms_per_batch=xs[len(xs) // 2], ms_per_batch_min=xs[0], ms_per_batch_max=xs[-1],
                           kernels_per_batch=n / E, kernel_us_per_batch=busy / E, span_us_per_batch=span / E)
            print(f"{att:12s} E={E:2d}: {rows[E]}")
        base = rows[Es[0]]["ms_per_batch"]
        for E in Es:
            rows[E]["gain_vs_E%d" % Es[0]] = 1.0 - rows[E]["ms_per_batch"] / base
        res[att] = rows
        del eng
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(os.path.join(args.out, "group_encode.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
