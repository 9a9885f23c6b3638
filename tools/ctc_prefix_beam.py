"""Timing of the device CTC prefix beam search (CTCPrefixBeamSearcher, csrc/ctc_prefix_beam.cu) on one GPU, with CUDA
events after warm-up (median, min and max over the timed runs), on the two workloads of the CTC beam table in DESIGN.md
section 9 (32 x 251 synthetic frames, relative lengths 1.0 ... 0.6): the LibriSpeech CTC recipes' settings on 31 symbols
(beam 100, -12 / -1.2, no history pruning) and the defaults on 5000 sentencepiece-style pieces.  Per workload:

* the device search alone (token-count pre-pass, workspace, ctc_prefix_beam_kernel; `CTCPrefixBeamSearcher.search`);
* `decode_beams`, and its host parts: the replay of the final beams and finalize_decoding (host clock).

Every timed output is checked against the NumPy oracle (tests/ctc_prefix_beam_oracle.py).  Prints the card name, the
power limit and one JSON line; `--out DIR` also writes it to DIR/ctc_prefix_beam.json.  `--cpu-reference` instead times,
on the CPU and on the same posteriors, the reference searcher when `speechbrain` is importable, otherwise the oracle.

    python tools/ctc_prefix_beam.py [--iters 10] [--out DIR]
    python tools/ctc_prefix_beam.py --cpu-reference"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from ctc_beam import time_events, workloads  # noqa: E402

import ctc_prefix_beam_oracle as PO  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: stdout only)")
    ap.add_argument("--cpu-reference", action="store_true")
    args = ap.parse_args()
    res = {}
    if args.cpu_reference:
        try:
            from speechbrain.decoders.ctc import CTCPrefixBeamSearcher as Ref
        except ImportError:
            Ref = None
        for name, vocab, params, lp, lens in workloads():
            t0 = time.perf_counter()
            if Ref is not None:
                Ref(vocab_list=vocab, **params)(lp, lens)
            else:
                PO.decode(lp, lens, vocab, 0, **{k: v for k, v in params.items() if k != "blank_index"})
            what = "reference CTCPrefixBeamSearcher" if Ref is not None else "NumPy oracle"
            res[name] = dict(cpu_seconds=time.perf_counter() - t0, what=what)
            print(f"{name}: CPU, {what}: {res[name]['cpu_seconds']:.2f} s")
        print(json.dumps(res))
        return
    if not torch.cuda.is_available():
        raise SystemExit("tools/ctc_prefix_beam.py: no CUDA device (timings are only taken on the GPU)")
    from test_gpu_ctc_prefix_beam import check, tuples
    from test_ctc_prefix_beam_golden import oracle

    from speechbrain_b200.decoders.ctc import CTCPrefixBeamSearcher
    dev = torch.device("cuda:0")
    res["card"] = torch.cuda.get_device_name(0)
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        res["power_limit"] = f"unavailable ({e})"
    print(f"card {res['card']}, power limit {res['power_limit']}")
    for name, vocab, params, lp, lens in workloads():
        s = CTCPrefixBeamSearcher(vocab_list=vocab, **params)
        x, ld = lp.to(dev), lens.to(dev)
        T = lp.shape[1]
        nlen = [len(range(T)[:n]) for n in (T * lens).numpy().astype(int).tolist()]
        worst = check(name, oracle(lp, lens, vocab, params), tuples(s(x, ld)))
        out = [t.cpu().numpy() for t in s.search(x, nlen)]
        fb, par, tok, score, nfin = out
        host = []
        for _ in range(3):
            t0 = time.perf_counter()
            beams = [s._replay(nlen[b], fb[b], par[b], tok[b], score[b], int(nfin[b])) for b in range(len(nlen))]
            t1 = time.perf_counter()
            [s._finalize(bm) for bm in beams]
            host.append(((t1 - t0) * 1e3, (time.perf_counter() - t1) * 1e3))
        host.sort()
        res[name] = dict(search=time_events(lambda: s.search(x, nlen), args.iters),
                         decode_beams=time_events(lambda: s(x, ld), args.iters),
                         replay_ms=host[1][0], finalize_ms=host[1][1], frames=sum(nlen), worst_score_diff=worst)
        r = res[name]
        print(f"{name}: device search {r['search']['median_ms']:.2f} ms, decode_beams {r['decode_beams']['median_ms']:.2f} ms "
              f"(replay {r['replay_ms']:.2f} ms, finalize {r['finalize_ms']:.2f} ms; 32 utterances, {sum(nlen)} frames); "
              f"equal to the oracle (worst score difference {worst:.1e})")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ctc_prefix_beam.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
