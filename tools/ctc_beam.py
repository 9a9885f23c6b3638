"""Timing of the device CTC beam search (CTCBeamSearcher, csrc/ctc_beam.cu) on one GPU, with CUDA events after warm-up:

* the device search alone (token-count pre-pass, workspace, ctc_beam_kernel; `CTCBeamSearcher.search`) and the whole
  `decode_beams` call (search + host replay + finalize) on 32 x 251 synthetic frames, at the LibriSpeech CTC recipes'
  settings (31 symbols, beam 100, -12 / -1.2, no history pruning) and at the defaults on 5000 sentencepiece-style pieces;
* `EncoderASR.transcribe_batch` of the Branchformer CTC recipe (18 layers, d_model 256) with the recipe's beam search on
  32 x 10 s, and the same call with greedy decoding.

Every timed output is checked against the NumPy oracle (tests/ctc_beam_oracle.py).  Prints the card name, the power limit
and one JSON line; `--out DIR` also writes it to DIR/ctc_beam.json.  `--cpu-reference` instead times, on the CPU and on the
same posteriors, the reference searcher when `speechbrain` is importable, otherwise the NumPy oracle (bit-equal to it).

    python tools/ctc_beam.py [--iters 20] [--out DIR]
    python tools/ctc_beam.py --cpu-reference"""
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
import ctc_beam_oracle as CO  # noqa: E402

RECIPE = dict(blank_index=0, beam_size=100, beam_prune_logp=-12.0, token_prune_min_logp=-1.2, prune_history=False)
SPM = dict(blank_index=0)


def workloads():
    spm = CO.spm_vocab(5000, 0)
    active = list(range(11)) + [17, 40, 99, 512, 1024, 2048, 3001, 4999]
    lens = torch.linspace(1.0, 0.6, 32)
    return [("recipe_char31", CO.CHAR_VOCAB, RECIPE, CO.synthetic_log_probs(301, 32, 251, 31), lens),
            ("defaults_spm5000", spm, SPM, CO.synthetic_log_probs(302, 32, 251, 5000, peak=12.0, active=active), lens)]


def time_events(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return dict(median_ms=ts[len(ts) // 2], min_ms=ts[0], max_ms=ts[-1], iters=iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: stdout only)")
    ap.add_argument("--cpu-reference", action="store_true")
    args = ap.parse_args()
    res = {}
    if args.cpu_reference:   # the reference searcher when it is importable (PYTHONPATH), else the bit-equal NumPy oracle
        try:
            from speechbrain.decoders.ctc import CTCBeamSearcher as Ref
        except ImportError:
            Ref = None
        for name, vocab, params, lp, lens in workloads():
            kw = {k: v for k, v in params.items() if k != "blank_index"}
            t0 = time.perf_counter()
            if Ref is not None:
                Ref(vocab_list=vocab, **params)(lp, lens)
            else:
                CO.decode(lp, lens, vocab, 0, **kw)
            what = "reference CTCBeamSearcher" if Ref is not None else "NumPy oracle"
            res[name] = dict(cpu_seconds=time.perf_counter() - t0, what=what)
            print(f"{name}: CPU, {what}: {res[name]['cpu_seconds']:.2f} s")
        print(json.dumps(res))
        return
    if not torch.cuda.is_available():
        raise SystemExit("tools/ctc_beam.py: no CUDA device (timings are only taken on the GPU)")
    from test_gpu_ctc_beam import _branchformer_ctc_asr, check_hyps

    from speechbrain_b200.decoders.ctc import CTCBeamSearcher, ctc_greedy_decode
    dev = torch.device("cuda:0")
    res["card"] = torch.cuda.get_device_name(0)
    try:
        res["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        res["power_limit"] = f"unavailable ({e})"
    print(f"card {res['card']}, power limit {res['power_limit']}")
    for name, vocab, params, lp, lens in workloads():
        s = CTCBeamSearcher(vocab_list=vocab, **params)
        x, ld = lp.to(dev), lens.to(dev)
        T = lp.shape[1]
        nlen = [len(range(T)[:n]) for n in (T * lens).numpy().astype(int).tolist()]
        out = CO.as_tuples(s(x, ld))
        kw = {k: v for k, v in params.items() if k != "blank_index"}
        check_hyps(name, CO.as_tuples(CO.decode(lp, lens, vocab, 0, **kw)), out)
        res[name] = dict(search=time_events(lambda: s.search(x, nlen), args.iters),
                         decode_beams=time_events(lambda: s(x, ld), max(3, args.iters // 4)), frames=sum(nlen))
        print(f"{name}: device search {res[name]['search']['median_ms']:.2f} ms, decode_beams "
              f"{res[name]['decode_beams']['median_ms']:.2f} ms (32 utterances, {sum(nlen)} frames); equal to the oracle")
    asr, _, _ = _branchformer_ctc_asr(dev, CTCBeamSearcher, dict(test_beam_search=dict(RECIPE)))
    g = torch.Generator().manual_seed(5)
    wav = torch.randn(32, 160000, generator=g)
    lens = torch.linspace(1.0, 0.7, 32)
    for b in range(32):
        wav[b, int(round(float(lens[b]) * 160000)):] = 0
    wav_d, lens_d = wav.to(dev), lens.to(dev)
    words, hyps = asr.transcribe_batch(wav_d, lens_d)
    lpd = asr.encode_batch(wav_d, lens_d).cpu()
    check_hyps("EncoderASR 32x10s", CO.as_tuples(CO.decode(lpd, lens, CO.CHAR_VOCAB, 0, **{k: v for k, v in RECIPE.items() if k != "blank_index"})),
               CO.as_tuples(hyps))
    res["encoder_asr_branchformer_ctc_32x10s"] = dict(beam=time_events(lambda: asr.transcribe_batch(wav_d, lens_d), 10),
                                                      encode_batch=time_events(lambda: asr.encode_batch(wav_d, lens_d), 10))
    greedy, _, _ = _branchformer_ctc_asr(dev, __import__("functools").partial(ctc_greedy_decode, blank_id=0), {})
    res["encoder_asr_branchformer_ctc_32x10s"]["greedy"] = time_events(lambda: greedy.transcribe_batch(wav_d, lens_d), 10)
    r = res["encoder_asr_branchformer_ctc_32x10s"]
    print(f"EncoderASR.transcribe_batch Branchformer CTC 32 x 10 s: beam {r['beam']['median_ms']:.1f} ms, greedy "
          f"{r['greedy']['median_ms']:.1f} ms, encode_batch {r['encode_batch']['median_ms']:.1f} ms; beam equal to the oracle")
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ctc_beam.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
