"""Time the transducer greedy search (csrc/transducer.cu) on 32 x 10 s (T = 251) with the LibriSpeech transducer recipe's
sizes (joint 640, LSTM 512, 1000 tokens): the device search alone (CUDA events, median and range over --iters calls after
warm-up), its rounds and grid barriers per call and the emitted symbols per utterance; EncoderDecoderASR.transcribe_batch
end to end for the fixture's LibriSpeech transducer model (12-layer Conformer, tests/golden/transducer.pt "e2e", which
emits tokens) on 32 x 10 s; and, for comparison, the attention decoder's 48-step greedy decode of the same batch (the
Conformer-L engine of bench.py: encode + 48 steps minus encode alone).  Prints one JSON line (--out DIR also writes it)
with the card name and power limit read in the same run.

    python tools/transducer_greedy.py [--iters 20] [--out DIR]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_gpu_transducer as TG  # noqa: E402
import transducer_oracle as TO  # noqa: E402


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return dict(median_ms=statistics.median(ms), min_ms=min(ms), max_ms=max(ms), n=iters)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in q.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = card()
    J, H, V = TO.RECIPE_SIZES["librispeech"]
    s, W, _ = TG.build(J, H, V, 0)
    tn = TO.seeded_tn(7, 32, 251, W).cuda()
    dsearch = s.device_search(tn.device)
    r = dsearch.greedy(tn, 0, 5, want_stats=True)
    torch.cuda.synchronize()
    rounds, barriers = r["stats"].tolist()
    n_tok = r["n_tokens"].cpu().tolist()
    search = timed(lambda: dsearch.greedy(tn, 0, 5), args.iters)
    decode = timed(lambda: s(tn), args.iters)
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    fx, cfg, sd, w_enc, Wf, wav4, lens4 = TG._fixture_e2e()
    mods, _ = TG._transducer_modules(sd, w_enc, Wf)
    asr = EncoderDecoderASR(modules=mods, hparams={"tokenizer": None, "transducer_beam_search": True},
                            run_opts={"device": "cuda:0"})
    wav = wav4.repeat(8, 1).cuda()
    lens = lens4.repeat(8).cuda()
    e2e_tokens = [len(h) for h in asr.transcribe_batch(wav, lens)[1]]
    e2e = timed(lambda: asr.transcribe_batch(wav, lens), args.iters)
    enc_only = timed(lambda: asr.encode_batch(wav, lens), args.iters)
    eng = AsrEngine(CONFORMER_LARGE, seeded_asr_state(CONFORMER_LARGE, 0), device="cuda:0")
    att48 = timed(lambda: eng.transcribe_greedy_dev(wav, lens, 48, 1, 2), args.iters)
    att0 = timed(lambda: eng.encode_wav(wav, lens), args.iters)
    ctas, smem = dsearch.info()
    res = dict(card=name, power_limit=power, B=32, T=251, joint=J, hidden=H, vocab=V, ctas=ctas, smem_bytes_b1=smem,
               rounds=rounds, grid_barriers=barriers, emitted_per_utt=dict(mean=sum(n_tok) / len(n_tok), min=min(n_tok),
                                                                            max=max(n_tok)),
               search=search, transducer_greedy_decode=decode,
               transcribe_batch_12layer=dict(e2e, tokens_per_utt_mean=sum(e2e_tokens) / len(e2e_tokens)),
               encode_batch_12layer=enc_only, attention_greedy48=att48, attention_encode_only=att0,
               attention_decode48_ms=att48["median_ms"] - att0["median_ms"])
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "transducer_greedy.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
