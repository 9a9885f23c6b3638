"""Time the transducer beam search (csrc/transducer.cu, sbk_transducer_beam) on 32 x 10 s (T = 251) with the LibriSpeech
transducer recipe's sizes (joint 640, LSTM 512, 1000 tokens, seeded weights) at beam 10 and beam 4 (nbest 1, state_beam and
expand_beam 2.3): the device search alone (CUDA events, median and range over --iters calls after warm-up), its rounds,
pops, pops per frame, prediction-network steps and grid barriers, and the time per round; then
EncoderDecoderASR.transcribe_batch (wav -> words) with a beam-10 decoder on the fixture's LibriSpeech transducer model
(12-layer Conformer, tests/golden/transducer.pt "e2e") on 32 x 10 s.  Prints one JSON line (--out DIR also writes it) with
the card name and power limit read in the same run.

    python tools/transducer_beam.py [--iters 20] [--out DIR]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import test_gpu_transducer as TG  # noqa: E402
import test_gpu_transducer_beam as TB  # noqa: E402
import transducer_oracle as TO  # noqa: E402
from transducer_greedy import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    name, power = card()
    J, H, V = TO.RECIPE_SIZES["librispeech"]
    B, T = 32, 251
    res = dict(card=name, power_limit=power, B=B, T=T, joint=J, hidden=H, vocab=V)
    for beam in (10, 4):
        s, W, _ = TB.build(J, H, V, 0, beam, 1)
        tn = TO.seeded_tn(7, B, T, W).cuda()
        d = s.device_search(tn.device)
        r = d.beam(tn, 0, beam, 1, 2.3, 2.3, want_stats=True)
        torch.cuda.synchronize()
        rounds, pops, steps, barriers = r["stats"].tolist()
        search = timed(lambda: d.beam(tn, 0, beam, 1, 2.3, 2.3), args.iters)
        decode = timed(lambda: s(tn), args.iters)
        res[f"beam{beam}"] = dict(rounds=rounds, pops=pops, pops_per_frame=pops / (B * T), pn_steps=steps,
                                  grid_barriers=barriers, search=search, us_per_round=1e3 * search["median_ms"] / rounds,
                                  transducer_beam_search_decode=decode)
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    _, cfg, sd, w_enc, Wf, wav4, lens4 = TG._fixture_e2e()
    mods, parts = TG._transducer_modules(cfg, sd, w_enc, Wf)
    mods["decoder"] = TB._beam_decoder(parts)
    asr = EncoderDecoderASR(modules=mods, hparams={"tokenizer": None, "transducer_beam_search": True},
                            run_opts={"device": "cuda:0"})
    wav, lens = wav4.repeat(8, 1).cuda(), lens4.repeat(8).cuda()
    toks = [len(h) for h in asr.transcribe_batch(wav, lens)[1]]
    res["transcribe_batch_beam10_12layer"] = dict(timed(lambda: asr.transcribe_batch(wav, lens), args.iters),
                                                  tokens_per_utt_mean=sum(toks) / len(toks))
    res["encode_batch_12layer"] = timed(lambda: asr.encode_batch(wav, lens), args.iters)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "transducer_beam.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
