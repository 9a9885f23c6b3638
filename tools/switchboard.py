"""Time the Switchboard transformer.yaml recipe's device path on seeded weights:

* the recipe's test search (beam 60, TransformerLM 0.3 with the 264-wide LM + CTC 0.3, temperature 1.0) over STEPS decode
  steps on 16 x 10 s: the searcher alone on encoder states, and EncoderDecoderASR.transcribe_batch (host waveforms in,
  token lists out);
* TransformerLM.forward at n = 64 sequences of s = 80 tokens.

Times are medians of CUDA-event-timed calls after a warm-up call.  Prints the card name and power limit read in the same
run, then one JSON line (``--out DIR`` also writes it to a file).  Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B, L, STEPS, BEAM = 16, 160000, 48, 60


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10, help="timed calls per measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("switchboard.py needs a CUDA device")
    from mirrors import build_mirror
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
    from speechbrain_b200.utils.seeded_init import SWITCHBOARD_LM, SWITCHBOARD_TRANSFORMER as CFG, seeded_asr_state
    from speechbrain_b200.utils.seeded_init import seeded_state_dict

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    sd = seeded_asr_state(CFG, 0)
    lm = TransformerLM(**SWITCHBOARD_LM, dropout=0.0, activation=torch.nn.ReLU)
    lm.load_state_dict(seeded_state_dict(lm, seed=1))

    tokens = torch.randint(3, 2000, (64, 80), generator=g)
    tokens[:, 0] = 1
    td = tokens.to(dev)
    lm(td)
    lm_ms = _time(lambda: lm(td), args.reps * 5)

    m = build_mirror(CFG, sd)
    kwargs = dict(min_decode_ratio=0.0, beam_size=BEAM, temperature=1.0, using_eos_threshold=False, eos_threshold=1.5,
                  length_normalization=True)
    dec = m.searcher(kwargs, (STEPS + 0.5) / 251.0, scorers=dict(transformerlm=0.3, ctc=0.3), lm=lm, lm_temperature=1.0,
                     scorer_beam_scale=0.3)
    asr = EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=dec),
                            hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})
    wav = torch.randn(B, L, generator=g)
    lens = torch.linspace(1.0, 0.5, B)
    enc = asr.encode_batch(wav, lens)
    lens_d = lens.to(dev)
    dec(enc, lens_d)
    search_ms = _time(lambda: dec(enc, lens_d), args.reps)
    asr.transcribe_batch(wav, lens)
    tb_ms = _time(lambda: asr.transcribe_batch(wav, lens), args.reps)
    res = dict(card=card, batch=f"{B} x 10 s", beam=BEAM, decode_steps=STEPS, beam60_lm_ctc_search_ms=search_ms,
               transcribe_beam60_lm_ctc_ms=tb_ms, lm_forward_n64_s80_ms=lm_ms)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "switchboard.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
