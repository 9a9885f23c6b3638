"""Time the Transformer recipe's device path at 32 x 10 s (seeded transformer.yaml-sized weights), with CUDA events:

* Transformer-L encode (Fbank -> CMVN -> 3-block CNN -> 12 regularMHA layers) against Conformer-L (RoPEMHA), in one process,
  alternated round by round;
* the front-end kernels alone (3-block CNN on fp32 features), with TFLOP/s over the operations counted from the shapes
  (multiply-adds x 2 of the three blocks' convolutions);
* EncoderDecoderASR.transcribe_batch with the recipe's test search at beam 10 (CTC 0.4 + TransformerLM 0.6, the 12 x 768 LM)
  over 48 decode steps, host waveforms in, token lists out.

Prints the card name and power limit read in the same run, then one JSON line (``--out DIR`` also writes it to a file).
Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B, L, STEPS = 32, 160000, 48


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


def front_end_flops(Bn, T0, F0=80, C=64):
    T1, F1 = (T0 - 1) // 2 + 1, (F0 - 1) // 2 + 1
    T2, F2 = (T1 - 1) // 2 + 1, (F1 - 1) // 2 + 1
    macs = Bn * T1 * F1 * C * 25 + Bn * T2 * F2 * C * 25 * C + Bn * T2 * F2 * 2 * C * C
    return 2.0 * macs


def build_asr(sd, dev):
    """EncoderDecoderASR of the recipe's modules with its test search: beam 10, CTC 0.4 + the 12 x 768 TransformerLM 0.6"""
    from mirrors import build_mirror
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE
    m = build_mirror(TRANSFORMER_LARGE, sd)
    kwargs = dict(min_decode_ratio=0.0, beam_size=10, temperature=1.15, using_eos_threshold=False, length_normalization=True)
    dec = m.searcher(kwargs, (STEPS + 0.5) / 251.0, scorers=dict(ctc=0.4, transformerlm=0.6))
    return EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=dec),
                             hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternated encode rounds")
    ap.add_argument("--reps", type=int, default=10, help="timed calls per round / measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("transformer_encode.py needs a CUDA device")
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, TRANSFORMER_LARGE, seeded_asr_state

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    wav = torch.randn(B, L, generator=g)
    lens = torch.linspace(1.0, 0.5, B)
    wav_d, lens_d = wav.to(dev), lens.to(dev)
    sd_t = seeded_asr_state(TRANSFORMER_LARGE, 0)
    parts = ("fbank", "cnn", "encoder")
    eng_t = AsrEngine(TRANSFORMER_LARGE, sd_t, device=dev, parts=parts)
    eng_c = AsrEngine(CONFORMER_LARGE, seeded_asr_state(CONFORMER_LARGE, 0), device=dev, parts=parts)
    for e in (eng_t, eng_c):
        e.encode_wav(wav_d, lens_d)
    torch.cuda.synchronize()
    t_ms, c_ms = [], []
    for _ in range(args.rounds):
        t_ms.append(_time(lambda: eng_t.encode_wav(wav_d, lens_d), args.reps))
        c_ms.append(_time(lambda: eng_c.encode_wav(wav_d, lens_d), args.reps))
    # the front-end alone, on the features the Fbank stage produces for these waveforms
    T0 = 1 + L // 160
    feats = torch.randn(B, T0, 80, generator=g).to(dev)
    eng_t.cnn(feats)
    fe_ms = _time(lambda: eng_t.cnn(feats), args.reps * 5)
    flops = front_end_flops(B, T0)
    # transcribe_batch, beam 10 + CTC + LM
    asr = build_asr(sd_t, dev)
    asr.transcribe_batch(wav, lens)
    tb_ms = _time(lambda: asr.transcribe_batch(wav, lens), max(2, args.reps // 3))
    med = lambda xs: sorted(xs)[len(xs) // 2]  # noqa: E731
    res = dict(card=card, batch=f"{B} x 10 s", transformer_encode_ms=med(t_ms), conformer_encode_ms=med(c_ms),
               transformer_encode_rounds_ms=t_ms, conformer_encode_rounds_ms=c_ms, front_end_ms=fe_ms,
               front_end_tflops=flops / fe_ms / 1e9, front_end_share_of_encode=fe_ms / med(t_ms),
               transcribe_beam10_ctc_lm_ms=tb_ms, decode_steps=STEPS)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "transformer_encode.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
