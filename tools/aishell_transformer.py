"""Time the AISHELL-1 Transformer recipe's device path at 32 x 10 s (seeded train_ASR_transformer.yaml-sized weights):

* the 256-channel front-end kernels at T0 = 1001 (T1 = 501, T2 = 251), each alone: conv1 (1 -> 256 + LayerNorm) and conv2
  (the wgmma implicit GEMM, M = 32 * 251 * 20, N = 256, K = 2304, with its fused LayerNorm), from torch.profiler's kernel
  records over repeated calls, and both together with CUDA events; conv2's TFLOP/s over 2 * M * N * K;
* the same front-end in eager torch on the same GPU (fp16, cuDNN F.conv2d + layer_norm + leaky_relu, with the reflect
  padding and the layout changes the reference makes), with CUDA events, and its conv2 F.conv2d alone;
* EncoderDecoderASR.encode_batch and transcribe_batch with the recipe's test search (beam 10, CTC 0.4) over 48 decode
  steps, host waveforms in, token lists out.

Prints the card name and power limit read in the same run, then one JSON line (``--out DIR`` also writes it to a file).
Needs a GPU; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

B, L, STEPS, C = 32, 160000, 48, 256


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


def shapes(T0, F0=80):
    T1, F1 = (T0 - 1) // 2 + 1, (F0 - 1) // 2 + 1
    return T1, F1, (T1 - 1) // 2 + 1, (F1 - 1) // 2 + 1


def kernel_ms(fn, names, reps):
    """Mean device time (ms) per call of the kernels whose names contain each of `names`, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    tot = {n: 0.0 for n in names}
    for e in prof.events():
        for n in names:
            if n in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
                tot[n] += e.device_time / 1000.0
    return {n: t / reps for n, t in tot.items()}


def eager_front_end(sd, dev):
    """ConvolutionFrontEnd(out_channels=(256, 256)) in eager fp16 torch, the reference's ops: (x [B, T0, F0] fp16 ->
    [B, T2, F2 * 256], act1 NCHW for conv2 alone)"""
    w = {k: v.to(dev, torch.float16) for k, v in sd.items() if k.startswith("CNN.")}

    def block(x, i):  # x [B, C, F, T]
        p = f"CNN.convblock_{i}.convs."
        x = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), w[p + "conv_0.conv.weight"], w[p + "conv_0.conv.bias"], stride=2)
        x = x.permute(0, 3, 2, 1)  # [B, T, F, C]
        g = w[p + "norm_0.norm.weight"]
        return F.leaky_relu(F.layer_norm(x, g.shape, g, w[p + "norm_0.norm.bias"], 1e-5), 0.01)

    def run(x):
        a1 = block(x.transpose(1, 2).unsqueeze(1), 0)
        y = block(a1.permute(0, 3, 2, 1), 1)
        return y.reshape(y.shape[0], y.shape[1], -1)

    def conv2_only(a1):
        p = "CNN.convblock_1.convs."
        return F.conv2d(F.pad(a1, (1, 1, 1, 1), mode="reflect"), w[p + "conv_0.conv.weight"], w[p + "conv_0.conv.bias"],
                        stride=2)
    return run, conv2_only


def build_asr(sd, dev):
    """EncoderDecoderASR of the recipe's modules with its test search: beam 10, CTC 0.4"""
    from mirrors import build_mirror
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER
    m = build_mirror(AISHELL_TRANSFORMER, sd)
    kwargs = dict(min_decode_ratio=0.0, beam_size=10, using_eos_threshold=False, length_normalization=True)
    dec = m.searcher(kwargs, (STEPS + 0.5) / 251.0, scorers=dict(ctc=0.4))
    return EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=dec),
                             hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="timed calls per measurement")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("aishell_transformer.py needs a CUDA device")
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER, seeded_asr_state

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    sd = seeded_asr_state(AISHELL_TRANSFORMER, 0)
    T0 = 1 + L // 160
    T1, F1, T2, F2 = shapes(T0)
    conv2_flops = 2.0 * (B * T2 * F2) * C * (9 * C)
    feats = torch.randn(B, T0, 80, generator=g).to(dev)

    eng = AsrEngine(AISHELL_TRANSFORMER, sd, device=dev, parts=("cnn",))
    ours = eng.cnn(feats)
    fe_ms = _time(lambda: eng.cnn(feats), args.reps)
    k = kernel_ms(lambda: eng.cnn(feats), ("conv1c256_ln_kernel", "conv2c256_ln_kernel"), args.reps)
    run, conv2_only = eager_front_end(sd, dev)
    feats16 = feats.half()
    ref = run(feats16)
    act1 = torch.randn(B, C, F1, T1, generator=g).to(dev, torch.float16)
    conv2_only(act1)
    eager_ms = _time(lambda: run(feats16), args.reps)
    eager_conv2_ms = _time(lambda: conv2_only(act1), args.reps)
    err = float((ours - ref.float()).norm() / ref.float().norm())
    del eng
    torch.cuda.empty_cache()

    wav = torch.randn(B, L, generator=g)
    lens = torch.linspace(1.0, 0.5, B)
    asr = build_asr(sd, dev)
    asr.encode_batch(wav, lens)
    enc_ms = _time(lambda: asr.encode_batch(wav, lens), args.reps)
    asr.transcribe_batch(wav, lens)
    tb_ms = _time(lambda: asr.transcribe_batch(wav, lens), max(3, args.reps // 4))
    res = dict(card=card, batch=f"{B} x 10 s", conv1_ms=k["conv1c256_ln_kernel"], conv2_ms=k["conv2c256_ln_kernel"],
               conv2_tflops=conv2_flops / k["conv2c256_ln_kernel"] / 1e9, front_end_ms=fe_ms,
               eager_front_end_ms=eager_ms, eager_conv2_ms=eager_conv2_ms,
               eager_conv2_tflops=conv2_flops / eager_conv2_ms / 1e9, ours_vs_eager_fp16_rel=err,
               encode_batch_ms=enc_ms, transcribe_beam10_ctc_ms=tb_ms, decode_steps=STEPS)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "aishell_transformer.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
