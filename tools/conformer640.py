"""Timings of the d_model 640 Conformer (Libriheavy conformer_large: 14 layers, 8 heads of 80, RelPosMHAXL) on one GPU, on
seeded weights, 32 x 10 s:

* encode (wav -> encoder states), and encode + 48 greedy steps (AsrEngine.transcribe_greedy_dev), CUDA events around
  whole calls after warm-up, median of --reps;
* one step of the recipe's test search, beam 66 + TransformerLM 0.6 + CTC 0.4: (time of a 24-step search - time of a 1-step
  search) / 23 on the same encoder states;
* the attention kernels alone through the test hooks, CUDA events over 50 launches, median of 5 windows: RelPosMHAXL
  encoder attention at head width 80 and 64 on the same shapes (B = 32, 8 heads, T = 251 and 2500), and decode-step
  cross-attention with the templated kernel at 80 and 64 and the generic kernel at 60 (the widest it takes);
* --profile: a separate torch.profiler run of one encode (wav -> encoder states) at head width 80 and one of the same
  encoder at 8 heads of 64 (d_model 512), the encoder attention kernel's total CUDA time from each trace.

Prints one JSON object with the GPU name and power limit read in the same run."""
import argparse
import ctypes
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def events(fn, n, windows=5):
    """median over windows of the mean time (ms) of n calls of fn"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(windows):
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / n)
    return sorted(out)[len(out) // 2]


def enc_attention(dev, B, T, H, dh):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    d = H * dh
    qkv = torch.randn(B * T, 3 * d, device=dev).half()
    out = torch.empty(B * T, d, device=dev, dtype=torch.float16)
    u = 0.1 * torch.randn(d, device=dev)
    P = torch.randn(T, d, device=dev).half()
    lens = torch.full((B,), T, dtype=torch.int32, device=dev)
    lens[1::2] = int(0.7 * T)
    f = lambda: check(lib().sbk_encoder_attention_test(ptr(qkv), B, T, H, dh, ptr(lens), 1, ptr(u), ptr(u), ptr(P),  # noqa: E731
                                                       ctypes.c_float(1 / math.sqrt(d)), 0, -1, ptr(out), stream_ptr(dev)),
                      "encoder attention")
    return events(f, 50) * 1000


def dec_cross_attention(dev, rows, rpu, T, H, dh):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    d, U = H * dh, rows // rpu
    q = torch.randn(rows, d, device=dev).half()
    kv = torch.randn(U, T, 2 * d, device=dev).half()
    out = torch.empty(rows, d, device=dev, dtype=torch.float16)
    lens = torch.full((U,), T, dtype=torch.int32, device=dev)
    kb, vb = ctypes.c_void_p(kv.data_ptr()), ctypes.c_void_p(kv.data_ptr() + 2 * d)
    f = lambda: check(lib().sbk_dec_attention_test(ptr(q), d, kb, vb, ctypes.c_longlong(T * 2 * d), 2 * d, 0, rpu, rows, H,  # noqa: E731
                                                   dh, T, -1, ptr(lens), None, None, 0, 0, ptr(out), d, stream_ptr(dev)),
                      "decode attention")
    return events(f, 50) * 1000


def model_times(dev, B, reps):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import conformer640_oracle as CO
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_640
    cfg = CONFORMER_640
    sd = CO.state(cfg)
    eng = AsrEngine(cfg, sd, device=str(dev))
    g = torch.Generator().manual_seed(0)
    wav = torch.randn(B, 160000, generator=g).to(dev)
    lens = torch.ones(B, device=dev)
    res = {}
    res["encode_ms"] = events(lambda: eng.encode_wav(wav, lens), 1, reps)
    res["encode_greedy48_ms"] = events(lambda: eng.transcribe_greedy_dev(wav, lens, 48, CO.BOS, CO.EOS), 1, reps)
    enc = eng.encode_wav(wav, lens)
    import importlib
    T = importlib.import_module("test_gpu_conformer640")
    times = {}
    for steps in (1, 24):
        _, _, _, bs = T._search_modules(cfg, 66, 0.6, 0.4, (steps + 0.5) / enc.shape[1])
        times[steps] = events(lambda: bs(enc, lens), 1, reps)
    res["beam66_lm_ctc_step_ms"] = (times[24] - times[1]) / 23
    return res


def profile_encode(dev, out_dir):
    from torch.profiler import ProfilerActivity, profile

    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_640, seeded_asr_state
    res = {}
    wav = torch.randn(32, 160000, device=dev)
    lens = torch.ones(32, device=dev)
    for name, cfg in (("head80", CONFORMER_640), ("head64", dict(CONFORMER_640, name="c512", d_model=512, input_size=640))):
        eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device=str(dev))
        eng.encode_wav(wav, lens)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.encode_wav(wav, lens)
            torch.cuda.synchronize()
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, f"conformer640_{name}.json"))
        att = [e for e in prof.key_averages() if "encoder_attention_kernel" in e.key]
        res[f"encoder_attention_{name}_us_per_encode"] = sum(e.device_time_total for e in att)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="only the torch.profiler run")
    ap.add_argument("--out-dir", default=None, help="where --profile writes its traces")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conformer640.py measures on a GPU; none found")
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info()}
    if args.profile:
        res.update(profile_encode(dev, args.out_dir))
    else:
        for T in (251, 2500):
            for dh in (80, 64):
                res[f"enc_attention_relpos_B32_H8_T{T}_dh{dh}_us"] = enc_attention(dev, 32, T, 8, dh)
        for rows, rpu, T in ((320, 10, 251), (66, 66, 2500)):
            for dh in (80, 64, 60):
                res[f"dec_cross_attention_rows{rows}_T{T}_dh{dh}_us"] = dec_cross_attention(dev, rows, rpu, T, 8, dh)
        res.update(model_times(dev, args.batch, args.reps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
