"""Event-timed encoder (wav -> encoder states, 32 x 10 s) of Branchformer-L (18 layers, csgu_linear_units 3072) and
Conformer-L (12 layers) in one process, alternated, median of --repeats calls each; then the CSGU kernels alone from a
torch.profiler run of one Branchformer-L encode, against a device-to-device copy of the bytes the CSGU must move at least
(read u [B*T, C] fp16, write g [B*T, C/2] fp16).  Prints the GPU name and power limit with the numbers.

    python tools/branchformer_encode.py [--repeats 9] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from speechbrain_b200.engine import AsrEngine  # noqa: E402
from speechbrain_b200.utils.seeded_init import (BRANCHFORMER_LARGE, CONFORMER_LARGE, scale_csgu_conv,  # noqa: E402
                                                seeded_asr_state)


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def time_call(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--out", default=None, help="directory for the JSON result (default: stdout only)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    B, L = args.batch, 160000
    g = torch.Generator().manual_seed(5)
    wav = torch.randn(B, L, generator=g).to(dev)
    lens = torch.linspace(1.0, 0.5, B).to(dev)
    engines = {}
    for name, cfg in (("branchformer_large", BRANCHFORMER_LARGE), ("conformer_large", CONFORMER_LARGE)):
        sd = scale_csgu_conv(seeded_asr_state(cfg, 0))
        engines[name] = AsrEngine(cfg, sd, device=dev, parts=("fbank", "cnn", "encoder"))
    out = {n: torch.empty(B, 251, c["d_model"], device=dev) for n, c in (("branchformer_large", BRANCHFORMER_LARGE),
                                                                          ("conformer_large", CONFORMER_LARGE))}
    for n, e in engines.items():  # warm-up: workspace, modules, tensor maps
        for _ in range(3):
            e.encode_wav(wav, lens, out[n])
    torch.cuda.synchronize()
    ms = {n: [] for n in engines}
    for _ in range(args.repeats):
        for n, e in engines.items():
            ms[n].append(time_call(lambda: e.encode_wav(wav, lens, out[n]), 3))
    med = {n: sorted(v)[len(v) // 2] for n, v in ms.items()}
    # CSGU kernels alone: torch.profiler over one Branchformer encode
    from torch.profiler import ProfilerActivity, profile
    e = engines["branchformer_large"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.encode_wav(wav, lens, out["branchformer_large"])
        torch.cuda.synchronize()
    csgu_us = {}
    for ev in prof.events():
        if "csgu" in ev.name and ev.device_type.name == "CUDA":
            csgu_us[ev.name.split("(")[0]] = csgu_us.get(ev.name.split("(")[0], 0.0) + ev.device_time
    L_enc, C, T = BRANCHFORMER_LARGE["num_encoder_layers"], BRANCHFORMER_LARGE["csgu_linear_units"], 251
    per_layer_bytes = B * T * C * 2 + B * T * (C // 2) * 2
    csgu_s = sum(csgu_us.values()) * 1e-6 / L_enc
    # device-to-device copy of the same bytes (half read, half written)
    src = torch.empty(per_layer_bytes // 2, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    for _ in range(5):
        dst.copy_(src)
    copy_ms = sorted(time_call(lambda: dst.copy_(src), 20) for _ in range(7))[3]
    copy_bw = 2 * src.numel() / (copy_ms * 1e-3)
    csgu_bw = per_layer_bytes / csgu_s
    res = dict(gpu=gpu_info(), batch=f"{B} x 10 s (T = {T})", repeats=args.repeats,
               encoder_ms={n: round(v, 3) for n, v in med.items()}, encoder_ms_all={n: [round(x, 3) for x in v] for n, v in ms.items()},
               csgu_us_per_layer={k: round(v / L_enc, 2) for k, v in csgu_us.items()},
               csgu_min_bytes_per_layer=per_layer_bytes, csgu_GBps=round(csgu_bw / 1e9, 1),
               copy_GBps=round(copy_bw / 1e9, 1), csgu_share_of_copy=round(csgu_bw / copy_bw, 3))
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "branchformer_encode.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
