"""Event-timed encoder (wav -> encoder states, 32 x 10 s) of HyperConformer-22M (10 layers, HyperMixing with 8 heads of 32
channels, k = 128) and of the same model with attention_type="RoPEMHA", in one process, alternated, median of --repeats
calls each; then the three HyperMixing kernels alone from a torch.profiler run of one HyperConformer encode, next to the
FLOPs and bytes counted from the shapes.  Prints the GPU name and power limit with the numbers.

    python tools/hyperconformer_encode.py [--repeats 9] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from speechbrain_b200.engine import AsrEngine  # noqa: E402
from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M, scale_hypernet, seeded_asr_state  # noqa: E402


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
    B, L, T = args.batch, 160000, 251
    g = torch.Generator().manual_seed(5)
    wav = torch.randn(B, L, generator=g).to(dev)
    lens = torch.linspace(1.0, 0.5, B).to(dev)
    cfgs = {"hyperconformer_22M": HYPERCONFORMER_22M, "rope_22M": dict(HYPERCONFORMER_22M, attention_type="RoPEMHA")}
    engines = {n: AsrEngine(c, scale_hypernet(seeded_asr_state(c, 0)), device=dev, parts=("fbank", "cnn", "encoder"))
               for n, c in cfgs.items()}
    out = {n: torch.empty(B, T, c["d_model"], device=dev) for n, c in cfgs.items()}
    for n, e in engines.items():  # warm-up: workspace, modules, tensor maps
        for _ in range(3):
            e.encode_wav(wav, lens, out[n])
    torch.cuda.synchronize()
    ms = {n: [] for n in engines}
    for _ in range(args.repeats):
        for n, e in engines.items():
            ms[n].append(time_call(lambda: e.encode_wav(wav, lens, out[n]), 3))
    med = {n: sorted(v)[len(v) // 2] for n, v in ms.items()}
    # the HyperMixing kernels alone: torch.profiler over one HyperConformer encode
    from torch.profiler import ProfilerActivity, profile
    e = engines["hyperconformer_22M"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.encode_wav(wav, lens, out["hyperconformer_22M"])
        torch.cuda.synchronize()
    hm_us = {}
    for ev in prof.events():
        if "hypermix" in ev.name and ev.device_type.name == "CUDA":
            key = ev.name.split("(")[0].replace("void ", "")
            hm_us[key] = hm_us.get(key, 0.0) + ev.device_time
    c = HYPERCONFORMER_22M
    n_layers, d, M = c["num_encoder_layers"], c["d_model"], c["nhead"]
    e_, k = d // M, c["d_ffn"] // M
    rows = int(round(float(lens.sum().item()) * T))  # valid frames (padded frames skip the reduction but not the expansion)
    rows_all = B * T
    # counted from shapes, per layer: each hypernetwork e -> e -> k per head and frame; reduce runs w1_gen + xm^T W1 on the
    # valid frames, expand runs w2_gen + W2 G^T on every frame
    mac_gen = M * (e_ * e_ + e_ * k)
    flop_reduce = 2 * rows * (mac_gen + M * e_ * k)
    flop_expand = 2 * rows_all * (mac_gen + M * e_ * k)
    bytes_min = 2 * rows_all * d * 2 + 2 * rows_all * d * 4  # h16 read twice, x fp32 read and written
    bytes_w_materialised = 2 * 2 * rows_all * M * k * 2      # W1 and W2 written and read back in fp16
    hm_s = sum(hm_us.values()) * 1e-6 / n_layers
    res = dict(gpu=gpu_info(), batch=f"{B} x 10 s (T = {T}, {rows} valid frames)", repeats=args.repeats,
               encoder_ms={n: round(v, 3) for n, v in med.items()}, encoder_ms_all={n: [round(x, 3) for x in v] for n, v in ms.items()},
               hypermix_us_per_layer={k_: round(v / n_layers, 2) for k_, v in hm_us.items()},
               hypermix_us_per_layer_total=round(hm_s * 1e6, 2),
               counted_gflop_per_layer=dict(reduce=round(flop_reduce / 1e9, 3), expand=round(flop_expand / 1e9, 3)),
               counted_min_MB_per_layer=round(bytes_min / 1e6, 1), counted_W1W2_materialised_MB_per_layer=round(bytes_w_materialised / 1e6, 1),
               achieved_TFLOPs=round((flop_reduce + flop_expand) / hm_s / 1e12, 2) if hm_s > 0 else None,
               achieved_GBps_min_bytes=round(bytes_min / hm_s / 1e9, 1) if hm_s > 0 else None)
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "hyperconformer_encode.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
