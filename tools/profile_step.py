"""One warm-up + one profiled pass of the bench workload.

    python tools/profile_step.py [att] [steps] [B] [G]             bracket for ncu --profile-from-start off
    python tools/profile_step.py [att] [steps] [B] [G] OUT_DIR     torch.profiler (CUDA activities): per-kernel table on
                                                                   stdout, trace in OUT_DIR/profile_step.pt.trace.json
"""
import json
import os
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from speechbrain_b200.engine import AsrEngine  # noqa: E402
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state  # noqa: E402

att = sys.argv[1] if len(sys.argv) > 1 else "RoPEMHA"
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 48
B = int(sys.argv[3]) if len(sys.argv) > 3 else 32
G = int(sys.argv[4]) if len(sys.argv) > 4 else 1  # > 1: G batches encoded in passes of up to 8 and decoded together
out_dir = sys.argv[5] if len(sys.argv) > 5 else None
cfg = dict(CONFORMER_LARGE, attention_type=att)
eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device="cuda:0")
g = torch.Generator().manual_seed(1234)
wav = torch.randn(B, 160000, generator=g).cuda()
lens = torch.ones(B).cuda()
outs = [torch.empty(B, steps, dtype=torch.int32, device="cuda") for _ in range(G)]


def run():
    if G == 1:
        eng.transcribe_greedy_dev(wav, lens, steps, 1, 2)
    else:
        eng.transcribe_greedy_group_dev([wav] * G, [lens] * G, steps, 1, 2, outs)


def kernel_table(trace_path):
    """name (template arguments kept, parameters dropped) -> launches, total us, share of the summed kernel time"""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    tot = defaultdict(float)
    cnt = defaultdict(int)
    t0, t1 = float("inf"), 0.0
    for e in ev:
        if e.get("cat") != "kernel":
            continue
        name = e["name"].split("(")[0].replace("void ", "").replace("sbk::", "")
        tot[name] += e["dur"]
        cnt[name] += 1
        t0, t1 = min(t0, e["ts"]), max(t1, e["ts"] + e["dur"])
    busy = sum(tot.values())
    print(f"{'kernel':<60} {'launches':>8} {'total us':>11} {'share':>7}")
    for name, us in sorted(tot.items(), key=lambda kv: -kv[1]):
        print(f"{name[:60]:<60} {cnt[name]:>8} {us:>11.1f} {100 * us / busy:>6.1f}%")
    print(f"{'sum of kernel times':<60} {sum(cnt.values()):>8} {busy:>11.1f}")
    print(f"first kernel start -> last kernel end: {t1 - t0:.1f} us")


for _ in range(2):
    run()
torch.cuda.synchronize()
if out_dir is None:
    torch.cuda.profiler.start()
    run()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
else:
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(out_dir, exist_ok=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    path = os.path.join(out_dir, "profile_step.pt.trace.json")
    prof.export_chrome_trace(path)
    print(f"{torch.cuda.get_device_name(0)}: {att}, {G} x {B} utterances, {steps} decode steps, one group call")
    kernel_table(path)
