"""Event-timed decoder step at the bench shape: one 32 x 10 s batch is encoded once and replicated to `rows` hypotheses, then

    step time = (greedy_from_enc at 48 steps - greedy_from_enc at 1 step) / 47

which removes the one-off cross-attention K/V projection.  Early exit is off (set_poll_interval(0)), so every call runs
exactly its steps.  Prints the median and range over the repeats for each row count; 224 rows is the bench group
(7 batches decoded together), 160 is beam10_lm's 16 x 10 hypotheses.

    python tools/decode_step.py [--rows 224 160 96] [--repeats 9] [--att RoPEMHA] [--lib path/to/libsbk.so]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import speechbrain_b200._lib as _lib  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, nargs="+", default=[224, 160, 96])
ap.add_argument("--repeats", type=int, default=9)
ap.add_argument("--steps", type=int, default=48)
ap.add_argument("--att", default="RoPEMHA")
ap.add_argument("--lib", default=None, help="load this libsbk.so instead of the package's (A/B of two builds)")
args = ap.parse_args()
if args.lib:
    _lib.LIB_PATH = os.path.abspath(args.lib)

from speechbrain_b200.engine import AsrEngine  # noqa: E402
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state  # noqa: E402

B, BOS, EOS = 32, 1, 2
cfg = dict(CONFORMER_LARGE, attention_type=args.att)
eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device="cuda:0")
eng.set_poll_interval(0)
g = torch.Generator().manual_seed(1234)
wav = torch.randn(B, 160000, generator=g).cuda()
lens = torch.ones(B).cuda()
enc = eng.encode_wav(wav, lens)


def call_ms(enc_r, lens_r, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    eng.greedy_from_enc(enc_r, lens_r, steps, BOS, EOS)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


props = torch.cuda.get_device_properties(0)
res = {"gpu": props.name, "att": args.att, "steps": args.steps, "rows": {}}
for rows in args.rows:
    assert rows % B == 0, "rows must be a multiple of the 32-utterance batch"
    enc_r = enc.repeat(rows // B, 1, 1).contiguous()
    lens_r = lens.repeat(rows // B).contiguous()
    for _ in range(3):  # warm-up: step graph capture, module load
        call_ms(enc_r, lens_r, args.steps)
        call_ms(enc_r, lens_r, 1)
    per = []
    for _ in range(args.repeats):
        full = call_ms(enc_r, lens_r, args.steps)
        one = call_ms(enc_r, lens_r, 1)
        per.append((full - one) / (args.steps - 1) * 1e3)
    res["rows"][rows] = {"median_us": statistics.median(per), "min_us": min(per), "max_us": max(per), "n": len(per)}
    print(f"rows={rows:4d}: decode step {statistics.median(per):8.1f} us  (min {min(per):.1f}, max {max(per):.1f}, "
          f"{len(per)} repeats)", flush=True)
print(json.dumps(res))
