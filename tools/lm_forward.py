"""Event-timed TransformerLM whole-sequence forward against the KV-cached step path on the same tokens.

    forward: TransformerLM.forward(tokens)                   -> logits [n, s, vocab]   (one pass of n * s-row GEMMs)
    step:    AsrEngine.lm_rescore(tokens, lens, T = 1.0)      -> scores [n]             (s - 1 dependent LM steps)

Recipe-size LM (12 x 768, 12 heads, d_ffn 3072, vocab 5000, seeded weights), full-length sequences (bos = 1, random ids), so
both paths see all n * s positions.  The two calls do not produce the same output: the step path also runs the per-step
log_softmax and score kernels the rescorer needs, the forward writes all n * s * vocab logits.  Prints the median and range
over the repeats per shape, the card and its power limit.

    python tools/lm_forward.py [--shapes 64x48 16x128] [--repeats 11]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM  # noqa: E402
from speechbrain_b200.utils.seeded_init import seeded_state_dict  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--shapes", nargs="+", default=["64x48", "16x128"], help="n x s")
ap.add_argument("--repeats", type=int, default=11)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("tools/lm_forward.py: needs a CUDA device")

dev = torch.device("cuda:0")
lm = TransformerLM(vocab=5000, d_model=768, nhead=12, num_encoder_layers=12, num_decoder_layers=0, d_ffn=3072, dropout=0.0,
                   activation=torch.nn.GELU, normalize_before=False)
lm.load_state_dict(seeded_state_dict(lm, seed=1))
eng = lm._get_engine(dev)


def timed_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1)


def stats(v):
    return {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v), "n": len(v)}


try:
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
except Exception as e:  # the timings stand without it; say why it is missing
    smi = f"nvidia-smi unavailable ({e})"
res = {"gpu": torch.cuda.get_device_properties(0).name, "nvidia_smi": smi, "shapes": {}}
g = torch.Generator().manual_seed(7)
for shape in args.shapes:
    n, s = (int(x) for x in shape.split("x"))
    tokens = torch.randint(3, 5000, (n, s), generator=g)
    tokens[:, 0] = 1
    td = tokens.to(dev)
    lens = torch.full((n,), s, dtype=torch.int32, device=dev)
    fwd = lambda: lm(td)  # noqa: E731
    step = lambda: eng.lm_rescore(td, lens, 1.0, 0)  # noqa: E731
    for _ in range(3):  # warm-up: module load, workspaces
        fwd()
        step()
    f_ms, s_ms = [], []
    for _ in range(args.repeats):  # alternated, so both see the same clock / neighbours
        f_ms.append(timed_ms(fwd))
        s_ms.append(timed_ms(step))
    res["shapes"][shape] = {"forward": stats(f_ms), "step_path": stats(s_ms),
                            "speedup": statistics.median(s_ms) / statistics.median(f_ms)}
    print(f"n={n:3d} s={s:4d}: forward {statistics.median(f_ms):8.2f} ms (min {min(f_ms):.2f}, max {max(f_ms):.2f})   "
          f"step path {statistics.median(s_ms):8.2f} ms (min {min(s_ms):.2f}, max {max(s_ms):.2f})   "
          f"x{statistics.median(s_ms) / statistics.median(f_ms):.1f}", flush=True)
print(smi)
print(json.dumps(res))
