"""Every diagnostic switch that selects a code path of libsbk.so (DESIGN.md section 8, "Diagnostic switches") must stay
parity-green: the switches are read once per process, so each variant runs the 2 s golden in its own interpreter -- fused
wav -> ids pipeline for one 32-utterance batch (weight-streaming decode) and a 3-batch group (96 live rows: tensor-core GEMM
decode projections, or the weight-streaming kernels with SBK_DEC_TC_ROWS=128) -- and must reproduce the reference's encoder
states (1e-3 rel-L2) and greedy tokens.  Every variant runs with both encoder attention types (RoPEMHA, RelPosMHAXL)."""
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

SCRIPT = r"""
import json, os, sys, torch
sys.path.insert(0, %r)
from speechbrain_b200.engine import AsrEngine
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
g = torch.load(os.path.join(%r, "tests", "golden", sys.argv[1] + ".pt"))
cfg = dict(CONFORMER_LARGE, attention_type=g["cfg"]["attention_type"])
eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device="cuda:0")
wav = g["wav"].repeat(16, 1).cuda(); lens = g["wav_lens"].repeat(16).cuda()
S = g["greedy_logits"].shape[1]
pred, score, enc, done = eng.transcribe_greedy_dev(wav, lens, S, 1, 2, want_enc=True)
rel = float((enc[:2].cpu().double() - g["enc_out"].double()).norm() / g["enc_out"].double().norm())
outs = [torch.empty(32, S, dtype=torch.int32, device="cuda") for _ in range(3)]
eng.transcribe_greedy_group_dev([wav] * 3, [lens] * 3, S, 1, 2, outs)
eng.set_poll_interval(0)  # and the whole-pipeline graph
outs2 = [torch.empty(32, S, dtype=torch.int32, device="cuda") for _ in range(3)]
eng.transcribe_greedy_group_dev([wav] * 3, [lens] * 3, S, 1, 2, outs2)
torch.cuda.synchronize()
print(json.dumps({"rel": rel, "finite": bool(torch.isfinite(enc).all()), "tok": pred[:2].cpu().tolist(),
                  "rows_equal": bool(all(torch.equal(pred[2 * i:2 * i + 2], pred[:2]) for i in range(16))),
                  "group_tok": outs[0][:2].cpu().tolist(),
                  "group_equal": bool(all(torch.equal(o, outs[0]) for o in outs) and all(torch.equal(a, b) for a, b in zip(outs, outs2)))}))
""" % (ROOT, ROOT)

VARIANTS = [{}, {"SBK_XATT_ROWMAJOR": "1"}, {"SBK_NO_GRAPH": "1"}, {"SBK_DEC_TC_ROWS": "1"}, {"SBK_DEC_PRIORITY": "0"},
            {"SBK_DEC_TC_ROWS": "128"}, {"SBK_XATT_ROWMAJOR": "1", "SBK_DEC_TC_ROWS": "128"},
            {"SBK_NO_GRAPH": "1", "SBK_DEC_TC_ROWS": "128"}]
GOLDENS = {"conformer_large_rope": "", "conformer_large_relpos": "-relpos"}  # golden -> test id suffix


def _env_id(env):
    return "+".join(k if v in ("0", "1") else f"{k}={v}" for k, v in sorted(env.items())) or "default"


@pytest.mark.parametrize("env,tag", [(e, t) for t in GOLDENS for e in VARIANTS],
                         ids=[_env_id(e) + s for s in GOLDENS.values() for e in VARIANTS])
def test_kernel_variant_parity(env, tag):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g = torch.load(os.path.join(ROOT, "tests", "golden", tag + ".pt"))
    full_env = dict(os.environ, **env)
    p = subprocess.run([sys.executable, "-c", SCRIPT, tag], env=full_env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    r = json.loads(p.stdout.strip().splitlines()[-1])
    print(tag, env, r)
    assert r["finite"] and r["rel"] < 1e-3
    assert r["tok"] == g["hyps"] and r["group_tok"] == g["hyps"] and r["rows_equal"] and r["group_equal"]


@pytest.mark.parametrize("env", [{"SBK_BEAM_SERIAL": "1"}, {"SBK_NO_GRAPH": "1"}, {"SBK_BEAM_RADIX": "1"}],
                         ids=lambda e: "+".join(sorted(e)))
def test_beam_variant_parity(env):
    """The beam-search goldens (beam 10 with every scorer combination, beam 66, coverage) with the scorer branch serialised,
    without the per-step CUDA graph, and with the radix-select beam kernel forced for every width."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    p = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_bench_shapes.py"), "-q", "-m", "gpu",
                        "-k", "beam", "-p", "no:cacheprovider"], env=dict(os.environ, **env), capture_output=True, text=True,
                       timeout=900, cwd=ROOT)
    print(p.stdout[-1500:])
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-1000:]
