"""The 2 s goldens through both decode-projection back ends: the fused wav -> ids pipeline for one 32-utterance batch and a
3-batch group (96 live rows) at the default live-row threshold (32 rows on the weight-streaming kernels, 96 on the wgmma
GEMM), at 1 (both on the wgmma GEMM) and at 128 (both weight-streaming).  Each must reproduce the reference's encoder
states (1e-3 rel-L2) and greedy tokens, with both encoder attention types (RoPEMHA, RelPosMHAXL)."""
import functools
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

GOLDENS = {"conformer_large_rope": "", "conformer_large_relpos": "-relpos"}  # golden -> test id suffix
TC_ROWS = {64: "default", 1: "tc_rows=1", 128: "tc_rows=128"}  # live-row threshold -> test id


@functools.lru_cache(maxsize=None)
def _engine(tag):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    g = torch.load(os.path.join(ROOT, "tests", "golden", tag + ".pt"))
    cfg = dict(CONFORMER_LARGE, attention_type=g["cfg"]["attention_type"])
    return g, AsrEngine(cfg, seeded_asr_state(cfg, 0), device="cuda:0")


@pytest.mark.parametrize("tag,tc_rows", [(t, r) for t in GOLDENS for r in TC_ROWS],
                         ids=[TC_ROWS[r] + s for s in GOLDENS.values() for r in TC_ROWS])
def test_kernel_variant_parity(tag, tc_rows):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    g, base = _engine(tag)
    eng = base.clone()  # a lane of its own: the threshold and the poll interval set here do not reach the other tests
    eng.set_decoder_tc_min_rows(tc_rows)
    wav = g["wav"].repeat(16, 1).cuda()
    lens = g["wav_lens"].repeat(16).cuda()
    S = g["greedy_logits"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(wav, lens, S, 1, 2, want_enc=True)
    outs = [torch.empty(32, S, dtype=torch.int32, device="cuda") for _ in range(3)]
    eng.transcribe_greedy_group_dev([wav] * 3, [lens] * 3, S, 1, 2, outs)
    eng.set_poll_interval(0)  # and the whole-pipeline graph
    outs2 = [torch.empty(32, S, dtype=torch.int32, device="cuda") for _ in range(3)]
    eng.transcribe_greedy_group_dev([wav] * 3, [lens] * 3, S, 1, 2, outs2)
    torch.cuda.synchronize()
    rel = float((enc[:2].cpu().double() - g["enc_out"].double()).norm() / g["enc_out"].double().norm())
    print(tag, tc_rows, rel)
    assert bool(torch.isfinite(enc).all()) and rel < 1e-3
    assert pred[:2].cpu().tolist() == g["hyps"] and outs[0][:2].cpu().tolist() == g["hyps"]
    assert all(torch.equal(pred[2 * i:2 * i + 2], pred[:2]) for i in range(16))
    assert all(torch.equal(o, outs[0]) for o in outs) and all(torch.equal(a, b) for a, b in zip(outs, outs2))
