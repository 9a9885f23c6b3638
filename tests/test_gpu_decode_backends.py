"""-m gpu tests of the KV-cached decoder and TransformerLM step loops (csrc/engine.cu) on each projection back end: weight
streaming with the pre-norms fused into the projections, weight streaming with separate LayerNorm kernels, and the wgmma
GEMM.  Every entry point that runs a step loop must enqueue the launches its layer structure implies, keep the step's
projections on the back end its row count selects, and give bit-identical results when run again."""
import ctypes
import os
import sys

import pytest
import torch

from speechbrain_b200 import _lib
from speechbrain_b200.engine import AsrEngine
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, CONFORMER_SMALL, seeded_asr_state, seeded_tensor
from speechbrain_b200.utils.shapes import transformer_lm_shapes

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401

pytestmark = pytest.mark.gpu
LM = dict(d_model=128, nhead=2, num_encoder_layers=2, d_ffn=256)
CFG = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=2, lm=LM)
BEAM = dict(beam_size=4, max_steps=12, min_steps=0, bos=1, eos=2, lm_weight=0.6, ctc_weight=0.4, blank_index=0)
LD, LL = CFG["num_decoder_layers"], LM["num_encoder_layers"]
BACKENDS = ("stream_fused", "stream_ln", "wgmma")

# Launches (sbk_launch_count) of one step.  A decoder layer: the self-attention in_proj, self-attention, out_proj, the
# cross-attention query projection, cross-attention, out_proj, ffn1 and ffn2, plus one LayerNorm kernel in front of each of
# the three pre-normed projections unless the LayerNorm is fused into it.  The head: the final LayerNorm (the same rule)
# and seq_lin.  An LM layer: in_proj, attention, out_proj, LayerNorm, ffn1, ffn2, LayerNorm; then encoder.norm, Linear,
# LayerNorm, Linear and the weighted log_softmax.
def dec_layers(n_layers, ln_kernels):
    return n_layers * (8 + 3 * ln_kernels)


def dec_head(ln_kernels):
    return 1 + ln_kernels


LM_STEP = LL * 7 + 5
# wgmma GEMM launches of one teacher-forced step on that back end (none on weight streaming): 6 per decoder layer (no
# head), 4 per LM layer and 2 for the LM's output projection
DEC_GEMMS, LM_GEMMS = LD * 6, LL * 4 + 2


@pytest.fixture(scope="module")
def eng(dev):
    sd = seeded_asr_state(CFG, 0)  # decoder, seq_lin and ctc_lin
    for k, shp in transformer_lm_shapes(CFG["vocab"], LM["d_model"], LM["nhead"], LM["num_encoder_layers"], LM["d_ffn"]).items():
        sd["lm." + k] = seeded_tensor(1, "lm." + k, shp)
    return AsrEngine(CFG, sd, device=dev, parts=("fbank", "cnn", "encoder", "decoder", "lm"))


def _configure(eng, backend):
    """The back end's settings; returns the LayerNorm kernels per pre-normed projection (0: fused into it)."""
    eng.set_decoder_ln_fusion(backend == "stream_fused")
    eng.set_decoder_tc_min_rows(1 if backend == "wgmma" else 64)  # 64: the default, above every row count used here
    return 0 if backend == "stream_fused" else 1


def _counted(fn):
    """(fn(), launches it enqueued)"""
    n0 = _lib.lib().sbk_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, _lib.lib().sbk_launch_count() - n0


def _gemms(fn):
    """wgmma GEMM launches of fn() (only for calls that replay no CUDA graph: a graph's launches are not timed)"""
    L = _lib.lib()
    L.sbk_gemm_profile_enable(1)
    try:
        fn()
        torch.cuda.synchronize()
        n = ctypes.c_int()
        _lib.check(L.sbk_gemm_profile_read(ctypes.byref(n), None, None), "sbk_gemm_profile_read")
    finally:
        L.sbk_gemm_profile_enable(0)
    return n.value


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    if isinstance(a, tuple):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def _inputs(dev):
    g = torch.Generator().manual_seed(3)
    enc = torch.randn(2, 100, CFG["d_model"], generator=g).to(dev)
    enc_lens = torch.tensor([1.0, 0.85], device=dev)
    tgt = torch.randint(3, CFG["vocab"], (2, 7), generator=g).to(dev)
    toks = torch.randint(3, CFG["vocab"], (3, 9), generator=g)
    toks[:, 0] = 1
    toks[1, 6:] = 0  # pad-filled tails, masked as keys
    toks[2, 4:] = 0
    lens = torch.tensor([9, 6, 4], dtype=torch.int32)
    return enc, enc_lens, tgt, toks.to(dev), lens.to(dev)


@pytest.mark.parametrize("backend", BACKENDS)
def test_step_loops(eng, dev, backend):
    ln = _configure(eng, backend)
    wg = backend == "wgmma"
    enc, enc_lens, tgt, toks, lens = _inputs(dev)
    S = tgt.shape[1]
    L = toks.shape[1]
    calls = {
        "greedy": lambda: eng.greedy_from_enc(enc, enc_lens, 12, 1, 2),
        "beam": lambda: eng.beam_from_enc(enc, enc_lens, **BEAM),
        "teacher": lambda: eng.decode_teacher_forced(tgt, enc),
        "rescore": lambda: eng.lm_rescore(toks, lens),
        "step_logits": lambda: eng.lm_step_logits(toks),
    }
    for name, fn in calls.items():
        first, n_first = _counted(fn)
        again, n_again = _counted(fn)
        assert _same(first, again), f"{backend} {name}: a rerun differs"
        if name == "greedy":
            steps = first[3]
            assert steps > 0
            # relative lengths -> frame counts, cross-attention K / V, greedy_reset; per step the layers, head and arg-max
            want = 4 + steps * (dec_layers(LD, ln) + dec_head(ln) + 1)
        elif name == "beam":
            steps = len(first[0])
            assert steps > 0
            # relative lengths, cross-attention K / V, ctc_lin, CTC reset (2), beam_reset; per step the CTC state update, the
            # LM step, the decoder layers and head, the CTC scores and the beam step
            want = 7 + steps * (1 + LM_STEP + dec_layers(LD, ln) + dec_head(ln) + 2)
        elif name == "teacher":
            # cross-attention K / V; per position the embedding, the layers without the head and decoder.norm
            want = 2 + S * (1 + dec_layers(LD, ln) + 1)
        elif name == "rescore":
            want = 1 + (L - 1) * (1 + LM_STEP + 1)  # reset; per position the embedding, the LM step and the score
        else:
            want = 1 + L * (1 + LM_STEP)
        assert n_first == n_again == want, f"{backend} {name}: {n_first} / {n_again} launches, formula {want}"
    # the back end the teacher-forced loops ran on: their step projections are wgmma GEMMs exactly when it is selected
    assert _gemms(calls["teacher"]) == 1 + wg * S * DEC_GEMMS  # 1: the cross-attention K / V of every layer
    assert _gemms(calls["rescore"]) == wg * (L - 1) * LM_GEMMS
    assert _gemms(calls["step_logits"]) == wg * L * LM_GEMMS


def test_width_fallback_stays_on_weight_streaming(dev):
    """A decoder width the wgmma QKV -> cache epilogue does not take (d_model % 32 != 0, Conformer-small's 144) runs its
    steps on weight streaming at any row count, with separate LayerNorm kernels (no fused projection for that width)."""
    cfg = dict(CONFORMER_SMALL, num_encoder_layers=1, num_decoder_layers=2)
    eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device=dev)
    assert cfg["d_model"] % 32 != 0
    rows, S = 96, 5
    g = torch.Generator().manual_seed(4)
    enc = torch.randn(rows, 40, cfg["d_model"], generator=g).to(dev)
    enc_lens = torch.ones(rows, device=dev)
    tgt = torch.randint(3, cfg["vocab"], (rows, S), generator=g).to(dev)
    ld = cfg["num_decoder_layers"]
    (pred, score, _, steps), n = _counted(lambda: eng.greedy_from_enc(enc, enc_lens, 6, 1, 2))
    # cross-attention K / V in one GEMM per layer (no head-major layout at head width 36)
    assert steps > 0 and n == 3 + ld + steps * (dec_layers(ld, 1) + dec_head(1) + 1)
    again = eng.greedy_from_enc(enc, enc_lens, 6, 1, 2)
    assert torch.equal(pred, again[0]) and torch.equal(score, again[1])
    out, n = _counted(lambda: eng.decode_teacher_forced(tgt, enc))
    assert n == 1 + ld + S * (1 + dec_layers(ld, 1) + 1)
    assert _gemms(lambda: eng.decode_teacher_forced(tgt, enc)) == ld  # only the cross-attention K / V
    assert torch.equal(out, eng.decode_teacher_forced(tgt, enc))
