"""-m gpu tests of the Branchformer encoder (TransformerASR(encoder_module="branchformer")): the CSGU kernel (sbk_csgu_test)
against fp32 torch, and the whole device pipeline against the reference outputs in tests/golden/branchformer.pt
(generator: tools/make_branchformer_golden.py).  The fixture keeps the reference's encoder states as per-frame norms and
sampled rows; the whole states are recomputed with the fp32 CPU oracle (tests/branchformer_oracle.py), which is first
checked against those (1e-5) and equals the reference to 1e-7 (test_branchformer_golden.py).

Encoder bar: rel-L2 <= 1.5e-3 over all frames and over each utterance's valid frames.  The CPU oracle with every GEMM
operand rounded to fp16 already sits at 1.0e-3 on this input (test_branchformer_golden.py::test_fp16_operand_error_estimate):
18 layers without a LayerNorm on the residual stream let the operand rounding accumulate (5e-4 after layer 1, 1.0e-3 after
layer 18), so the Conformer's 1e-3 bar is below what fp16 operands allow here.  Greedy: tokens identical up to the first
decision whose reference top-1/top-2 margin is below 5e-3, chosen log-probs within 2e-2 (parity.check_greedy)."""
import functools
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import (case_wav, check_alone_vs_batch, check_ctc_argmax, check_encoder, check_greedy, check_summary,  # noqa: E402,F401
                    dev, seeded_wav)
import branchformer_oracle as BO  # noqa: E402
from mirrors import build_mirror  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ENC_BAR = 1.5e-3

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "branchformer.pt"))


# ------------------------------------------------------------------------------------------------ CSGU kernel
def _csgu_ref(u, g, bta, taps, bias):
    """ConvolutionalSpatialGatingUnit.forward in fp32 on the fp16 input: LN(b) -> reflect pad -> depthwise conv -> a * (.)"""
    a, b = u.float().chunk(2, dim=-1)
    b = F.layer_norm(b, (b.shape[-1],), g, bta, 1e-5)
    K = taps.shape[-1]
    h = F.pad(b.transpose(1, 2), ((K - 1) // 2, (K - 1) // 2), mode="reflect")
    return F.conv1d(h, taps, bias, groups=taps.shape[0]).transpose(1, 2) * a


def _csgu_dev(u, g, bta, taps, bias):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    B, T, C = u.shape
    out = torch.empty(B, T, C // 2, device=u.device, dtype=torch.float16)
    check(lib().sbk_csgu_test(ptr(u), B, T, C, ptr(g), ptr(bta), ptr(taps), ptr(bias), taps.shape[-1], ptr(out),
                              stream_ptr(u.device)), "sbk_csgu_test")
    return out


@pytest.mark.parametrize("K", [31, 15])
@pytest.mark.parametrize("C2", [1200, 1536])
@pytest.mark.parametrize("T", [16, 17, 30, 31, 32, 251, 1000])
def test_csgu_kernel_vs_torch(dev, T, C2, K):
    gen = torch.Generator().manual_seed(T * 7919 + C2 + K)
    B = 3
    u = torch.randn(B, T, 2 * C2, generator=gen)
    for b, frac in enumerate((1.0, 0.7, 0.4)):  # ragged batch: the padded frames hold other values, never masked
        n = max(1, int(frac * T))
        u[b, n:] = 0.25 * torch.randn(T - n, 2 * C2, generator=gen) - 0.1
    g = 1.0 + 0.1 * torch.randn(C2, generator=gen)
    bta = 0.05 * torch.randn(C2, generator=gen)
    taps = torch.randn(C2, 1, K, generator=gen) * (1.4 / K ** 0.5)
    bias = 1.0 + 0.05 * torch.randn(C2, generator=gen)
    cases = {"plain": u}
    if T in (16, 251):
        big = u.clone()
        big[..., C2:] += 60.0 + 20.0 * torch.rand(B, T, 1, generator=gen)  # large row means of the normalised half
        cases["large_mean"] = big
    for name, x in cases.items():
        x16 = x.half().to(dev)
        args = [t.to(dev).contiguous() for t in (g, bta, taps, bias)]
        out = _csgu_dev(x16, *args).float()
        ref = _csgu_ref(x16, *args)
        err = float(((out - ref).abs() / (ref.abs() + ref.pow(2).mean().sqrt())).max())
        print(f"csgu T={T} C/2={C2} K={K} {name}: max |d| / (|ref| + rms) = {err:.2e}")
        assert torch.isfinite(out).all() and err <= 2e-3
        assert torch.equal(out, _csgu_dev(x16, *args).float())


def test_csgu_kernel_rejects_short_and_bad_shapes(dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    C2 = 64
    u = torch.zeros(1, 15, 2 * C2, device=dev, dtype=torch.float16)
    out = torch.empty(1, 15, C2, device=dev, dtype=torch.float16)
    v = torch.ones(C2, device=dev)
    taps = torch.ones(C2, 1, 31, device=dev)
    st = stream_ptr(dev)
    assert lib().sbk_csgu_test(ptr(u), 1, 15, 2 * C2, ptr(v), ptr(v), ptr(taps), ptr(v), 31, ptr(out), st) != 0  # T <= 15
    assert lib().sbk_csgu_test(ptr(u), 1, 15, 2 * C2, ptr(v), ptr(v), ptr(taps), ptr(v), 30, ptr(out), st) != 0  # even K
    assert lib().sbk_csgu_test(ptr(u), 1, 15, 2 * C2, ptr(v), ptr(v), ptr(taps), ptr(v), 15, ptr(out), st) == 0  # T = 15, K = 15


# ------------------------------------------------------------------------------------------------ whole encoder
def _engine(cfg, fx, dev, parts=("fbank", "cnn", "encoder", "decoder")):
    from speechbrain_b200.engine import AsrEngine
    return AsrEngine(cfg, BO.state(cfg, fx), device=dev, parts=parts)


def _oracle_states(cfg, fx, case):
    """The reference's encoder states of a fixture case, recomputed by the CPU oracle and checked against the stored
    per-frame norms and sampled rows."""
    with torch.no_grad():
        ref = BO.wav_to_states(*case_wav(case), BO.state(cfg, fx), cfg)
    check_summary(f"{cfg['name']} oracle", ref, case["frame_norm"], case["sample_idx"], case["sample_rows"], 1e-5)
    return ref


def test_branchformer_large_encoder_and_greedy(dev, fx):
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_LARGE
    g = fx["large"]
    eng = _engine(BRANCHFORMER_LARGE, fx, dev)
    wav, lens = case_wav(g)
    S = g["greedy_tokens"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), lens.to(dev), S, 1, 2, want_enc=True)
    torch.cuda.synchronize()
    assert done == S
    check_encoder("branchformer_large 4x10s", enc.cpu(), _oracle_states(BRANCHFORMER_LARGE, fx, g), g["abs_len"], ENC_BAR)
    check_greedy("branchformer_large", pred.cpu(), score.cpu(), g["greedy_tokens"], g["greedy_margin"], g["greedy_chosen_lp"])
    check_alone_vs_batch(lambda w, ln: eng.encode_wav(w.to(dev), ln.to(dev)), wav, lens, 1e-5)


def test_branchformer_shortest_input(dev, fx):
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_LARGE
    s = fx["short"]
    eng = _engine(BRANCHFORMER_LARGE, fx, dev, parts=("fbank", "cnn", "encoder"))
    wav, lens = case_wav(s)
    enc = eng.encode_wav(wav.to(dev), lens.to(dev)).cpu()
    assert enc.shape == (1, 16, 512)
    check_encoder("branchformer_large T=16", enc, s["enc_out"], torch.tensor([16]), ENC_BAR)
    wav15, lens15 = seeded_wav(s["short_wav_seed"], s["short_wav_shape"])
    with pytest.raises(RuntimeError, match="reflect"):
        eng.encode_wav(wav15.to(dev), lens15.to(dev))


def test_branchformer_ctc_encoder_asr(dev, fx):
    from speechbrain_b200.decoders.ctc import ctc_greedy_decode
    from speechbrain_b200.inference.ASR import EncoderASR
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC as cfg
    c = fx["ctc"]
    m = build_mirror(cfg, BO.state(cfg, fx))
    enc = m.front_end(m.ctc_lin)
    asr = EncoderASR(modules=dict(encoder=enc), hparams=dict(tokenizer=None, decoding_function=functools.partial(ctc_greedy_decode, blank_id=0)),
                     run_opts={"device": str(dev)})
    wav, lens = case_wav(c)
    lp = asr.encode_batch(wav, lens).cpu()
    assert lp.shape == c["log_probs"].shape
    check_ctc_argmax("branchformer_ctc", lp, c["log_probs"], c["argmax"], c["margin"], lens, 0, c["hyps"])
    _, toks = asr.transcribe_batch(wav, lens)
    assert toks == c["hyps"]
    states = _engine(cfg, fx, dev, parts=("fbank", "cnn", "encoder")).encode_wav(wav.to(dev), lens.to(dev)).cpu()
    check_encoder("branchformer_ctc 3x8s", states, _oracle_states(cfg, fx, c), torch.round(lens * lp.shape[1]).int(), ENC_BAR)
