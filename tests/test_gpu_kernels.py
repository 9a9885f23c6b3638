"""-m gpu parity tests: every CUDA path is called through the C ABI (libsbk.so) and compared with the
CPU oracle / the committed reference goldens on the same seeded inputs."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mirrors import build_mirror, seeded  # noqa: E402
from parity import check_greedy, dev, lm_scorer, rel  # noqa: E402,F401

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------- wgmma GEMM
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 512), (200, 256, 512), (251, 5000, 512),
                                   (1000, 1536, 640), (8032, 2048, 512), (8032, 512, 2048), (300, 144, 144),
                                   (8032, 1536, 512), (8032, 1024, 512), (37, 512, 640), (20000, 256, 64)])
@pytest.mark.parametrize("out_f32,act", [(1, 0), (0, 1)])
def test_gemm_tc(dev, M, N, K, out_f32, act):
    import ctypes

    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, generator=g).half()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    bias = torch.randn(N, generator=g)
    ref = A.float() @ W.float().T + bias
    if act == 1:
        ref = torch.nn.functional.silu(ref)
    Ad, Wd, bd = A.to(dev), W.to(dev), bias.to(dev)
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if out_f32 else torch.float16)
    check(lib().sbk_gemm_f16_test(ptr(Ad), ptr(Wd), ptr(bd), ptr(out), out_f32, act, M, N, K, stream_ptr(dev)), "gemm")
    torch.cuda.synchronize()
    got = out.float().cpu()
    err = (got - ref).abs().max().item()
    tol = 2e-3 if out_f32 else 2e-2
    print(f"gemm M={M} N={N} K={K} f32={out_f32} act={act}: max abs err {err:.3e}")
    assert err < tol, f"max abs err {err}"


@pytest.mark.parametrize("M,N,K,alpha", [(8032, 512, 512, 1.0), (8032, 512, 2048, 0.5), (300, 512, 512, 1.0), (1000, 256, 64, 0.5)])
def test_gemm_residual_epilogue(dev, M, N, K, alpha):
    """x += alpha * (A W^T + b) in place (fp32 residual stream): the epilogue of FFN2 / out-proj / conv pw2."""
    import ctypes

    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    g = torch.Generator().manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).half()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    bias = torch.randn(N, generator=g)
    x = torch.randn(M, N, generator=g)
    ref = x + alpha * (A.float() @ W.float().T + bias)
    Ad, Wd, bd, xd = A.to(dev), W.to(dev), bias.to(dev), x.to(dev)
    check(lib().sbk_gemm_f16_resid_test(ptr(Ad), ptr(Wd), ptr(bd), ptr(xd), ctypes.c_float(alpha), M, N, K, stream_ptr(dev)),
          "gemm resid")
    torch.cuda.synchronize()
    err = (xd.cpu() - ref).abs().max().item()
    print(f"gemm resid M={M} N={N} K={K} alpha={alpha}: max abs err {err:.3e}")
    assert err < 2e-3


# ----------------------------------------------------------------------------------------- Fbank
def _assert_fbank_close(out, ref, name=""):
    """north_star: 'Fbank within 1e-4 rel FP32'.  Outputs are dB values that cross 0, where a pure relative error
    is singular (two correct fp32 FFTs differ by ~4e-6 dB, i.e. 'rel' 4e-4 at |x| = 0.01 dB), so the bound is the
    usual mixed form |a-b| <= 1e-4 * max(|b|, 1 dB); the plain max-abs error is printed beside it."""
    bad = ((out - ref).abs() > 1e-4 * ref.abs().clamp_min(1.0))
    assert not bad.any(), f"{name}: {int(bad.sum())} elements outside 1e-4*max(|ref|,1)"


def test_fbank_golden(dev):
    """Fbank vs the reference's outputs (BASELINE config 1 + ragged / n_fft=512 / n_mels=40 cases).
    Tolerance from north_star: 1e-4 relative fp32, |a-b| / max(|b|, 1e-3)."""
    from speechbrain_b200.lobes.features import Fbank
    gold = torch.load(os.path.join(GOLDEN, "fbank.pt"))
    for name, case in gold.items():
        fb = Fbank(**case["kwargs"]).to(dev)
        out = fb(case["wav"].to(dev)).cpu()
        ref = case["out"]
        assert out.shape == ref.shape, name
        relm = (out - ref).abs() / ref.abs().clamp_min(1e-3)
        i = int(relm.argmax())
        print(f"fbank[{name}] shape {tuple(ref.shape)} max rel err {relm.max():.3e} at ref={ref.flatten()[i]:.5f} "
              f"(abs err {(out - ref).abs().flatten()[i]:.2e}); max abs err {(out - ref).abs().max():.2e} dB")
        _assert_fbank_close(out, ref, name)


def test_fbank_large_matches_oracle(dev):
    from oracle import asr_oracle as O
    from speechbrain_b200.lobes.features import Fbank
    g = torch.Generator().manual_seed(5)
    wav = torch.randn(4, 160000, generator=g)
    wav[1, 100000:] = 0
    ref = O.fbank(wav, n_fft=512, n_mels=80, win_length_ms=32)
    out = Fbank(n_fft=512, n_mels=80, win_length=32).to(dev)(wav.to(dev)).cpu()
    print("fbank 4x10s max abs err (dB)", (out - ref).abs().max().item())
    _assert_fbank_close(out, ref, "4x10s")
    # L % 4 != 0 exercises the non-TMA staging path
    wav2 = wav[:, :159999].contiguous()
    out2 = Fbank(n_fft=512, n_mels=80, win_length=32).to(dev)(wav2.to(dev)).cpu()
    ref2 = O.fbank(wav2, n_fft=512, n_mels=80, win_length_ms=32)
    _assert_fbank_close(out2, ref2, "L%4!=0")


def test_input_norm_golden(dev):
    from speechbrain_b200.processing.features import InputNormalization
    gold = torch.load(os.path.join(GOLDEN, "input_norm.pt"))
    x, lens = gold["x"].to(dev), gold["lens"].to(dev)
    n = InputNormalization(norm_type="global")
    n.glob_mean, n.glob_std, n.count = gold["glob_mean"], gold["glob_std"], 1
    n.eval()
    assert (n(x, lens).cpu() - gold["global"]).abs().max() < 1e-5
    n = InputNormalization(norm_type="sentence").eval()
    assert (n(x, lens).cpu() - gold["sentence"]).abs().max() < 1e-4
    n = InputNormalization(norm_type="sentence", avoid_padding_norm=True).eval()
    assert (n(x, lens).cpu() - gold["sentence_avoid_pad"]).abs().max() < 1e-4
    kat = InputNormalization(norm_type="sentence").eval()(torch.tensor([[[1.0], [3.0], [0.0], [0.0], [0.0]]], device=dev),
                                                          torch.tensor([0.4], device=dev))
    assert torch.allclose(kat.cpu(), gold["kat"], atol=1e-5)  # tests/unittests/test_features.py:112-118


# ----------------------------------------------------------------------------------------- model stages
def _engine(cfg, dev, parts=("fbank", "cnn", "encoder", "decoder")):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    sd = seeded_asr_state(cfg, 0)
    return AsrEngine(cfg, sd, device=dev, parts=parts), sd


def _cfg_from_gold(g):
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, CONFORMER_SMALL
    base = CONFORMER_LARGE if g["cfg"]["name"] == "conformer_large" else CONFORMER_SMALL
    return dict(base, attention_type=g["cfg"]["attention_type"])


def test_conformer_small_encoder_golden(dev):
    """BASELINE config 2 family: Conformer-small (12L / 144d / 4 heads of 36 / RelPosMHAXL / n_fft 400) CNN + encoder
    vs the reference goldens (head_dim 36 is zero-padded to 48 in the attention kernel; K = 144 GEMMs)."""
    g = torch.load(os.path.join(GOLDEN, "conformer_small_relpos.pt"))
    cfg = _cfg_from_gold(g)
    eng, sd = _engine(cfg, dev, parts=("cnn", "encoder"))
    cnn_shape = (g["cnn_out"].shape[0], g["cnn_out"].shape[1], -1)
    enc = eng.encode_from_cnn(g["cnn_out"].reshape(cnn_shape).to(dev), g["wav_lens"].to(dev)).cpu()
    r = rel(enc, g["enc_out"])
    print(f"[conformer_small_relpos] encoder rel-L2 err {r:.3e} max abs {(enc - g['enc_out']).abs().max():.3e}")
    assert r < 1e-3


@pytest.mark.parametrize("tag", ["conformer_large_rope", "conformer_large_relpos"])
def test_model_stages_golden(dev, tag):
    """CNN front-end, Conformer encoder and KV-cached greedy search vs the REFERENCE outputs in tests/golden
    (B=2 x 2 s, ragged lengths).  Tolerances: CNN 2e-3 abs (fp16 conv2 operands), encoder <= 1e-3 rel-L2
    (north_star 'within 1e-3 rel'), greedy tokens identical unless the reference top-2 margin is below 5e-3."""
    from oracle import asr_oracle as O
    g = torch.load(os.path.join(GOLDEN, tag + ".pt"))
    cfg = _cfg_from_gold(g)
    eng, sd = _engine(cfg, dev)
    chk = float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))
    assert abs(chk - g["weight_checksum"]) / g["weight_checksum"] < 1e-9, "seeded weights differ from golden run"
    feats = O.input_norm(g["fbank"], g["wav_lens"], "global", sd["normalize.glob_mean"], sd["normalize.glob_std"])
    cnn = eng.cnn(feats.to(dev)).cpu()
    ref_cnn = g["cnn_out"].reshape(cnn.shape)
    e = (cnn - ref_cnn).abs().max().item()
    print(f"[{tag}] cnn max abs err {e:.3e} (ref absmax {ref_cnn.abs().max():.2f})")
    assert e < 5e-3
    enc = eng.encode_from_cnn(g["cnn_out"].reshape(cnn.shape).to(dev), g["wav_lens"].to(dev)).cpu()
    r = rel(enc, g["enc_out"])
    print(f"[{tag}] encoder rel-L2 err {r:.3e} max abs {(enc - g['enc_out']).abs().max():.3e}")
    assert r < 1e-3
    n_steps = g["greedy_logits"].shape[1]
    ref_lp = torch.log_softmax(g["greedy_logits"], -1)
    top2 = g["greedy_logits"].topk(2, -1).values
    margin = top2[..., 0] - top2[..., 1]
    ref_tok = g["greedy_logits"].argmax(-1)
    # both decode-step implementations: weight-streaming projections (default below 64 rows) and wgmma GEMM projections
    for tc_rows, name in ((1 << 30, "skinny"), (1, "wgmma")):
        eng.set_decoder_tc_min_rows(tc_rows)
        pred, score, lp, done = eng.greedy_from_enc(g["enc_out"].to(dev), g["wav_lens"].to(dev), n_steps, 1, 2, want_log_probs=True)
        print(f"[{tag}] greedy[{name}] tokens {pred.tolist()} ref {g['hyps']}")
        check_greedy(f"{tag}/{name}", pred.cpu(), lp.cpu(), ref_tok, margin, ref_lp)


@pytest.mark.parametrize("n_mels", [90, 96, 4])
def test_cnn_frontend_two_kernel_golden(dev, n_mels):
    """ConvolutionFrontEnd at feature widths the fused front-end kernel does not take (n_mels 81-96: F1 > 40; n_mels <= 4:
    F1 < 3), which run conv1_ln_kernel + conv2_ln_kernel, vs the CPU oracle.  Same bar as the CNN check of
    test_model_stages_golden."""
    from oracle import asr_oracle as O
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    cnn = ConvolutionFrontEnd(input_shape=(8, 10, n_mels), num_blocks=2, num_layers_per_block=1, out_channels=(64, 32),
                              kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
    sd = seeded_state_dict(cnn, 0)
    cnn.load_state_dict(sd)
    x = torch.randn(2, 151, n_mels, generator=torch.Generator().manual_seed(n_mels))
    out = cnn(x.to(dev)).cpu()
    ref = O.cnn_frontend(x, sd)
    assert out.shape == ref.shape, (out.shape, ref.shape)
    e = (out - ref).abs().max().item()
    print(f"[n_mels={n_mels}] cnn max abs err {e:.3e} (ref absmax {ref.abs().max():.2f})")
    assert e < 5e-3


def test_transcribe_end_to_end(dev):
    """wav -> tokens through the fused device pipeline and through the host-buffer entry point."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    cfg = _cfg_from_gold(g)
    eng, sd = _engine(cfg, dev)
    n_steps = g["greedy_logits"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(g["wav"].to(dev), g["wav_lens"].to(dev), n_steps, 1, 2, want_enc=True)
    r = rel(enc.cpu(), g["enc_out"])
    print("e2e encoder rel-L2", r, "tokens", pred.cpu().tolist(), "ref", g["hyps"])
    assert r < 1.5e-3
    pred_h, done_h = eng.transcribe_greedy_host(g["wav"].pin_memory(), g["wav_lens"], n_steps, 1, 2)
    assert torch.equal(pred_h, pred.cpu())


def _conformer_large():
    """the mirror of the seeded Conformer-L the beam fixtures were written from"""
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE
    return build_mirror(CONFORMER_LARGE, seeded(CONFORMER_LARGE))


@pytest.mark.parametrize("case", ["thr_on", "recipe", "no_eos"])
def test_beam_search_golden(dev, case):
    """S2STransformerBeamSearcher (no scorer) vs the REFERENCE's hypotheses / scores / log-probs on the golden encoder
    states: EOS threshold on, the recipe's settings (temperature 1.15, min steps, no threshold), and the path where no
    hypothesis ever ends (final fill).  Scores within 2e-2 (fp16 decoder), hypotheses identical."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_conformer_large_rope.pt"))[case]
    bs = _conformer_large().searcher(gb["kwargs"], gb["max_decode_ratio"], gb["eos_bias"])
    for name, tc_rows in (("skinny", None), ("wgmma", 1)):  # both decode-step projection implementations
        if tc_rows is not None:
            bs._get_engine(dev).set_decoder_tc_min_rows(tc_rows)
        hyps, lens, scores, lp = bs(g["enc_out"].to(dev), g["wav_lens"].to(dev))
        print(f"beam[{case}/{name}] hyps {hyps} ref {gb['hyps']} scores {scores.tolist()} ref {gb['scores'].tolist()}")
        assert hyps == gb["hyps"]
        assert (scores.cpu() - gb["scores"]).abs().max() < 2e-2
        assert torch.allclose(lens.cpu(), gb["lens"])
        assert (lp.cpu() - gb["log_probs"]).abs().max() < 3e-2


# ----------------------------------------------------------------------------------------- full-size properties
def test_full_size_properties(dev):
    """BASELINE full size (32 x 10 s, Conformer-L) is too slow for the CPU oracle, so parity is checked through
    size-independent properties:
      * Fbank: scaling the waveform by 10 adds exactly 20 dB everywhere (the top_db clip is relative to the maximum);
      * batch invariance: utterance i of the 32-batch gets the same encoder states / tokens as when transcribed alone;
      * determinism: two runs give identical token ids;
      * decode coalescing: transcribing two batches as one group gives the same ids as two separate calls;
      * ragged lengths: rows with wav_len < 1 only differ from the full-length run where the reference's masks act."""
    from speechbrain_b200.lobes.features import Fbank
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE
    g = torch.Generator().manual_seed(99)
    B, L, steps = 32, 160000, 12
    wav = torch.randn(B, L, generator=g).to(dev)
    fb = Fbank(n_fft=512, n_mels=80, win_length=32)
    f1, f10 = fb(wav), fb(wav * 10.0)
    assert f1.shape == (B, 1001, 80)
    assert (f10 - f1 - 20.0).abs().max().item() < 2e-3
    eng, _ = _engine(dict(CONFORMER_LARGE), dev)
    ones = torch.ones(B, device=dev)
    pred, _, enc, _ = eng.transcribe_greedy_dev(wav, ones, steps, 1, 2, want_enc=True)
    pred2, _, _, _ = eng.transcribe_greedy_dev(wav, ones, steps, 1, 2)
    assert torch.equal(pred, pred2), "non-deterministic decode"
    assert torch.isfinite(enc).all()
    for i in (0, 17, 31):
        p1, _, e1, _ = eng.transcribe_greedy_dev(wav[i:i + 1].contiguous(), ones[:1], steps, 1, 2, want_enc=True)
        assert rel(e1[0].cpu(), enc[i].cpu()) < 1e-5, f"encoder states of utterance {i} depend on the batch"
        assert torch.equal(p1[0], pred[i]), f"tokens of utterance {i} depend on the batch"
    # decode coalescing == separate calls
    wav_b = torch.randn(B, L, generator=g).to(dev)
    pb, _, _, _ = eng.transcribe_greedy_dev(wav_b, ones, steps, 1, 2)
    outs = [torch.empty(B, steps, dtype=torch.int32, device=dev) for _ in range(2)]
    eng.set_decoder_tc_min_rows(1 << 30)  # same projection kernels as the separate calls: bit-identical ids
    eng.transcribe_greedy_group_dev([wav, wav_b], [ones, ones.clone()], steps, 1, 2, outs)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], pred) and torch.equal(outs[1], pb)
    # default: 64 live rows switch the projections to the wgmma GEMM (other summation order): ids may only differ after
    # a near-tie, so almost every utterance must still agree
    eng.set_decoder_tc_min_rows(64)
    eng.transcribe_greedy_group_dev([wav, wav_b], [ones, ones.clone()], steps, 1, 2, outs)
    torch.cuda.synchronize()
    same = sum(int(torch.equal(outs[0][i], pred[i])) + int(torch.equal(outs[1][i], pb[i])) for i in range(B))
    print(f"coalesced decode (wgmma GEMM projections) vs separate (weight-streaming): {same}/{2 * B} utterances identical")
    assert same >= int(0.9 * 2 * B)
    eng.set_decoder_tc_min_rows(1 << 30)
    # ragged: shortening utterance 5 must not change any other utterance
    lens = ones.clone()
    lens[5] = 0.6
    pr, _, er, _ = eng.transcribe_greedy_dev(wav, lens, steps, 1, 2, want_enc=True)
    keep = [i for i in range(B) if i != 5]
    assert torch.equal(pr[keep], pred[keep]) and torch.equal(er[keep], enc[keep])
    assert not torch.equal(er[5], enc[5])


@pytest.mark.parametrize("case", ["lm_recipe", "lm_eos"])
def test_beam_search_with_transformerlm_scorer_golden(dev, case):
    """S2STransformerBeamSearcher + ScorerBuilder(full_scorers=[TransformerLMScorer], weight 0.6, temperature 1.15) with the
    recipe's 12 x 768 TransformerLM vs the REFERENCE (shallow fusion, scorer.py:510-543,1221-1268)."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_lm_conformer_large_rope.pt"))[case]
    bs = _conformer_large().searcher(gb["kwargs"], gb["max_decode_ratio"], gb["eos_bias"],
                                     scorers={"transformerlm": gb["lm_weight"]}, lm_temperature=gb["lm_temperature"])
    hyps, lens, scores, lp = bs(g["enc_out"].to(dev), g["wav_lens"].to(dev))
    print(f"beam+lm[{case}] hyps {hyps} ref {gb['hyps']} scores {scores.tolist()} ref {gb['scores'].tolist()}")
    assert hyps == gb["hyps"]
    assert (scores.cpu() - gb["scores"]).abs().max() < 3e-2
    assert (lp.cpu() - gb["log_probs"]).abs().max() < 3e-2


@pytest.mark.parametrize("case", ["ctc_lm_test", "ctc_valid", "ctc_eos"])
def test_beam_search_with_ctc_scorer_golden(dev, case):
    """Joint CTC/attention decoding: S2STransformerBeamSearcher + ScorerBuilder(full_scorers=[TransformerLMScorer, CTCScorer]
    (test search) or [CTCScorer] (valid search), ctc 0.4 / lm 0.6) vs the REFERENCE: hypotheses identical, scores within
    5e-2 (fp16 GEMM operands in the decoder, LM and CTC head; the prefix scores sum ~T log-posteriors)."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_ctc_conformer_large_rope.pt"))[case]
    scorers = dict(transformerlm=gb["lm_weight"], ctc=gb["ctc_weight"]) if gb["with_lm"] else dict(ctc=gb["ctc_weight"])
    bs = _conformer_large().searcher(gb["kwargs"], gb["max_decode_ratio"], gb["eos_bias"], scorers=scorers,
                                     lm_temperature=gb["lm_temperature"])
    hyps, lens, scores, lp = bs(g["enc_out"].to(dev), g["wav_lens"].to(dev))
    print(f"beam+ctc[{case}] hyps {hyps} ref {gb['hyps']} scores {scores.tolist()} ref {gb['scores'].tolist()}")
    assert hyps == gb["hyps"]
    assert (scores.cpu() - gb["scores"]).abs().max() < 5e-2
    assert (lp.cpu() - gb["log_probs"]).abs().max() < 5e-2


def test_beam_search_return_topk_golden(dev):
    """return_topk=True, topk=3: padded n-best hypotheses, lengths, scores and log-probs vs the REFERENCE."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_topk_conformer_large_rope.pt"))
    bs = _conformer_large().searcher(gb["kwargs"], gb["max_decode_ratio"], gb["eos_bias"], topk=gb["topk"])
    hyps, lens, scores, lp = bs(g["enc_out"].to(dev), g["wav_lens"].to(dev))
    print(f"beam topk hyps {hyps.tolist()} ref {gb['hyps'].tolist()} scores {scores.tolist()} ref {gb['scores'].tolist()}")
    assert torch.equal(hyps.cpu(), gb["hyps"]) and torch.allclose(lens.cpu(), gb["lens"])
    assert (scores.cpu() - gb["scores"]).abs().max() < 2e-2 and (lp.cpu() - gb["log_probs"]).abs().max() < 3e-2


def test_lm_rescorer_golden(dev):
    """TransformerLMRescorer + RescorerBuilder mirrors (teacher-forced KV-cached LM on the device) vs the REFERENCE's n-best
    rescoring: LM scores within 5e-2 of sums of up to 24 log-probs (|score| ~ 35..200), identical re-ranking."""
    from oracle.asr_oracle import StubTokenizer
    from speechbrain_b200.decoders.scorer import RescorerBuilder, TransformerLMRescorer
    gb = torch.load(os.path.join(GOLDEN, "lm_rescore.pt"))
    lm = lm_scorer()
    resc = TransformerLMRescorer(language_model=lm, tokenizer=StubTokenizer(), device=dev, temperature=gb["temperature"],
                                 bos_index=1, eos_index=2, pad_index=0)
    scores = resc.rescore_hyps(gb["hyps"]).cpu()
    print("lm rescore", scores.tolist(), "ref", gb["lm_scores"].tolist())
    assert (scores - gb["lm_scores"]).abs().max() < 5e-2
    import copy
    rb = RescorerBuilder(weights={"transformerlm": gb["weight"]}, rescorers=[resc])
    out_c, out_s = rb.rescore(gb["hyps"], copy.deepcopy(gb["scores"]))
    assert out_c == gb["out_candidates"]
    assert max(abs(a - b) for ra, rb_ in zip(out_s, gb["out_scores"]) for a, b in zip(ra, rb_)) < 5e-2


def test_beam_search_with_length_scorer_golden(dev):
    """ScorerBuilder(full_scorers=[LengthScorer], weights={"length": w}) with length_normalization=False vs the REFERENCE."""
    from speechbrain_b200.decoders.scorer import LengthScorer, ScorerBuilder
    from speechbrain_b200.decoders.seq2seq import S2STransformerBeamSearcher
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_len_conformer_large_rope.pt"))
    m = _conformer_large()
    scorer = ScorerBuilder(full_scorers=[LengthScorer(5000)], weights={"length": gb["length_weight"]})
    with pytest.raises(ValueError):  # "Length normalization is not compatible with length rewarding."
        S2STransformerBeamSearcher(modules=[m.tr, m.seq_lin], bos_index=1, eos_index=2, beam_size=4, scorer=scorer)
    bs = m.searcher(gb["kwargs"], gb["max_decode_ratio"], gb["eos_bias"], scorers={"length": gb["length_weight"]})
    hyps, lens, scores, lp = bs(g["enc_out"].to(dev), g["wav_lens"].to(dev))
    print(f"beam+length hyps {hyps} ref {gb['hyps']} scores {scores.tolist()} ref {gb['scores'].tolist()}")
    assert hyps == gb["hyps"]
    assert (scores.cpu() - gb["scores"]).abs().max() < 2e-2 and (lp.cpu() - gb["log_probs"]).abs().max() < 3e-2
