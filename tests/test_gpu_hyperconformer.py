"""-m gpu tests of the HyperConformer encoder (TransformerASR(attention_type="hypermixing")): the HyperMixing kernels
(sbk_hypermix_test) against fp32 torch, and the whole device pipeline against the reference outputs in
tests/golden/hyperconformer.pt (generator: tools/make_hyperconformer_golden.py).  The fixture keeps the reference's encoder
states as per-frame norms and sampled rows; the whole states are recomputed with the fp32 CPU oracle
(tests/hyperconformer_oracle.py), which is first checked against those and equals the reference to 1e-6
(test_hyperconformer_golden.py).

Encoder bar: rel-L2 <= 7.5e-3 over all frames and over each utterance's valid frames.  The CPU oracle with every product's
operands rounded to fp16 already sits at 3.2e-3 (all frames) and 4.9e-3 (worst utterance) on this input
(test_hyperconformer_golden.py::test_fp16_operand_error_estimate).  Greedy: tokens identical up to the first decision whose
reference top-1/top-2 margin is below 5e-3, chosen log-probs within 2e-2 (parity.check_greedy).  Beam 10
with [TransformerLM 0.6, CTC 0.4]: parity.check_beam."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import (best_tokens, case_wav, check_alone_vs_batch, check_beam, check_encoder, check_greedy,  # noqa: E402,F401
                    check_summary, dev, oracle_lm, rel)
import hyperconformer_oracle as HO  # noqa: E402
from mirrors import load, seeded  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ENC_BAR = 7.5e-3
KERNEL_BAR = 4e-3  # rel-L2 of the HyperMixing block's LayerNorm output against fp32 torch on the same fp16 input

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "hyperconformer.pt"))


def _state(fx, gain=None, cfg=None):
    """the fixture's weights of HYPERCONFORMER_22M (or of cfg: a reduced model's are the full one's first layers)"""
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M, scale_hypernet
    return seeded(cfg or HYPERCONFORMER_22M, fx["weight_seed"],
                  lambda sd: scale_hypernet(sd, fx["hypernet_gain"] if gain is None else gain))


# ------------------------------------------------------------------------------------------------ HyperMixing kernels
def _hm_weights(d, nhead, k, gen, w1_bias_shift=0.0):
    e = d // nhead
    w = {}
    for g in ("w1_gen", "w2_gen"):
        w[f"hyper.{g}.fc1_weights"] = torch.randn(nhead, e, e, generator=gen) * (2.0 / (2 * e)) ** 0.5
        w[f"hyper.{g}.fc1_biases"] = 0.1 * torch.randn(nhead, e, generator=gen)
        w[f"hyper.{g}.fc2_weights"] = torch.randn(nhead, k, e, generator=gen) * (2.0 / (e + k)) ** 0.5
        w[f"hyper.{g}.fc2_biases"] = 0.1 * torch.randn(nhead, k, generator=gen)
    w["hyper.w1_gen.fc2_biases"] += w1_bias_shift
    w["layer_norm.weight"] = 1.0 + 0.1 * torch.randn(d, generator=gen)
    w["layer_norm.bias"] = 0.1 * torch.randn(d, generator=gen)
    return w


def _hm_dev(x16, lens, w, nhead, k):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    B, T, d = x16.shape
    dw = {n: t.to(x16.device).contiguous() for n, t in w.items()}
    out = torch.empty(B, T, d, device=x16.device, dtype=torch.float32)
    names = [f"hyper.{g}.{n}" for g in ("w1_gen", "w2_gen") for n in ("fc1_weights", "fc1_biases", "fc2_weights", "fc2_biases")]
    check(lib().sbk_hypermix_test(ptr(x16), ptr(lens) if lens is not None else None, B, T, d, nhead, k,
                                  *[ptr(dw[n]) for n in names], ptr(dw["layer_norm.weight"]), ptr(dw["layer_norm.bias"]),
                                  ptr(out), stream_ptr(x16.device)), "sbk_hypermix_test")
    return out


@pytest.mark.parametrize("d,nhead,k", [(256, 8, 128), (512, 8, 256), (128, 2, 48)])
@pytest.mark.parametrize("T", [1, 15, 16, 17, 63, 64, 65, 251, 1000, 3000])
def test_hypermix_kernel_vs_torch(dev, T, d, nhead, k):
    if T == 3000 and d == 128:
        pytest.skip("T = 3000 runs at the two recipe widths")
    gen = torch.Generator().manual_seed(T * 131 + d + k)
    B = 3
    x = torch.randn(B, T, d, generator=gen)
    lens = torch.tensor([T, max(1, (2 * T) // 3), 1], dtype=torch.int32)  # full, ragged (T not a multiple of 64), 1 frame
    x[1, int(lens[1]):] = 5.0 * torch.randn(T - int(lens[1]), d, generator=gen)  # padded frames hold values: must be masked
    x16 = x.half()
    cases = [("plain", _hm_weights(d, nhead, k, gen), lens, x16)]
    if T in (251, 1000):
        cases.append(("no_lens", cases[0][1], None, x16))
    if T == 1000 and d != 128:  # W1 biases and the inputs shifted so that max |H| > 65504: G needs its power-of-two scale
        cases.append(("large_H", _hm_weights(d, nhead, k, gen, w1_bias_shift=60.0), lens, (x + 2.0).half()))
    for name, w, ln, x16 in cases:
        kpm = None if ln is None else torch.arange(T)[None, :] >= ln[:, None].long()
        sd = {"m." + n: t for n, t in w.items()}
        ref = HO.hypermixing(x16.float(), sd, "m.", kpm)
        if name == "large_H":
            assert HO.max_abs_h(x16.float(), sd, "m.", kpm) > 65504.0
        out = _hm_dev(x16.to(dev), None if ln is None else ln.to(dev), w, nhead, k).cpu()
        valid = torch.ones(B, T, dtype=torch.bool) if kpm is None else ~kpm
        r_all = rel(out, ref)
        r_utt = [rel(out[b][valid[b]], ref[b][valid[b]]) for b in range(B)]
        print(f"hypermix T={T} d={d} nhead={nhead} k={k} {name}: rel-L2 {r_all:.2e}, valid frames per utterance "
              f"{['%.1e' % r for r in r_utt]}, max abs {float((out - ref).abs().max()):.2e}")
        assert torch.isfinite(out).all() and r_all <= KERNEL_BAR and max(r_utt) <= KERNEL_BAR
        if kpm is not None:  # a padded frame mixes nothing: its output is the LayerNorm's beta, exactly
            assert torch.equal(out[kpm], w["layer_norm.bias"].expand(int(kpm.sum()), d))
        assert torch.equal(out, _hm_dev(x16.to(dev), None if ln is None else ln.to(dev), w, nhead, k).cpu())


def test_hypermix_kernel_rejects_what_is_not_built(dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    x16 = torch.zeros(1, 3001, 144, device=dev, dtype=torch.float16)
    out = torch.empty(1, 3001, 144, device=dev)
    v = torch.ones(8 * 256 * 64, device=dev)
    st = stream_ptr(dev)
    args = [ptr(v)] * 10
    assert lib().sbk_hypermix_test(ptr(x16), None, 1, 16, 144, 8, 128, *args, ptr(out), st) != 0   # head width 18
    assert lib().sbk_hypermix_test(ptr(x16), None, 1, 16, 256, 8, 120, *args, ptr(out), st) != 0   # k not a multiple of 16
    assert lib().sbk_hypermix_test(ptr(x16), None, 1, 16, 256, 8, 272, *args, ptr(out), st) != 0   # k > 256
    assert lib().sbk_hypermix_test(ptr(x16), None, 1, 3001, 128, 4, 128, *args, ptr(out), st) != 0  # T > 3000
    assert lib().sbk_hypermix_test(ptr(x16), None, 1, 3000, 128, 4, 128, *args, ptr(out), st) == 0


# ------------------------------------------------------------------------------------------------ whole model
def _engine(fx, dev, parts=("fbank", "cnn", "encoder", "decoder"), gain=None):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    return AsrEngine(HYPERCONFORMER_22M, _state(fx, gain), device=dev, parts=parts)


def _oracle_states(fx, case):
    """The reference's encoder states of a fixture case, recomputed by the CPU oracle and checked against the stored
    per-frame norms and sampled rows."""
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    with torch.no_grad():
        ref = HO.wav_to_states(*case_wav(case), _state(fx), HYPERCONFORMER_22M)
    check_summary("hyperconformer_22M oracle", ref, case["frame_norm"], case["sample_idx"], case["sample_rows"], 1e-5)
    return ref


def test_hyperconformer_encoder_and_greedy(dev, fx):
    g = fx["main"]
    eng = _engine(fx, dev)
    wav, lens = case_wav(g)
    S = g["greedy_tokens"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), lens.to(dev), S, 1, 2, want_enc=True)
    torch.cuda.synchronize()
    assert done == S
    check_encoder("hyperconformer_22M 4x10s", enc.cpu(), _oracle_states(fx, g), g["abs_len"], ENC_BAR)
    check_greedy("hyperconformer_22M", pred.cpu(), score.cpu(), g["greedy_tokens"], g["greedy_margin"], g["greedy_chosen_lp"])
    check_alone_vs_batch(lambda w, ln: eng.encode_wav(w.to(dev), ln.to(dev)), wav, lens, 1e-5)


def test_hyperconformer_short_utterance(dev, fx):
    s = fx["short"]
    eng = _engine(fx, dev, parts=("fbank", "cnn", "encoder"))
    wav, lens = case_wav(s)
    enc = eng.encode_wav(wav.to(dev), lens.to(dev)).cpu()
    assert enc.shape == s["enc_out"].shape
    check_encoder("hyperconformer_22M short", enc, s["enc_out"], torch.tensor([enc.shape[1]]), ENC_BAR)


def test_hyperconformer_beam10_lm_ctc(dev, fx):
    """The recipe's test search (beam 10, [TransformerLM 0.6, CTC 0.4], temperature 1.15) on the reference's encoder states,
    judged by parity.check_beam: best scores and every rank of the n-best within 3e-2; a
    different best hypothesis only where the oracle, walked along our tokens, scores it within 3e-2 of ours and no worse
    than the reference's best."""
    import bench
    from oracle import asr_oracle as O
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    g, gb = fx["main"], fx["main"]["beam"]
    sd = _state(fx)
    asr = bench.build_product_asr(HYPERCONFORMER_22M, sd, dev, decoder="beam", beam=gb["kwargs"]["beam_size"], lm=True, ctc=True)
    bs = asr.mods["decoder"]
    bs.max_decode_ratio, bs.min_decode_ratio = gb["max_decode_ratio"], 0.0
    bs.return_topk, bs.topk = True, gb["kwargs"]["beam_size"]
    ref_enc = _oracle_states(fx, g)
    lens = g["wav_lens"]
    hyps, hlens, scores, _ = bs(ref_enc.to(dev), lens.to(dev))

    @torch.no_grad()
    def rescore_forced(idx, tokens):
        kw = {k_: v for k_, v in gb["kwargs"].items() if k_ != "beam_size"}
        ctc = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=0.4, blank_index=0)
        return O.beam_search(ref_enc[idx], lens[idx], sd, dict(HYPERCONFORMER_22M), sd["seq_lin.w.weight"], sd["seq_lin.w.bias"],
                             1, 2, beam_size=1, prefix="Transformer.", lm=oracle_lm(0.6, 1.15), ctc=ctc, forced=tokens, **kw)
    check_beam("beam10 lm+ctc", best_tokens(hyps, hlens), scores, best_tokens(gb["hyps"].long(), gb["lens"]), gb["scores"],
               rescore_forced)


def test_group_host_entry_matches_device(dev, fx):
    """The pinned-host group call (eager and one-graph modes) gives the ids of the device-resident group call."""
    import bench
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    cfg = dict(HYPERCONFORMER_22M, num_encoder_layers=3, num_decoder_layers=2)
    asr = bench.build_product_asr(cfg, _state(fx), dev)
    eng = asr.engine()
    gen = torch.Generator().manual_seed(3)
    B, L, S, G = 4, 48000, 16, 3
    wavs = [torch.randn(B, L, generator=gen).pin_memory() for _ in range(G)]
    lens = [torch.tensor([1.0, 0.8, 0.9, 0.5]).pin_memory() for _ in range(G)]
    asr.mods["decoder"].max_decode_ratio = (S + 0.5) / eng.num_frames(L)[1]
    ref = [torch.empty(B, S, dtype=torch.int32, device=dev) for _ in range(G)]
    eng.transcribe_greedy_group_dev([w.to(dev) for w in wavs], [l_.to(dev) for l_ in lens], S, 1, 2, ref)
    torch.cuda.synchronize()
    for poll in (8, 0):
        eng.set_poll_interval(poll)
        out = [torch.full((B, S), -7, dtype=torch.int32).pin_memory() for _ in range(G)]
        out_dev = [torch.full((B, S), -7, dtype=torch.int32, device=dev) for _ in range(G)]
        for _ in range(2):
            asr.transcribe_batches_async(wavs, lens, out, out_dev)
            torch.cuda.synchronize()
        for g_ in range(G):
            assert torch.equal(out[g_], ref[g_].cpu()) and torch.equal(out_dev[g_], ref[g_]), f"poll={poll} batch {g_}"


def test_load_state_dict_after_first_use(dev, fx):
    """New hypernetwork weights loaded into the mirror after it has run reach the device: the encoder states equal those
    of an engine built from the new weights, and differ from the old ones."""
    import bench
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    cfg = dict(HYPERCONFORMER_22M, num_encoder_layers=2, num_decoder_layers=1)
    asr = bench.build_product_asr(cfg, _state(fx), dev)
    wav, lens = case_wav(fx["short"])
    before = asr.encode_batch(wav.to(dev), lens.to(dev)).cpu()
    sd2 = _state(fx, gain=0.7, cfg=cfg)
    load(asr.transformer, sd2, "Transformer.")
    after = asr.encode_batch(wav.to(dev), lens.to(dev)).cpu()
    fresh = bench.build_product_asr(cfg, sd2, dev).encode_batch(wav.to(dev), lens.to(dev)).cpu()
    print(f"load_state_dict: change {rel(after, before):.2e}, vs a fresh engine max abs {float((after - fresh).abs().max()):.2e}")
    assert rel(after, before) > 1e-2 and torch.equal(after, fresh)
