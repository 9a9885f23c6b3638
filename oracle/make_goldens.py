"""Generate tests/golden/*.pt of the Conformer recipes by RUNNING THE REFERENCE (how to run it: oracle/goldens.py).

TEST INFRASTRUCTURE.  For every case it (1) builds the reference modules with the recipe's kwargs
(recipes/LibriSpeech/ASR/transformer/hparams/conformer_{large,small}.yaml), (2) loads seeded weights
(speechbrain_b200.utils.seeded_init -- regenerated, not stored), (3) runs the reference on seeded inputs, (4) checks
oracle/asr_oracle.py against it, and (5) stores inputs + reference outputs as small fixtures.
"""
import sys

import torch

from oracle import asr_oracle as O
from oracle import goldens as G
from speechbrain_b200.utils.seeded_init import seeded_asr_state

CFG_L = dict(name="conformer_large", d_model=512, nhead=8, num_encoder_layers=12, num_decoder_layers=6,
             d_ffn=2048, vocab=5000, n_fft=512, win_length=32, n_mels=80, kernel_size=31,
             cnn_channels=(64, 32), input_size=640)
CFG_S = dict(name="conformer_small", d_model=144, nhead=4, num_encoder_layers=12, num_decoder_layers=4,
             d_ffn=1024, vocab=5000, n_fft=400, win_length=25, n_mels=80, kernel_size=31,
             cnn_channels=(64, 32), input_size=640)


def weight_checksum(cfg, attention_type):
    """sum of |w| over the product's seeded state of the recipe (pins the seeded weights the tests regenerate)"""
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, CONFORMER_SMALL
    base = CONFORMER_LARGE if cfg["name"] == "conformer_large" else CONFORMER_SMALL
    state = seeded_asr_state(dict(base, attention_type=attention_type), 0)
    return float(sum(v.double().abs().sum() for k, v in sorted(state.items())))


def rope_case():
    """the reference of conformer_large with RoPE and the encoder states of conformer_large_rope.pt"""
    g = G.load("conformer_large_rope.pt")
    return G.build_reference(CFG_L, "RoPEMHA"), g["enc_out"], g["wav_lens"]


def fbank_cases():
    from speechbrain.lobes.features import Fbank
    g = torch.Generator().manual_seed(1234)
    out = {}
    for name, kw, B, L in [("cfg1_nfft400", dict(n_fft=400, n_mels=80), 1, 16000),
                           ("nfft400_b3_ragged", dict(n_fft=400, n_mels=80), 3, 12345),
                           ("nfft512_win32", dict(n_fft=512, n_mels=80, win_length=32), 2, 24000),
                           ("default_nmels40", dict(), 2, 8000),
                           ("nfft512_win25", dict(n_fft=512, n_mels=40), 1, 4800)]:
        wav = torch.randn(B, L, generator=g) * (0.1 if "ragged" in name else 1.0)
        if "ragged" in name:
            wav[1, 9000:] = 0
            wav[2, 5000:] = 0
        ref = Fbank(**kw)(wav)
        okw = dict(n_fft=kw.get("n_fft", 400), n_mels=kw.get("n_mels", 40), win_length_ms=kw.get("win_length", 25))
        ora = O.fbank(wav, **okw)
        err = (ora - ref).abs().max().item()
        print(f"fbank {name}: ref {tuple(ref.shape)} oracle max-abs err {err:.3e}")
        assert err < 1e-3
        out[name] = dict(kwargs=kw, wav=wav, out=ref)
    # all-zero utterance: amin clamp + top_db
    wav = torch.zeros(1, 1600)
    out["zeros"] = dict(kwargs=dict(n_fft=400, n_mels=80), wav=wav, out=Fbank(n_fft=400, n_mels=80)(wav))
    G.save(out, "fbank.pt")


def norm_cases():
    from speechbrain.processing.features import InputNormalization
    g = torch.Generator().manual_seed(7)
    x = torch.randn(3, 50, 80, generator=g) * 5 - 10
    lens = torch.tensor([1.0, 0.62, 0.3])
    out = {"x": x, "lens": lens}
    n = InputNormalization(norm_type="global")
    n.glob_mean = torch.randn(80, generator=g)
    n.glob_std = torch.rand(80, generator=g) + 0.5
    n.count = 1
    n.eval()
    out["glob_mean"], out["glob_std"] = n.glob_mean, n.glob_std
    out["global"] = n(x, lens)
    assert torch.equal(O.input_norm(x, lens, "global", n.glob_mean, n.glob_std), out["global"])
    n = InputNormalization(norm_type="sentence").eval()
    out["sentence"] = n(x, lens)
    print("norm sentence err", (O.input_norm(x, lens, "sentence") - out["sentence"]).abs().max().item())
    n = InputNormalization(norm_type="sentence", avoid_padding_norm=True).eval()
    out["sentence_avoid_pad"] = n(x, lens)
    assert (O.input_norm(x, lens, "sentence", avoid_padding_norm=True) - out["sentence_avoid_pad"]).abs().max() < 1e-5
    # KAT from tests/unittests/test_features.py:112-118
    kat = InputNormalization(norm_type="sentence").eval()(torch.tensor([[[1.0], [3.0], [0.0], [0.0], [0.0]]]),
                                                            torch.tensor([0.4]))
    out["kat"] = kat
    G.save(out, "input_norm.pt")


def model_case(cfg, attention_type, B, L, lens, n_steps, tag):
    ref = G.build_reference(cfg, attention_type)
    sd, mods = ref.sd, ref.mods
    wav, wav_lens, _ = G.wav_case(1234, B, L, lens)
    with torch.no_grad():
        f = ref.fb(wav)
        fn = ref.norm(f, wav_lens)
        c = mods["CNN"](fn)
        enc = mods["Transformer"].encode(c, wav_lens)
        T = enc.shape[1]
        hyps, logits = G.greedy_case(ref, enc, wav_lens, n_steps, tag)
        ctc_logits = mods["ctc_lin"](enc)
        # oracle checks
        of = O.fbank(wav, n_fft=cfg["n_fft"], n_mels=cfg["n_mels"], win_length_ms=cfg["win_length"])
        ofn = O.input_norm(of, wav_lens, "global", sd["normalize.glob_mean"], sd["normalize.glob_std"])
        oc = O.cnn_frontend(fn, sd, "CNN.")
        oenc, olayers = O.encode(c, wav_lens, sd, ref.cfg, "Transformer.", return_layers=True)
    print(f"[{tag}] fbank err {(of - f).abs().max():.2e}  norm err {(ofn - fn).abs().max():.2e} "
          f"cnn err {(oc - c).abs().max():.2e}  enc rel {G.rel(oenc, enc):.2e}")
    assert (oc - c).abs().max() < 1e-4 and G.rel(oenc, enc) < 1e-5
    top2 = logits.topk(2, dim=-1).values
    print(f"   T={T} steps={logits.shape[1]} min top1-top2 margin {float((top2[..., 0] - top2[..., 1]).min()):.4f}")
    gold = dict(cfg=dict(cfg, attention_type=attention_type), wav=wav, wav_lens=wav_lens, fbank=f, cnn_out=c, enc_out=enc,
                enc_layer0=olayers[0], enc_layer5=olayers[5], hyps=hyps, greedy_logits=logits,
                ctc_logits_head=ctc_logits[:, :, :64].clone(), weight_checksum=weight_checksum(cfg, attention_type))
    G.save(gold, f"{tag}.pt")


def beam_case(tag="beam_conformer_large_rope"):
    """S2STransformerBeamSearcher (no scorer) on the conformer_large_rope golden's encoder states."""
    ref, enc, wav_lens = rope_case()
    T = enc.shape[1]
    out = {}
    for name, kwargs, eos_bias in [
            ("thr_on", dict(beam_size=4, using_eos_threshold=True, temperature=1.0, min_decode_ratio=0.0), 4.0),
            ("recipe", dict(beam_size=5, using_eos_threshold=False, temperature=1.15, min_decode_ratio=2.5 / T), 5.5),
            ("no_eos", dict(beam_size=3, using_eos_threshold=False, length_normalization=False, min_decode_ratio=0.0), 0.0)]:
        hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, 8.5 / T, eos_bias, tag=f"beam {name}")
        out[name] = dict(kwargs=kwargs, eos_bias=eos_bias, max_decode_ratio=8.5 / T, hyps=hyps, lens=lens, scores=scores,
                         log_probs=lp)
    G.save(out, f"{tag}.pt")


def beam_topk_case(tag="beam_topk_conformer_large_rope"):
    """return_topk=True, topk=3 (the n-best output the rescorers consume): padded (B, topk, L) hypotheses, lengths, scores and
    log-probs of the reference vs the oracle."""
    ref, enc, wav_lens = rope_case()
    T = enc.shape[1]
    kwargs = dict(beam_size=5, using_eos_threshold=False, temperature=1.15, min_decode_ratio=2.5 / T)
    eos_bias = 5.5
    hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, 8.5 / T, eos_bias, topk=3, tag="beam topk")
    G.save(dict(kwargs=kwargs, eos_bias=eos_bias, max_decode_ratio=8.5 / T, topk=3, hyps=hyps, lens=lens, scores=scores,
                log_probs=lp), f"{tag}.pt")


def rescore_case(tag="lm_rescore"):
    """TransformerLMRescorer.rescore_hyps + RescorerBuilder.rescore of the reference (n-best rescoring of text hypotheses) with
    the recipe-size TransformerLM (seed 1) and a stub tokenizer."""
    import copy

    from speechbrain.decoders.scorer import RescorerBuilder, TransformerLMRescorer
    lm, sd_lm = G.reference_lm()
    tok = O.StubTokenizer()
    hyps = [["hello world", "hello word", "yellow world peace"], ["a b", "abc", "the cat sat on the mat"]]
    scores = [[-1.0, -1.2, -1.5], [-0.3, -0.35, -0.4]]
    resc = TransformerLMRescorer(language_model=lm, tokenizer=tok, device="cpu", temperature=1.15, bos_index=1, eos_index=2,
                                 pad_index=0)
    with torch.no_grad():
        ref = resc.rescore_hyps(hyps)
        ours = O.lm_rescore_hyps(hyps, tok, sd_lm, G.CFG_LM, 1.15, 1, 2, 0)
        rb = RescorerBuilder(weights={"transformerlm": 0.5}, rescorers=[resc])
        out_c, out_s = rb.rescore(hyps, copy.deepcopy(scores))
    o_c, o_s = O.rescorer_builder_rescore(hyps, scores, ours, 0.5)
    print(f"[rescore] ref {ref.tolist()} oracle err {(ours - ref).abs().max():.2e}; reranked {out_c} equal: {o_c == out_c}")
    assert (ours - ref).abs().max() < 1e-3 and o_c == out_c
    G.save(dict(hyps=hyps, scores=scores, temperature=1.15, weight=0.5, lm_scores=ref, out_candidates=out_c, out_scores=out_s),
           f"{tag}.pt")


def beam_len_case(tag="beam_len_conformer_large_rope"):
    """ScorerBuilder(full_scorers=[LengthScorer]) (length reward, no length normalisation): with the reward the search keeps
    longer hypotheses than without it."""
    ref, enc, wav_lens = rope_case()
    T = enc.shape[1]
    kwargs = dict(beam_size=4, using_eos_threshold=False, temperature=1.0, min_decode_ratio=0.0, length_normalization=False)
    eos_bias, w_len = 4.0, 8.3
    without = G.run_beam(ref, enc, wav_lens, kwargs, 8.5 / T, eos_bias, check=False)[0]
    hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, 8.5 / T, eos_bias, scorers={"length": w_len},
                                        tag="beam len")
    print(f"[beam len] without {without} with {hyps}")
    assert without != hyps
    G.save(dict(kwargs=kwargs, eos_bias=eos_bias, length_weight=w_len, max_decode_ratio=8.5 / T, hyps=hyps, lens=lens,
                scores=scores, log_probs=lp, hyps_without=without), f"{tag}.pt")


def beam_lm_case(tag="beam_lm_conformer_large_rope"):
    """S2STransformerBeamSearcher + ScorerBuilder(full_scorers=[TransformerLMScorer]) -- shallow fusion with the recipe's
    12 x 768 TransformerLM (conformer_large.yaml:160-170, 215-223), weight 0.6, temperature 1.15."""
    from speechbrain_b200.utils.shapes import transformer_lm_shapes
    ref, enc, wav_lens = rope_case()
    T = enc.shape[1]
    lm = G.reference_lm()
    ours = {k: tuple(v) for k, v in transformer_lm_shapes(5000).items()}
    ref_shapes = {k: tuple(v.shape) for k, v in lm[0].state_dict().items() if not k.endswith(".pe")}
    assert ours == ref_shapes, (set(ours) ^ set(ref_shapes))
    out = {}
    for name, kwargs, eos_bias in [
            ("lm_recipe", dict(beam_size=4, using_eos_threshold=False, temperature=1.15, min_decode_ratio=0.0), 0.0),
            ("lm_eos", dict(beam_size=3, using_eos_threshold=True, temperature=1.0, min_decode_ratio=1.5 / T), 9.0)]:
        hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, 6.5 / T, eos_bias, scorers={"transformerlm": 0.6},
                                            lm=lm, tag=f"beam+lm {name}")
        out[name] = dict(kwargs=kwargs, eos_bias=eos_bias, max_decode_ratio=6.5 / T, lm_weight=0.6, lm_temperature=1.15,
                         hyps=hyps, lens=lens, scores=scores, log_probs=lp)
    G.save(out, f"{tag}.pt")


def scorers(with_lm, with_ctc):
    """the recipe's full scorers (conformer_large.yaml:209-228): TransformerLM 0.6 and / or CTC 0.4, in its order"""
    return dict(([("transformerlm", 0.6)] if with_lm else []) + ([("ctc", 0.4)] if with_ctc else []))


def beam_ctc_case(tag="beam_ctc_conformer_large_rope"):
    """Joint CTC/attention decoding: ScorerBuilder(full_scorers=[TransformerLMScorer, CTCScorer]) (the recipe's test search,
    conformer_large.yaml:209-223: lm 0.60, ctc 0.40) and full_scorers=[CTCScorer] (the valid search, :225-228)."""
    ref, enc, wav_lens = rope_case()
    T = enc.shape[1]
    lm = G.reference_lm()
    out = {}
    for name, with_lm, kwargs, eos_bias, steps in [
            ("ctc_lm_test", True, dict(beam_size=4, using_eos_threshold=False, temperature=1.15, min_decode_ratio=0.0), 0.0,
             10.5),
            ("ctc_valid", False, dict(beam_size=5, using_eos_threshold=False, temperature=1.15, min_decode_ratio=0.0), 0.0,
             10.5),
            ("ctc_eos", False, dict(beam_size=3, using_eos_threshold=True, temperature=1.0, min_decode_ratio=1.5 / T), 9.0,
             8.5)]:
        hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, steps / T, eos_bias, scorers=scorers(with_lm, True),
                                            lm=lm, bar=1e-3, tag=f"beam+ctc {name}")
        out[name] = dict(kwargs=kwargs, eos_bias=eos_bias, max_decode_ratio=steps / T, with_lm=with_lm, lm_weight=0.6,
                         lm_temperature=1.15, ctc_weight=0.4, hyps=hyps, lens=lens, scores=scores, log_probs=lp)
    G.save(out, f"{tag}.pt")


def bench_beam(ref, enc, wav_lens, kwargs, steps, eos_bias, tag, with_lm=False, with_ctc=False, lm=None, **record):
    """A bench-shape beam case: the n-best of all beam_size hypotheses, best hypothesis and every score checked against
    the oracle (1e-3); its fixture record"""
    T, beam = enc.shape[1], kwargs["beam_size"]
    hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, (steps + 0.5) / T, eos_bias,
                                        scorers=scorers(with_lm, with_ctc), lm=lm, topk=beam, bar=1e-3, rank0=True, tag=tag)
    print(f"   best lens {(lens[:, 0] * hyps.shape[2]).round().int().tolist()} max len {hyps.shape[2]}; "
          f"top1-top2 score gap {(scores[:, 0] - scores[:, 1]).tolist()}")
    return dict(kwargs=kwargs, with_lm=with_lm, with_ctc=with_ctc, eos_bias=eos_bias, max_decode_ratio=(steps + 0.5) / T,
                **record, hyps=hyps.int(), lens=lens, scores=scores, log_probs=lp)


def bench_shape_case(cfg, attention_type, B, L, lens, n_greedy, tag, beams=(), seed=4321):
    """Goldens at the shapes bench.py runs (VERDICT r1 #1): 10 s utterances -> T = 251 = four 64-key attention blocks, ragged
    lengths so that one trailing key block is partially and one fully masked, 48 greedy steps (KV-cache positions 0..47),
    beam = 10 with the recipe's scorers.  The waveform is regenerated from ``seed`` by the test (a checksum pins it); stored:
    reference enc_out (fp32), greedy tokens / chosen log-probs / top-2 margins, beam n-best (all `beam` hypotheses + scores)."""
    ref = G.build_reference(cfg, attention_type)
    wav, wav_lens, record = G.wav_case(seed, B, L, lens)
    gold = dict(cfg=dict(cfg, attention_type=attention_type), **record,
                weight_checksum=weight_checksum(cfg, attention_type))
    with torch.no_grad():
        enc = ref.encode(wav, wav_lens)
        T = enc.shape[1]
        oc = O.full_pipeline_features(wav, wav_lens, ref.sd, dict(cfg))
        oenc = O.encode(oc, wav_lens, ref.sd, ref.cfg, "Transformer.")
    print(f"[{tag}] T={T} encoder: oracle rel {G.rel(oenc, enc):.2e}")
    assert G.rel(oenc, enc) < 1e-5
    gold["enc_out"] = enc.clone()
    gold["abs_len"] = torch.round(wav_lens * T).int()
    if n_greedy > 0:
        hyps, logits = G.greedy_case(ref, enc, wav_lens, n_greedy, tag)
        gold.update(G.greedy_record(hyps, logits),
                    greedy_lp_sample=torch.log_softmax(logits, -1)[:, :, :128].clone().half())
    lm = G.reference_lm() if any(kw["with_lm"] for _, kw in beams) else None
    for name, kw in beams:
        kw = dict(kw)
        with_lm, with_ctc, eos_bias, steps = kw.pop("with_lm"), kw.pop("with_ctc"), kw.pop("eos_bias"), kw.pop("steps")
        kw.setdefault("min_decode_ratio", 0.0)
        gold["beam_" + name] = bench_beam(ref, enc, wav_lens, kw, steps, eos_bias, f"{tag} beam {name}", with_lm, with_ctc,
                                          lm, lm_weight=0.6, lm_temperature=1.15, ctc_weight=0.4)
    G.save(gold, f"{tag}.pt")


def bench_extra_case(tag="bench_decode_conformer_large_rope_10s"):
    """On the encoder states of the bench-shape RoPE golden: (1) TransformerASR.decode(tgt, enc, enc_len) of the reference,
    teacher-forced on the greedy tokens (48 positions, ragged memory lengths) -> decoder outputs [4, 48, 512];
    (2) beam = 10 without scorers, EOS bias chosen so that hypotheses finish gradually over many steps."""
    ref = G.build_reference(CFG_L, "RoPEMHA")
    g = G.load("bench_conformer_large_rope_10s.pt")
    enc, wav_lens = g["enc_out"], g["wav_lens"]
    T = enc.shape[1]
    out = {}
    with torch.no_grad():
        tgt = torch.cat([torch.full((enc.shape[0], 1), 1, dtype=torch.long), g["greedy_tokens"].long()[:, :-1]], 1)
        enc_len = torch.round(wav_lens * T).int()
        pred, attn = ref.mods["Transformer"].decode(tgt, enc, enc_len)
        opred, _ = O.decode(tgt, enc, enc_len, ref.sd, ref.cfg, "Transformer.")
    print(f"[decode] pred {tuple(pred.shape)} oracle rel {G.rel(opred, pred):.2e}")
    assert G.rel(opred, pred) < 1e-5
    out["decode"] = dict(tgt=tgt.int(), enc_len=enc_len, pred=pred.clone())
    for name, eos_bias, steps in (("b10_plain_eos12", 1.2, 48), ("b10_plain_eos16", 1.6, 48)):
        kw = dict(beam_size=10, using_eos_threshold=False, temperature=1.15, min_decode_ratio=3.5 / T)
        out["beam_" + name] = bench_beam(ref, enc, wav_lens, kw, steps, eos_bias, f"beam {name}")
    G.save(out, f"{tag}.pt")


def ctc_greedy_case(tag="ctc_greedy_conformer_large_rope"):
    """EncoderASR-style CTC greedy decoding (inference/ASR.py:325-373, decoders/ctc.py:335-378) of the reference on the golden
    encoder states: log_softmax(ctc_lin(enc)) -> ctc_greedy_decode(blank 0).  Random-init posteriors almost never repeat, so a
    second case adds a bias to the blank and to one token to exercise the merge / blank-filter rules."""
    from speechbrain.decoders.ctc import ctc_greedy_decode
    ref, enc, wav_lens = rope_case()
    sd, mods = ref.sd, ref.mods
    out = {}
    for name, bias_blank, bias_tok in (("plain", 0.0, 0.0), ("merge", 1.2, 1.1)):
        with torch.no_grad():
            bias = sd["ctc_lin.w.bias"].clone()
            bias[0] += bias_blank
            bias[17] += bias_tok
            mods["ctc_lin"].w.bias.copy_(bias)
            lp = torch.log_softmax(mods["ctc_lin"](enc), dim=-1)
            hyps = ctc_greedy_decode(lp, wav_lens, blank_id=0)
            olp = O.ctc_log_probs(enc, sd["ctc_lin.w.weight"], bias)
            ohyps = O.ctc_greedy_decode(olp, wav_lens, 0)
        top2 = lp.topk(2, -1).values
        print(f"[ctc greedy {name}] hyps lens {[len(h) for h in hyps]} of T={enc.shape[1]}; oracle equal {ohyps == hyps}; "
              f"min margin {float((top2[..., 0] - top2[..., 1]).min()):.4f}")
        assert ohyps == hyps and (olp - lp).abs().max() < 1e-4
        out[name] = dict(bias_blank=bias_blank, bias_tok=bias_tok, hyps=hyps, argmax=lp.argmax(-1).int(),
                         margin=(top2[..., 0] - top2[..., 1]).clone(), log_probs_head=lp[:, :, :64].clone())
    with torch.no_grad():
        mods["ctc_lin"].w.bias.copy_(sd["ctc_lin.w.bias"])
    G.save(out, f"{tag}.pt")


# "ffn": first FFN layers x200 and second layers / 200: hidden activations (the fp16-stored tensor) in the hundreds while the
# FFN output keeps its scale, so the residual structure of the model survives (x200 alone turns the encoder into a
# 24-deep non-residual chain in which ANY rounding error compounds: measured 2e-3 with fp16, same with exact SiLU).
SCALES = {"ffn": {"ffn_w1": 200.0, "ffn_w2": 1.0 / 200.0, "qkv": 1.0, "pw1": 1.0},
          "attn": {"ffn_w1": 1.0, "qkv": 3.0, "pw1": 4.0}}        # attention logits x9 (peaky softmax), GLU inputs x4


def scale_state(sd, scales):
    """Seeded weights with selected matrices scaled up (fp16-range test): FFN first layers, attention in_proj, conv pw1."""
    out = dict(sd)
    for k, v in sd.items():
        if ".ffn_module" in k and k.endswith("ffn.0.weight"):
            out[k] = v * scales["ffn_w1"]
        elif ".ffn_module" in k and k.endswith("ffn.3.weight"):
            out[k] = v * scales.get("ffn_w2", 1.0)
        elif k.endswith("mha_layer.in_proj_weight"):
            out[k] = v * scales["qkv"]
        elif k.endswith("convolution_module.bottleneck.0.weight"):
            out[k] = v * scales["pw1"]
    return out


def scaled_case(tag="conformer_large_rope_scaled"):
    """fp16 range (VERDICT r1 #8): the 2 s RoPE golden re-run by the reference with (a) FFN pre-activations pushed into the
    hundreds, (b) attention logits x9 and GLU inputs x4 -- far above what random init gives."""
    g = G.load("conformer_large_rope.pt")
    out = {}
    for name, sc in SCALES.items():
        ref = G.build_reference(CFG_L, "RoPEMHA")
        sds = scale_state(ref.sd, sc)
        ref.mods.load_state_dict({k: v for k, v in sds.items() if not k.startswith("normalize.")})
        stats = {"ffn_hidden_absmax": 0.0}

        def hook_ffn(m, i, o):
            stats["ffn_hidden_absmax"] = max(stats["ffn_hidden_absmax"], float(o.abs().max()))
        for layer in ref.mods["Transformer"].encoder.layers:
            layer.ffn_module1[1].ffn[0].register_forward_hook(hook_ffn)
            layer.ffn_module2[1].ffn[0].register_forward_hook(hook_ffn)
        with torch.no_grad():
            enc = ref.mods["Transformer"].encode(g["cnn_out"], g["wav_lens"])
            oenc = O.encode(g["cnn_out"].reshape(g["cnn_out"].shape[0], g["cnn_out"].shape[1], -1), g["wav_lens"], sds,
                            ref.cfg, "Transformer.")
        print(f"[scaled {name}] enc finite {bool(torch.isfinite(enc).all())} oracle rel {G.rel(oenc, enc):.2e} max |FFN "
              f"pre-activation| {stats['ffn_hidden_absmax']:.1f} enc absmax {float(enc.abs().max()):.2f}")
        assert G.rel(oenc, enc) < 1e-5
        out[name] = dict(scales=sc, enc_out=enc, ffn_hidden_absmax=stats["ffn_hidden_absmax"])
    G.save(out, f"{tag}.pt")


def beam66_case(tag="beam66_conformer_large_rope"):
    """beam_size = 66, the recipe's test_beam_size (conformer_large.yaml:132), on the 2 s golden: scorer-less, temperature
    1.15, a small EOS bias so that hypotheses finish at different steps.  All 66 hypotheses per utterance are stored."""
    ref, enc, wav_lens = rope_case()
    kw = dict(beam_size=66, using_eos_threshold=False, temperature=1.15, min_decode_ratio=2.5 / enc.shape[1])
    G.save(bench_beam(ref, enc, wav_lens, kw, 10, 1.5, "beam66"), f"{tag}.pt")


def beam_cov_case(tag="beam_cov_conformer_large_rope"):
    """ScorerBuilder(full_scorers=[CoverageScorer]) (scorer.py:788-955): coverage penalty on the last decoder layer's
    head-averaged cross-attention, weight chosen large enough to change the result of the scorer-less search."""
    ref, enc, wav_lens = rope_case()
    T = enc.shape[1]
    kwargs = dict(beam_size=5, using_eos_threshold=False, temperature=1.15, min_decode_ratio=2.5 / T)
    eos_bias, w_cov, thr, steps = 1.5, 40.0, 0.05, 10
    without = G.run_beam(ref, enc, wav_lens, kwargs, (steps + 0.5) / T, eos_bias, topk=5, check=False)[2]
    hyps, lens, scores, lp = G.run_beam(ref, enc, wav_lens, kwargs, (steps + 0.5) / T, eos_bias, scorers={"coverage": w_cov},
                                        coverage_threshold=thr, topk=5, bar=1e-3, rank0=True, tag="beam cov")
    print(f"[beam cov] best scores without {without[:, 0].tolist()} with {scores[:, 0].tolist()}")
    assert not torch.equal(without, scores)
    G.save(dict(kwargs=kwargs, with_lm=False, with_ctc=False, eos_bias=eos_bias, coverage_weight=w_cov, coverage_threshold=thr,
                max_decode_ratio=(steps + 0.5) / T, hyps=hyps.int(), lens=lens, scores=scores, log_probs=lp,
                scores_without=without), f"{tag}.pt")


def dynchunk_case(tag="dynchunk_conformer_large"):
    """TransformerASR.encode(src, wav_len, dynchunktrain_config=DynChunkTrainConfig(chunk_size, left_context_size)) -- the
    masked ("streaming-equivalent") evaluation mode (TransformerASR.py:46-105,475-544; Conformer.py:190-313 Dynamic Chunk
    Convolution): chunked attention masks + future-masked convolution.  RoPE with a finite left context and RelPos with an
    infinite one, ragged batch, chunk sizes that do not divide T = 51."""
    from speechbrain.utils.dynamic_chunk_training import DynChunkTrainConfig
    out = {}
    for att, cs, lc in (("RoPEMHA", 8, 2), ("RelPosMHAXL", 16, None), ("RoPEMHA", 5, 3), ("RelPosMHAXL", 4, 4)):
        ref = G.build_reference(CFG_L, att)
        g = G.load("conformer_large_rope.pt" if att == "RoPEMHA" else "conformer_large_relpos.pt")
        with torch.no_grad():
            enc = ref.mods["Transformer"].encode(g["cnn_out"], g["wav_lens"], dynchunktrain_config=DynChunkTrainConfig(cs, lc))
            src = g["cnn_out"].reshape(g["cnn_out"].shape[0], g["cnn_out"].shape[1], -1)
            oenc = O.encode(src, g["wav_lens"], ref.sd, ref.cfg, "Transformer.", dynchunk=(cs, lc))
        print(f"[dynchunk {att} chunk {cs} left {lc}] oracle rel {G.rel(oenc, enc):.2e}; differs from full-context by "
              f"{G.rel(enc, g['enc_out']):.2e}")
        assert G.rel(oenc, enc) < 1e-5 and G.rel(enc, g["enc_out"]) > 1e-2
        out[f"{att}_{cs}_{lc}"] = dict(attention_type=att, chunk_size=cs, left_context_size=lc, enc_out=enc)
    G.save(out, f"{tag}.pt")


BEAMS_10S = (
    ("b10_lm_ctc", dict(beam_size=10, using_eos_threshold=False, temperature=1.15, with_lm=True, with_ctc=True, eos_bias=0.0, steps=24)),
    ("b10_ctc_valid", dict(beam_size=10, using_eos_threshold=False, temperature=1.15, with_lm=False, with_ctc=True, eos_bias=0.0, steps=24)),
    ("b10_plain_eos", dict(beam_size=10, using_eos_threshold=False, temperature=1.15, min_decode_ratio=3.5 / 251, with_lm=False,
                           with_ctc=False, eos_bias=6.0, steps=48)),
)

CASES = {
    "fbank": fbank_cases,
    "norm": norm_cases,
    "L_rope": lambda: model_case(CFG_L, "RoPEMHA", 2, 32000, [1.0, 0.7], 6, "conformer_large_rope"),
    "L_relpos": lambda: model_case(CFG_L, "RelPosMHAXL", 2, 32000, [1.0, 0.7], 6, "conformer_large_relpos"),
    "S_relpos": lambda: model_case(CFG_S, "RelPosMHAXL", 2, 24000, [0.8, 1.0], 6, "conformer_small_relpos"),
    "beam": beam_case,
    "beam_topk": beam_topk_case,
    "beam_lm": beam_lm_case,
    "rescore": rescore_case,
    "beam_len": beam_len_case,
    "beam_ctc": beam_ctc_case,
    # not in the default list: minutes of CPU time each
    "bench_L_rope": lambda: bench_shape_case(CFG_L, "RoPEMHA", 4, 160000, [1.0, 0.9, 0.6, 0.3], 48,
                                             "bench_conformer_large_rope_10s", BEAMS_10S),
    "bench_L_relpos": lambda: bench_shape_case(CFG_L, "RelPosMHAXL", 4, 160000, [1.0, 0.9, 0.6, 0.3], 48,
                                               "bench_conformer_large_relpos_10s"),
    "dynchunk": dynchunk_case,
    "beam_cov": beam_cov_case,
    "beam66": beam66_case,
    "scaled": scaled_case,
    "ctc_greedy": ctc_greedy_case,
    "bench_extra": bench_extra_case,
    "bench_S_relpos": lambda: bench_shape_case(CFG_S, "RelPosMHAXL", 8, 80000, [1.0, 0.95, 0.9, 0.8, 0.7, 0.55, 0.4, 0.25],
                                               0, "bench_conformer_small_relpos_5s"),
}
DEFAULT = ["fbank", "norm", "L_rope", "L_relpos", "S_relpos", "beam", "beam_topk", "beam_lm", "beam_ctc", "rescore", "beam_len"]


if __name__ == "__main__":
    torch.manual_seed(0)
    which = sys.argv[1:] or DEFAULT
    for name, case in CASES.items():
        if name in which:
            case()
