"""-m gpu parity tests at the shapes bench.py runs (VERDICT r1 #1): 10 s utterances (T = 251 = four 64-key attention blocks),
ragged lengths [1.0, 0.9, 0.6, 0.3] so that trailing key blocks are partially / fully masked, 48 greedy steps (KV-cache
positions 0..47), beam = 10 with the recipe's scorers, Conformer-small 8 x 5 s -- all against outputs of the RUNNING
REFERENCE committed under tests/golden/bench_*.pt (generator: oracle/make_goldens.py bench_*).

Bars: encoder rel-L2 <= 1e-3 (north_star); greedy tokens identical up to the first decision whose reference top-1/top-2
margin is below 5e-3 (fp16 operands move logits by ~1e-3), chosen log-probs within 2e-2; beam search: identical best
hypothesis, or -- when fp16 rounding made the search pick another near-tied hypothesis -- a hypothesis the CPU oracle
(pinned against the reference by the generator) scores within 3e-2 of what we report and no worse than the reference's best
minus 3e-2."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mirrors import build_mirror, load, raise_bias, seeded  # noqa: E402
from parity import (best_tokens, case_wav, check_beam, check_ctc_argmax, check_encoder, check_greedy, dev,  # noqa: E402,F401
                    oracle_lm, rel)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

pytestmark = pytest.mark.gpu


def _cfg(g):
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, CONFORMER_SMALL
    base = CONFORMER_LARGE if g["cfg"]["name"] == "conformer_large" else CONFORMER_SMALL
    return dict(base, attention_type=g["cfg"]["attention_type"])


def _engine(cfg, dev, parts=("fbank", "cnn", "encoder", "decoder")):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    sd = seeded_asr_state(cfg, 0)
    return AsrEngine(cfg, sd, device=dev, parts=parts), sd


@pytest.mark.parametrize("tag", ["bench_conformer_large_rope_10s", "bench_conformer_large_relpos_10s"])
def test_bench_shape_encoder_and_greedy(dev, tag):
    """wav -> Fbank -> CMVN -> CNN -> 12 Conformer layers (multi-block flash attention, ragged key masks) -> 48 greedy steps,
    through the fused device pipeline (C ABI sbk_asr_transcribe_greedy_dev), vs the reference."""
    g = torch.load(os.path.join(GOLDEN, tag + ".pt"))
    cfg = _cfg(g)
    eng, sd = _engine(cfg, dev)
    chk = float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))
    assert abs(chk - g["weight_checksum"]) / g["weight_checksum"] < 1e-9, "seeded weights differ from the golden run"
    wav, lens = case_wav(g)
    S = g["greedy_tokens"].shape[1]
    for tc_rows, name in ((1 << 30, "weight-streaming"), (1, "wgmma")):
        eng.set_decoder_tc_min_rows(tc_rows)
        pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), lens.to(dev), S, 1, 2, want_enc=True)
        torch.cuda.synchronize()
        assert done == S
        check_encoder(f"{tag}/{name}", enc.cpu(), g["enc_out"], g["abs_len"], 1e-3)
        check_greedy(f"{tag}/{name}", pred.cpu(), score.cpu(), g["greedy_tokens"], g["greedy_margin"], g["greedy_chosen_lp"],
                     min_compared=0.6)


def test_bench_shape_conformer_small(dev):
    """BASELINE config 2: Conformer-small (12L / 144d / 4 heads of 36 / RelPosMHAXL / n_fft 400), 8 x 5 s ragged, wav ->
    encoder states through the fused pipeline vs the reference."""
    g = torch.load(os.path.join(GOLDEN, "bench_conformer_small_relpos_5s.pt"))
    cfg = _cfg(g)
    eng, sd = _engine(cfg, dev, parts=("fbank", "cnn", "encoder"))
    wav, lens = case_wav(g)
    enc = eng.encode_wav(wav.to(dev), lens.to(dev)).cpu()
    r = rel(enc, g["enc_out"])
    print(f"[conformer_small 8x5s] encoder rel-L2 err {r:.3e} max abs {(enc - g['enc_out']).abs().max():.3e}")
    assert enc.shape == g["enc_out"].shape and r < 1e-3
    eng.set_poll_interval(0)  # the encode-only CUDA-graph path
    enc2 = eng.encode_wav(wav.to(dev), lens.to(dev)).cpu()
    assert torch.equal(enc, enc2)


def test_bench_shape_decode_teacher_forced(dev):
    """TransformerASR.decode(tgt, encoder_out, enc_len) (TransformerASR.py:426-473) on 4 x T=251 memories with ragged
    lengths, 48 target positions, vs the reference's decoder outputs."""
    import bench
    g = torch.load(os.path.join(GOLDEN, "bench_conformer_large_rope_10s.pt"))
    gd = torch.load(os.path.join(GOLDEN, "bench_decode_conformer_large_rope_10s.pt"))["decode"]
    cfg = _cfg(g)
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    asr = bench.build_product_asr(cfg, seeded_asr_state(cfg, 0), dev)
    tr = asr.transformer
    pred, attn = tr.decode(gd["tgt"].to(dev), g["enc_out"].to(dev), gd["enc_len"].to(dev))
    r = rel(pred.cpu(), gd["pred"])
    print(f"decode(tgt, enc, enc_len): rel-L2 err {r:.3e} max abs {(pred.cpu() - gd['pred']).abs().max():.3e}")
    assert pred.shape == gd["pred"].shape and attn is None and r < 2e-3


BEAM_CASES = [("bench_conformer_large_rope_10s", "beam_b10_lm_ctc"), ("bench_conformer_large_rope_10s", "beam_b10_ctc_valid"),
              ("bench_decode_conformer_large_rope_10s", "beam_b10_plain_eos12"),
              ("bench_decode_conformer_large_rope_10s", "beam_b10_plain_eos16")]


@pytest.mark.parametrize("file,case", BEAM_CASES)
def test_bench_shape_beam10(dev, file, case):
    """BASELINE config 4 family: beam = 10 on T = 251 memories: [TransformerLM 0.6, CTC 0.4] (test search), [CTC] (valid
    search) for 24 steps, and scorer-less searches whose hypotheses finish gradually (up to 48 steps)."""
    g = torch.load(os.path.join(GOLDEN, "bench_conformer_large_rope_10s.pt"))
    gb = torch.load(os.path.join(GOLDEN, file + ".pt"))[case]
    _run_beam_case(dev, g, gb, case)


def test_beam66_recipe_width(dev):
    """beam_size = 66 (the recipe's test_beam_size, conformer_large.yaml:132) through the radix-select beam kernel, vs the
    reference on the 2 s golden."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam66_conformer_large_rope.pt"))
    _run_beam_case(dev, g, gb, "beam66")


def test_beam_search_with_coverage_scorer(dev):
    """ScorerBuilder(full_scorers=[CoverageScorer]) (scorer.py:788-955, penalty on the cumulative last-layer cross-attention)
    vs the reference on the 2 s golden; the weight is large enough that the result differs from the scorer-less search."""
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_cov_conformer_large_rope.pt"))
    _run_beam_case(dev, g, gb, "coverage")


def _run_beam_case(dev, g, gb, case):
    import bench
    from oracle import asr_oracle as O
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    cfg = _cfg(g)
    sd = seeded_asr_state(cfg, 0)
    sd["seq_lin.w.bias"] = sd["seq_lin.w.bias"].clone()
    sd["seq_lin.w.bias"][2] += gb["eos_bias"]
    cov = (gb["coverage_weight"], gb["coverage_threshold"]) if "coverage_weight" in gb else None
    asr = bench.build_product_asr(cfg, sd, dev, decoder="beam", beam=gb["kwargs"]["beam_size"], lm=gb["with_lm"], ctc=gb["with_ctc"],
                                  coverage=cov)
    bs = asr.mods["decoder"]
    bs.max_decode_ratio, bs.min_decode_ratio = gb["max_decode_ratio"], gb["kwargs"].get("min_decode_ratio", 0.0)
    bs.return_topk, bs.topk = True, gb["kwargs"]["beam_size"]
    enc, lens = g["enc_out"].to(dev), g["wav_lens"].to(dev)
    hyps, hlens, scores, lp = bs(enc, lens)
    if gb["with_lm"] or case.endswith("eos16"):
        # the same search with every projection (decoder AND TransformerLM step) on the wgmma GEMM instead of the
        # weight-streaming kernel (what wide beams / many utterances use): same hypotheses, scores within 2e-3
        bs._get_engine(dev).set_decoder_tc_min_rows(1)
        h2, l2, s2, _ = bs(enc, lens)
        bs._get_engine(dev).set_decoder_tc_min_rows(64)
        print(f"beam[{case}] wgmma GEMM projections: best scores {s2[:, 0].tolist()}")
        assert (s2[:, 0].cpu() - scores[:, 0].cpu()).abs().max() < 2e-3

    @torch.no_grad()
    def rescore_forced(idx, tokens):  # the CPU oracle walked along our tokens, with the case's scorers
        lm = oracle_lm(0.6, 1.15) if gb["with_lm"] else None
        ctc = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=0.4, blank_index=0) if gb["with_ctc"] else None
        kw = {k_: v for k_, v in gb["kwargs"].items() if k_ != "beam_size"}
        return O.beam_search(g["enc_out"][idx], g["wav_lens"][idx], sd, dict(g["cfg"]), sd["seq_lin.w.weight"], sd["seq_lin.w.bias"],
                             1, 2, beam_size=1, prefix="Transformer.", lm=lm, ctc=ctc, forced=tokens,
                             coverage=dict(weight=cov[0], threshold=cov[1]) if cov else None, **kw)
    check_beam(f"beam[{case}]", best_tokens(hyps, hlens), scores, best_tokens(gb["hyps"].long(), gb["lens"]), gb["scores"],
               rescore_forced)


def _sub_lens(g, idx):
    """Relative lengths of a subset: the oracle derives absolute lengths as round(T * rel) with T fixed, so they carry over."""
    return g["wav_lens"][idx]


def test_encoder_decoder_asr_interface(dev):
    """EncoderDecoderASR in the reference's module layout (encoder = LengthsCapableSequential(...), transformer, decoder):
    encode_batch / transcribe_batch on host and device tensors, greedy and beam decoders, one shared engine that follows
    load_state_dict."""
    import bench
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gb = torch.load(os.path.join(GOLDEN, "beam_conformer_large_rope.pt"))["recipe"]
    cfg = _cfg(g)
    sd = seeded_asr_state(cfg, 0)
    asr = bench.build_product_asr(cfg, sd, dev)
    T = g["enc_out"].shape[1]
    n_steps = g["greedy_logits"].shape[1]
    asr.mods["decoder"].max_decode_ratio = (n_steps + 0.5) / T
    enc = asr.encode_batch(g["wav"], g["wav_lens"])
    assert rel(enc.cpu(), g["enc_out"]) < 1.5e-3
    words_h, toks_h = asr.transcribe_batch(g["wav"].pin_memory(), g["wav_lens"])       # host tensors (C-ABI host entry)
    words_d, toks_d = asr(g["wav"].to(dev), g["wav_lens"].to(dev))                     # device tensors, forward()
    print("EncoderDecoderASR greedy tokens", toks_h, "reference", g["hyps"])
    assert toks_h == toks_d == g["hyps"] and words_h == [" ".join(map(str, h)) for h in toks_h]
    # the searcher and the interface share ONE engine; TransformerASR.encode reuses it too
    slot = asr.transformer.engine_slot(asr.mods["decoder"].engine_key())
    builds = slot.builds
    enc2 = asr.transformer.encode(g["cnn_out"].to(dev), g["wav_lens"].to(dev))
    hy, _, _, _ = asr.mods["decoder"](enc, g["wav_lens"].to(dev))
    assert slot.builds == builds and hy == g["hyps"] and rel(enc2.cpu(), g["enc_out"]) < 1e-3
    # load_state_dict after first use must take effect (ADVICE r1: stale snapshot)
    load(asr.mods["decoder"].fc, raise_bias(sd, "seq_lin", {7: 100.0}), "seq_lin.")
    _, toks_new = asr.transcribe_batch(g["wav"].to(dev), g["wav_lens"].to(dev))
    assert slot.builds == builds + 1 and all(set(t) == {7} for t in toks_new), toks_new
    # beam decoder through the same interface, reference wiring (eos bias so that hypotheses finish)
    asr_b = bench.build_product_asr(cfg, raise_bias(sd, "seq_lin", {2: gb["eos_bias"]}), dev, decoder="beam", beam=gb["kwargs"]["beam_size"])
    bs = asr_b.mods["decoder"]
    bs.max_decode_ratio, bs.min_decode_ratio, bs.temperature = gb["max_decode_ratio"], gb["kwargs"]["min_decode_ratio"], gb["kwargs"]["temperature"]
    bs.using_eos_threshold = gb["kwargs"]["using_eos_threshold"]
    words, toks = asr_b.transcribe_batch(g["wav"], g["wav_lens"])
    print("EncoderDecoderASR beam tokens", toks, "reference", gb["hyps"])
    assert toks == gb["hyps"]


def test_group_host_entry_matches_device(dev):
    """sbk_asr_transcribe_greedy_group_host_async (pinned host buffers, H2D/D2H inside, eager and whole-graph modes) gives the
    ids of the device-resident group call; also covers the greedy early-exit trimming with a forced EOS."""
    import bench
    from speechbrain_b200.decoders.seq2seq import greedy_exit_step
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    cfg = dict(CONFORMER_LARGE, num_encoder_layers=2, num_decoder_layers=2)
    sd = seeded_asr_state(cfg, 0)
    asr = bench.build_product_asr(cfg, sd, dev)
    eng = asr.engine()
    gen = torch.Generator().manual_seed(3)
    B, L, S, G = 4, 48000, 16, 3
    wavs = [torch.randn(B, L, generator=gen).pin_memory() for _ in range(G)]
    lens = [torch.tensor([1.0, 0.8, 0.9, 0.5]).pin_memory() for _ in range(G)]
    asr.mods["decoder"].max_decode_ratio = (S + 0.5) / eng.num_frames(L)[1]
    ref = [torch.empty(B, S, dtype=torch.int32, device=dev) for _ in range(G)]
    eng.transcribe_greedy_group_dev([w.to(dev) for w in wavs], [l_.to(dev) for l_ in lens], S, 1, 2, ref)
    torch.cuda.synchronize()
    for poll in (8, 0):  # eager launches, then the whole call as one CUDA graph (memcpy nodes included)
        eng.set_poll_interval(poll)
        out = [torch.full((B, S), -7, dtype=torch.int32).pin_memory() for _ in range(G)]
        out_dev = [torch.full((B, S), -7, dtype=torch.int32, device=dev) for _ in range(G)]
        for _ in range(2):  # second call replays the cached graph
            asr.transcribe_batches_async(wavs, lens, out, out_dev)
            torch.cuda.synchronize()
        for g_ in range(G):
            assert torch.equal(out[g_], ref[g_].cpu()) and torch.equal(out_dev[g_], ref[g_]), f"poll={poll} batch {g_}"
    words, toks = asr.tokens_to_words(out[0])
    assert len(words) == B and all(len(t) == S for t in toks)
    # early exit: an EOS bias makes every row end at step 0..2; the reference loop breaks right after the last first-EOS
    p = torch.tensor([[5, 2, 2, 2], [2, 2, 2, 2], [7, 8, 2, 2]], dtype=torch.int32)
    assert greedy_exit_step(p, 2) == 3 and greedy_exit_step(p[:, :2], 2) == 2


def test_encoder_asr_ctc_greedy(dev):
    """EncoderASR (inference/ASR.py:176-389) with the CTC head + ctc_greedy_decode (decoders/ctc.py:335-378) vs the reference
    on the 2 s golden: log-posteriors within 2e-2, per-frame arg-max identical wherever the reference's top-1/top-2 margin
    exceeds 5e-3, and -- with the near-tie frames taken from the reference -- identical token lists (merge + blank filter)."""
    import functools

    from speechbrain_b200.decoders.ctc import ctc_greedy_decode
    from speechbrain_b200.inference.ASR import EncoderASR
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gc = torch.load(os.path.join(GOLDEN, "ctc_greedy_conformer_large_rope.pt"))
    cfg = _cfg(g)
    m = build_mirror(cfg, seeded(cfg))
    for name in ("plain", "merge"):
        c = gc[name]
        enc = m.front_end(m.head("ctc_lin", {0: c["bias_blank"], 17: c["bias_tok"]}))
        asr = EncoderASR(modules=dict(encoder=enc), hparams=dict(tokenizer=None, decoding_function=functools.partial(ctc_greedy_decode, blank_id=0)),
                         run_opts={"device": str(dev)})
        lp = asr.encode_batch(g["wav"], g["wav_lens"]).cpu()
        assert lp.shape[:2] == g["enc_out"].shape[:2] and lp.shape[2] == 5000
        words, toks = asr.transcribe_batch(g["wav"], g["wav_lens"])
        print(f"EncoderASR[{name}] tokens {toks} ref {c['hyps']}")
        check_ctc_argmax(f"EncoderASR[{name}]", lp, c["log_probs_head"], c["argmax"], c["margin"], g["wav_lens"], 0, c["hyps"])
        # module-by-module use of the mirror function on a CUDA tensor of log-probs
        assert ctc_greedy_decode(lp.to(dev), g["wav_lens"], blank_id=0) == toks


def test_fp16_range_scaled_weights(dev):
    """fp16 operand range (VERDICT r1 #8), against the reference re-run on the 2 s golden with scaled weights:
    (a) FFN first layers x200, second layers / 200 (hidden activations -- the fp16-stored tensor -- in the hundreds, FFN output
        scale unchanged): still <= 1e-3 rel-L2 -- fp16 rounding is relative and the residual stream / LayerNorm statistics are
        fp32.  (x200 alone makes every FFN output dwarf the residual stream, i.e. a 24-deep NON-residual chain in which any
        rounding compounds: 2.0e-3 measured, 1.95e-3 with the exact-form SiLU -- a property of that construction, not of the
        number format);
    (b) attention in_proj x3 (logits x9, near one-hot softmax) and conv pw1 x4: the rounding of q and k (2^-11 relative)
        becomes an ABSOLUTE logit error 9x larger, so the attention branch is as accurate as fp16 (or TF32 / bf16) operands
        allow: bar 3e-3 here, printed beside the result;
    (c) FFN first layers x1e5: the FFN hidden exceeds the fp16 maximum (65504): the fp32 -> fp16 stores saturate
        (F2FP.SATFINITE), so the output stays finite (no inf -> NaN cascade)."""
    from oracle.make_goldens import scale_state
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    gs = torch.load(os.path.join(GOLDEN, "conformer_large_rope_scaled.pt"))
    cfg = _cfg(g)
    sd = seeded_asr_state(cfg, 0)
    cnn = g["cnn_out"].reshape(g["cnn_out"].shape[0], g["cnn_out"].shape[1], -1).to(dev)
    results = []
    for name, bar in (("ffn", 1e-3), ("attn", 3e-3)):
        eng = AsrEngine(cfg, scale_state(sd, gs[name]["scales"]), device=dev, parts=("encoder",))
        enc = eng.encode_from_cnn(cnn, g["wav_lens"].to(dev)).cpu()
        r = rel(enc, gs[name]["enc_out"])
        print(f"scaled weights [{name}] {gs[name]['scales']} (max |FFN pre-activation| {gs[name]['ffn_hidden_absmax']:.0f} in the "
              f"reference): encoder rel-L2 err {r:.3e} (bar {bar:g})")
        results.append((name, bool(torch.isfinite(enc).all()), r, bar))
    assert all(fin and r < bar for _, fin, r, bar in results), results
    eng2 = AsrEngine(cfg, scale_state(sd, dict(gs["ffn"]["scales"], ffn_w1=1e5, ffn_w2=1e-5)), device=dev, parts=("encoder",))
    enc2 = eng2.encode_from_cnn(cnn, g["wav_lens"].to(dev)).cpu()
    print(f"FFN x1e5 (hidden beyond the fp16 range): finite {bool(torch.isfinite(enc2).all())}, absmax {float(enc2.abs().max()):.2f}")
    assert torch.isfinite(enc2).all()


def test_conformer_small_decoder_greedy(dev):
    """conformer_small.yaml end to end (d_model 144, 4 heads of 36, 4 decoder layers): the decoder runs on the generic
    head-dim decode attention and the unfused-LayerNorm projections; greedy tokens / log-probs vs the reference golden."""
    g = torch.load(os.path.join(GOLDEN, "conformer_small_relpos.pt"))
    cfg = _cfg(g)
    eng, sd = _engine(cfg, dev)
    n_steps = g["greedy_logits"].shape[1]
    ref_lp = torch.log_softmax(g["greedy_logits"], -1)
    top2 = g["greedy_logits"].topk(2, -1).values
    margin = top2[..., 0] - top2[..., 1]
    ref_tok = g["greedy_logits"].argmax(-1)
    pred, score, lp, done = eng.greedy_from_enc(g["enc_out"].to(dev), g["wav_lens"].to(dev), n_steps, 1, 2, want_log_probs=True)
    pred, lp = pred.cpu(), lp.cpu()
    print(f"[conformer_small] greedy tokens {pred.tolist()} ref {g['hyps']}")
    check_greedy("conformer_small", pred, lp, ref_tok, margin, ref_lp, min_compared=1 / pred.shape[0])  # n_steps decisions
    # and the whole path from the waveform
    p2, _, enc, _ = eng.transcribe_greedy_dev(g["wav"].to(dev), g["wav_lens"].to(dev), n_steps, 1, 2, want_enc=True)
    assert rel(enc.cpu(), g["enc_out"]) < 1.5e-3


def test_dynamic_chunk_encode(dev):
    """TransformerASR.encode(src, wav_len, dynchunktrain_config=DynChunkTrainConfig(chunk, left)) -- chunked attention masks +
    Dynamic Chunk Convolution (the streaming-equivalent masked mode) -- vs the reference: RoPE and RelPos, finite and
    infinite left context, chunk sizes that do not divide T, ragged batch."""
    import bench
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    gd = torch.load(os.path.join(GOLDEN, "dynchunk_conformer_large.pt"))
    asrs = {}
    for key, c in gd.items():
        att = c["attention_type"]
        g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt" if att == "RoPEMHA" else "conformer_large_relpos.pt"))
        if att not in asrs:
            cfg = _cfg(g)
            asrs[att] = bench.build_product_asr(cfg, seeded_asr_state(cfg, 0), dev).transformer
        tr = asrs[att]
        src = g["cnn_out"].to(dev)
        enc = tr.encode(src, g["wav_lens"].to(dev), dynchunktrain_config=DynChunkTrainConfig(c["chunk_size"], c["left_context_size"])).cpu()
        r = rel(enc, c["enc_out"])
        full = tr.encode(src, g["wav_lens"].to(dev)).cpu()  # the engine is back in full-context mode afterwards
        print(f"[dynchunk {key}] encoder rel-L2 err {r:.3e}; full-context afterwards rel {rel(full, g['enc_out']):.3e}")
        assert r < 1e-3 and rel(full, g["enc_out"]) < 1e-3


def test_encode_streaming_equals_masked(dev):
    """encode_streaming(chunk, context) chunk by chunk == encode(full, dynchunktrain_config) (the reference's own streaming
    test, tests/unittests/test_conformer.py, asserts exactly this equivalence): finite left context with history trimming
    (a 3-layer model so that the stream is longer than the retained window) and infinite left context, a short last chunk."""
    import bench
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    for att, cs, lc, n_layers in (("RoPEMHA", 8, 1, 3), ("RelPosMHAXL", 6, None, 2)):
        cfg = dict(CONFORMER_LARGE, attention_type=att, num_encoder_layers=n_layers, num_decoder_layers=1)
        tr = bench.build_product_asr(cfg, seeded_asr_state(cfg, 0), dev).transformer
        gen = torch.Generator().manual_seed(5)
        T = 20 * cs + 3
        src = torch.randn(2, T, 640, generator=gen).to(dev)
        dc = DynChunkTrainConfig(cs, lc)
        full = tr.encode(src, None, dynchunktrain_config=dc)
        ctx = tr.make_streaming_context(dc)
        outs = [tr.encode_streaming(src[:, t:t + cs].contiguous(), ctx) for t in range(0, T, cs)]
        stream = torch.cat(outs, dim=1)
        r = rel(stream.cpu(), full.cpu())
        print(f"[streaming {att} chunk {cs} left {lc}] {len(outs)} chunks, retained history {ctx.history.shape[1]} of {T} frames, "
              f"rel diff vs masked {r:.2e}")
        assert stream.shape == full.shape and r < 3e-4  # same maths; the online-softmax key-block partition differs with the window
        if lc is not None:
            assert ctx.history.shape[1] < T


@pytest.mark.parametrize("B,L,lens,att", [(1, 16000, [1.0], "RoPEMHA"), (3, 12345, [1.0, 0.5, 0.21], "RelPosMHAXL"),
                                          (2, 1999, [1.0, 0.6], "RoPEMHA"), (5, 48000, [0.37, 1.0, 0.99, 0.5, 0.8], "RoPEMHA")])
def test_edge_shapes_vs_oracle(dev, B, L, lens, att):
    """Edge shapes through the fused wav -> ids pipeline vs the CPU oracle (pinned to the reference by the golden generator):
    a single utterance, sample counts that are not multiples of 4 (no TMA staging) or of the hop, very short audio (T = 4 encoder
    frames), batch sizes that are not powers of two, utterances padded to a fifth of the batch length."""
    from oracle import asr_oracle as O
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    cfg = dict(CONFORMER_LARGE, attention_type=att, num_encoder_layers=3, num_decoder_layers=2)
    sd = seeded_asr_state(cfg, 0)
    eng = AsrEngine(cfg, sd, device=dev)
    gen = torch.Generator().manual_seed(B * 1000 + L)
    wav = torch.randn(B, L, generator=gen)
    wl = torch.tensor(lens)
    for b in range(B):
        wav[b, int(round(lens[b] * L)):] = 0
    steps = 3
    pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), wl.to(dev), steps, 1, 2, want_enc=True)
    torch.cuda.synchronize()
    ocfg = dict(cfg, win_length=32)
    with torch.no_grad():
        feats = O.full_pipeline_features(wav, wl, sd, ocfg)
        ref = O.encode(feats, wl, sd, cfg, "Transformer.")
        T = ref.shape[1]
        out = O.greedy_search(ref, wl, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], 1, 2, 0.0, (steps + 0.5) / T,
                              "Transformer.", return_logits=True)
    r = rel(enc.cpu(), ref)
    logits = out[4]
    n = logits.shape[1]
    top2 = logits.topk(2, -1).values
    print(f"edge B={B} L={L} lens={lens} {att}: T={T} encoder rel-L2 {r:.3e}, steps {done}/{n}")
    assert enc.shape == ref.shape and torch.isfinite(enc).all() and r < 1e-3
    m = min(n, done)
    check_greedy(f"edge B={B} L={L}", pred.cpu()[:, :m], None, logits.argmax(-1)[:, :m], (top2[..., 0] - top2[..., 1])[:, :m])


def test_long_utterance_vs_oracle(dev):
    """Maximum-size direction, ragged, 2 Conformer layers, encoder vs the CPU oracle: RoPE at 2 x 40 s (T = 1001 encoder
    frames = 16 key blocks, 8 x the bench length); RelPosMHAXL at 2 x 48 s (T = 1201: past the 1036 frames at which a
    T-row shared-memory P table no longer fits)."""
    from oracle import asr_oracle as O
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    for att, L, frac, seed in (("RoPEMHA", 640000, 0.73, 40), ("RelPosMHAXL", 768000, 0.66, 48)):
        cfg = dict(CONFORMER_LARGE, attention_type=att, num_encoder_layers=2, num_decoder_layers=1)
        sd = seeded_asr_state(cfg, 0)
        eng = AsrEngine(cfg, sd, device=dev, parts=("fbank", "cnn", "encoder"))
        gen = torch.Generator().manual_seed(seed)
        wav = torch.randn(2, L, generator=gen)
        wl = torch.tensor([1.0, frac])
        wav[1, int(frac * L):] = 0
        enc = eng.encode_wav(wav.to(dev), wl.to(dev)).cpu()
        del eng
        with torch.no_grad():
            ref = O.encode(O.full_pipeline_features(wav, wl, sd, dict(cfg, win_length=32)), wl, sd, cfg, "Transformer.")
        r = rel(enc, ref)
        print(f"long utterance {att}: T={ref.shape[1]} encoder rel-L2 {r:.3e}")
        assert enc.shape == ref.shape and r < 1e-3, f"{att}: rel-L2 {r:.3e}"
