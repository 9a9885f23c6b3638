"""-m gpu tests of the Switchboard transformer.yaml recipe's device path, against tests/golden/switchboard.pt (written by
tools/make_switchboard_golden.py from the running reference) and the fp32 oracles:

- the recipe's TransformerLM (d_model 264, 12 heads of 22, d_embedding 128): the whole-sequence forward, the KV-cached step
  path position by position, lm_rescore against summed step log-probs, and reruns;
- its two attention kernels at the padded head width 32, alone, against float64 references: the causal flash kernel
  (lm_causal_attention) and the decode attention (dec_attention) in the step's cache layout;
- the ASR model (3-block front-end, 12 regularMHA layers of 4 heads of 64 at d_model 256): encoder states and greedy tokens;
- the recipe's test search (beam 60, TransformerLM 0.3 + CTC 0.3, temperature 1.0) and a from_hparams round trip.

Bars are tests/test_gpu_lm_forward.py's for the LM (rel-L2 <= 2e-3 per sequence, arg-max identical where the reference
margin is >= 5e-3) and tests/parity.py's for greedy and beam search.

test_lm_forward_reference_golden fails on the two padding mistakes the device path could make (worked out with the fp32
oracle on the fixture's batch).  A build that scaled the folded embedding table by sqrt(d_model), as for an LM without
embedding_proj, moves the logits by rel-L2 0.83: its arg-max assertion fails first (the logsumexp moves by only 0.017).  A
build whose LayerNorms took their statistics over the 272 padded channels instead of the 264 real ones moves them by 0.017:
the arg-max still agrees, and the sampled-row assertion (rel-L2 <= 2e-3 per row) fails."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import (BEAM_TOL, case_wav, check_alone_vs_batch, check_beam, check_encoder, check_greedy, check_summary,  # noqa: E402
                    dev, module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir)  # noqa: F401
import decoder_kernels_oracle as DK  # noqa: E402
import switchboard_oracle as SO  # noqa: E402
import transformer_oracle as TO  # noqa: E402
from mirrors import build_mirror, seeded  # noqa: E402

from oracle import asr_oracle as O  # noqa: E402
from speechbrain_b200.utils.seeded_init import SWITCHBOARD_LM, SWITCHBOARD_TRANSFORMER as CFG  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ENC_BAR = 1e-3
ATT_BAR = 3e-3
BOS, EOS = 1, 2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "switchboard.pt"))


@pytest.fixture(scope="module")
def sd(fx):
    return seeded(CFG, fx["weight_seed"])


def _lm(seed=1):
    from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    lm = TransformerLM(**SWITCHBOARD_LM, dropout=0.0, activation=torch.nn.ReLU)
    sd = seeded_state_dict(lm, seed=seed)
    lm.load_state_dict(sd)
    return lm, sd


@pytest.fixture(scope="module")
def lm(fx):
    return _lm(fx["lm"]["seed"])


def _batch(n, s, seed, interior_pad=0.2):
    """Ragged batch: bos = 1, ids in [3, 2000), padded with 0, the first row spanning all s positions; interior_pad: the
    share of positions after bos inside the valid lengths that hold id 0"""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, s + 1, (n,), generator=g)
    lens[0] = s
    tokens = torch.zeros(n, s, dtype=torch.long)
    for i, L in enumerate(lens.tolist()):
        tokens[i, 0] = 1
        tokens[i, 1:L] = torch.randint(3, 2000, (L - 1,), generator=g)
        if L > 1:
            tokens[i, 1:L][torch.rand(L - 1, generator=g) < interior_pad] = 0
    return tokens, lens


def _check_vs(logits, ref, what):
    """Per sequence on all its positions (pad positions too): rel-L2 <= 2e-3; arg-max identical where ref's top-1/top-2
    margin >= 5e-3."""
    logits, ref = logits.double().cpu(), ref.double().cpu()
    worst = 0.0
    for i in range(ref.shape[0]):
        a, b = logits[i], ref[i]
        worst = max(worst, float((a - b).norm() / b.norm()))
        top2 = b.topk(2, dim=-1).values
        sure = (top2[:, 0] - top2[:, 1]) >= 5e-3
        assert torch.equal(a.argmax(-1)[sure], b.argmax(-1)[sure]), f"{what}: arg-max differs in sequence {i}"
    print(f"MEASURE {what}: worst per-sequence rel-L2 {worst:.2e} (bar 2e-3)")
    assert worst <= 2e-3, what


# ------------------------------------------------------------------------------------------------ the LM
def test_lm_forward_reference_golden(dev, fx, lm):
    model, sd_lm = lm
    g = fx["lm"]
    tokens = g["tokens"]
    logits = model(tokens.to(dev)).cpu()
    assert logits.shape == (tokens.shape[0], tokens.shape[1], 2000) and torch.isfinite(logits).all()
    assert (logits.logsumexp(-1) - g["logsumexp"]).abs().max() < 5e-2
    top_v, top_i = logits.topk(8, dim=-1)
    sure = (g["top_values"][..., 0] - g["top_values"][..., 1]) >= 5e-3
    assert torch.equal(top_i[..., 0][sure], g["top_ids"][..., 0][sure].long())
    idx = g["sample_idx"].long()
    sample = logits[idx[:, 0], idx[:, 1]].double()
    for k in range(idx.shape[0]):
        ref = g["sample_logits"][k].double()
        assert float((sample[k] - ref).norm() / ref.norm()) <= 2e-3, tuple(idx[k].tolist())
    with torch.no_grad():
        oracle = SO.lm_forward(tokens, sd_lm)
    _check_vs(logits, oracle, "switchboard LM golden batch vs oracle")


@pytest.mark.parametrize("n,s,seed", [(4, 1, 11), (3, 70, 12), (2, 300, 13), (64, 80, 15)])
def test_lm_forward_vs_oracle(dev, lm, n, s, seed):
    """s = 1, s across the 64-key attention blocks, five key blocks, and n = 64 at s = 80 (the timed shape)"""
    model, sd_lm = lm
    tokens, _ = _batch(n, s, seed)
    logits = model(tokens.to(dev))
    assert torch.isfinite(logits).all()
    with torch.no_grad():
        ref = SO.lm_forward(tokens, sd_lm)
    _check_vs(logits, ref, f"switchboard LM n={n} s={s}")


@pytest.mark.parametrize("n,s,seed", [(5, 70, 41), (64, 24, 42)])  # 64 rows: the step's projections on the wgmma GEMM
def test_lm_step_path_position_by_position(dev, lm, n, s, seed):
    """The KV-cached step (the beam search's LM scorer) gives forward's logits at every position, with id 0 inside the
    valid lengths and as trailing padding"""
    model, _ = lm
    td = _batch(n, s, seed)[0].to(dev)
    fwd = model(td)
    step = model._get_engine(dev).lm_step_logits(td)
    assert torch.isfinite(step).all()
    _check_vs(fwd, step, f"switchboard LM forward vs step path n={n} s={s}")


def test_lm_rescore_equals_summed_step_log_probs(dev, lm):
    """lm_rescore = sum over positions of log_softmax(step logits) at the next token, pad column excluded from the
    normalisation (the rescorer's rule), within 1e-3 per sequence"""
    model, _ = lm
    tokens, lens = _batch(12, 40, 21, interior_pad=0.0)
    td = tokens.to(dev)
    eng = model._get_engine(dev)
    lp = torch.log_softmax(eng.lm_step_logits(td).double(), dim=-1)
    lp[:, :, 0] = float("-inf")
    tgt = lp[:, :-1].gather(2, td[:, 1:].unsqueeze(2)).squeeze(2) - lp[:, :-1].logsumexp(-1)
    mask = (torch.arange(tokens.shape[1], device=dev).unsqueeze(0) < lens.to(dev).unsqueeze(1))[:, 1:]
    ours = torch.nansum(tgt * mask, dim=-1).cpu()
    got = eng.lm_rescore(td, lens, 1.0, 0).double().cpu()
    print(f"MEASURE switchboard lm_rescore vs summed step log-probs: max |d| {(ours - got).abs().max():.2e}")
    assert (ours - got).abs().max() < 1e-3


def test_lm_reruns_bit_identical(dev, fx, lm):
    model, _ = lm
    td = fx["lm"]["tokens"].to(dev)
    eng = model._get_engine(dev)
    assert torch.equal(model(td), model(td))
    assert torch.equal(eng.lm_step_logits(td), eng.lm_step_logits(td))


# ------------------------------------------------------------------------------------------------ kernels at width 32
def _padded_heads(x, dh, dhp):
    """[..., H, dh] -> [..., H, dhp] with zero padding"""
    return torch.nn.functional.pad(x, (0, dhp - dh))


@pytest.mark.parametrize("n,s", [(1, 1), (3, 70), (2, 200)])
def test_causal_attention_kernel_width_32_vs_fp64(dev, n, s):
    """lm_causal_attention at 12 heads of 32 holding 22 real dims: out equals the float64 attention over the 22 real dims
    (look-ahead mask, key-padding mask on id 0, NaN for a query without a visible key), and the padded output dims are 0"""
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    H, dh, dhp = 12, 22, 32
    g = torch.Generator().manual_seed(100 + s)
    q, k, v = (torch.randn(n, s, H, dh, generator=g) for _ in range(3))
    q = q / dh ** 0.5 * 3.0
    tokens, _ = _batch(n, s, 200 + s, interior_pad=0.2)
    if n > 1:
        tokens[1, 0] = 0  # a sequence starting with the pad id: its first query sees no key
    qkv = torch.cat([_padded_heads(x, dh, dhp).reshape(n * s, H * dhp) for x in (q, k, v)], dim=1)
    qkv16 = qkv.half()
    out = torch.full((n * s, H * dhp), float("nan"), dtype=torch.float16, device=dev)
    qkv_d, td = qkv16.to(dev), tokens.to(torch.int32).to(dev)  # held until the call returns
    rc = lib().sbk_lm_causal_attention_test(ptr(qkv_d), n, s, H * dhp, H, ptr(td), 0, ptr(out), stream_ptr(dev))
    assert rc == 0
    qd, kd, vd = (x.reshape(n, s, H, dhp)[..., :dh].double() for x in qkv16.float().split(H * dhp, dim=1))
    sc = torch.einsum("bihd,bjhd->bhij", qd, kd)
    mask = torch.triu(torch.ones(s, s, dtype=torch.bool), 1).view(1, 1, s, s) | (tokens == 0).view(n, 1, 1, s)
    sc = sc.masked_fill(mask, float("-inf"))
    ref = torch.einsum("bhij,bjhd->bihd", torch.softmax(sc, dim=-1), vd)
    o = out.double().cpu().view(n, s, H, dhp)
    nan_ref = torch.isnan(ref)
    assert torch.equal(torch.isnan(o[..., :dh]), nan_ref)
    ok = ~nan_ref
    err = rel(o[..., :dh][ok], ref[ok])
    print(f"MEASURE lm_causal_attention dh 32 (22 real) n={n} s={s}: rel-L2 {err:.2e} (bar {ATT_BAR})")
    assert err <= ATT_BAR
    assert (o[..., dh:][~nan_ref.any(-1, keepdim=True).expand(-1, -1, -1, dhp - dh)] == 0).all()


@pytest.mark.parametrize("step", [0, 31, 77])
def test_lm_decode_attention_width_32_vs_fp64(dev, step):
    """The LM step's self-attention (dec_attention) in its cache layout: 12 heads of 32 (22 real) side by side in a
    384-wide key row, a lineage table and the pad-id mask, against the float64 attention over the 22 real dims"""
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    R, H, dh, dhp, S = 6, 12, 22, 32, 96
    g = torch.Generator().manual_seed(300 + step)
    q = _padded_heads(torch.randn(R, H, dh, generator=g) * (3.0 / dh ** 0.5), dh, dhp).half()
    kc = _padded_heads(torch.randn(R, S, H, dh, generator=g), dh, dhp).half()
    vc = _padded_heads(torch.randn(R, S, H, dh, generator=g), dh, dhp).half()
    lin = torch.randint(0, R, (2, R, S), generator=g, dtype=torch.int32)
    tok = torch.randint(1, 50, (R, S), generator=g, dtype=torch.int32)
    tok[1, step // 2] = 0
    tok[2, 0] = 0
    out = torch.full((R, H * dhp), float("nan"), dtype=torch.float16, device=dev)
    d = H * dhp
    qd, kd, vd, lind, tokd = (x.to(dev) for x in (q.view(R, d), kc, vc, lin, tok))  # held until the call returns
    rc = lib().sbk_dec_attention_test(ptr(qd), d, ptr(kd), ptr(vd), ctypes.c_longlong(S * d), d, 0, 1, R, H, dhp, S, step,
                                      None, ptr(lind), ptr(tokd), S, 0, ptr(out), d, stream_ptr(dev))
    assert rc == 0
    ref = DK.dec_attention_ref(q[..., :dh], kc[..., :dh], vc[..., :dh], step + 1, lineage=lin[step & 1], tok=tok)
    o = out.double().cpu().view(R, H, dhp)
    ok = ~torch.isnan(ref).view(R, -1).any(-1)
    assert torch.equal(torch.isnan(o[..., :dh]), torch.isnan(ref))
    err = rel(o[ok][..., :dh], ref[ok])
    print(f"MEASURE LM decode attention dh 32 (22 real) step={step}: rel-L2 {err:.2e} (bar {ATT_BAR})")
    assert err <= ATT_BAR and (o[ok][..., dh:] == 0).all()


# ------------------------------------------------------------------------------------------------ the ASR model
def test_encoder_and_greedy(dev, fx, sd):
    """The 3-block front-end at d_model 256 and the 12 regularMHA layers, then 48 greedy steps"""
    from speechbrain_b200.engine import AsrEngine
    g = fx["asr"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        ref = TO.encode(TO.wav_to_cnn(wav, lens, sd, CFG), lens, sd, CFG)
    check_summary("switchboard oracle", ref, g["enc"]["frame_norm"], g["enc"]["sample_idx"], g["enc"]["sample_rows"], 1e-5)
    eng = AsrEngine(CFG, sd, device=dev)
    S = g["greedy_tokens"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), lens.to(dev), S, BOS, EOS, want_enc=True)
    torch.cuda.synchronize()
    check_encoder("switchboard", enc.cpu(), ref, g["abs_len"], ENC_BAR)
    check_greedy("switchboard", pred.cpu(), None, g["greedy_tokens"], g["greedy_margin"], chosen_lp=None)
    check_alone_vs_batch(lambda w, ln: eng.encode_wav(w.to(dev), ln.to(dev)), wav, lens, 1e-5)


def _searcher(m, model, beam, max_decode_ratio):
    """the recipe's test search: [TransformerLM 0.3, CTC 0.3], temperature 1.0, no EOS threshold, length normalisation"""
    kwargs = dict(min_decode_ratio=0.0, beam_size=beam, temperature=1.0, using_eos_threshold=False, eos_threshold=1.5,
                  length_normalization=True)
    return m.searcher(kwargs, max_decode_ratio, scorers=dict(transformerlm=0.3, ctc=0.3), lm=model, lm_temperature=1.0,
                      scorer_beam_scale=0.3)


def test_beam60_lm_ctc_matches_reference(dev, fx, sd, lm):
    """The recipe's beam-60 search (240 live hypotheses: the LM step at 240 rows on the wgmma projections) for 16 steps on
    the oracle's encoder states: parity.check_beam against the reference; a rerun is bit-identical"""
    model, sd_lm = lm
    g, gb = fx["asr"], fx["beam60"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        enc = TO.encode(TO.wav_to_cnn(wav, lens, sd, CFG), lens, sd, CFG)
    bs = _searcher(build_mirror(CFG, sd), model, gb["kwargs"]["beam_size"], gb["max_decode_ratio"])
    hyps, _, scores, _ = bs(enc.to(dev), lens.to(dev))
    h2, _, s2, _ = bs(enc.to(dev), lens.to(dev))
    assert h2 == hyps and torch.equal(s2, scores), "rerun differs"
    olm = dict(sd=SO.plain_state(sd_lm), cfg=SO.CFG, weight=gb["lm_weight"], temperature=gb["lm_temperature"])
    octc = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=gb["ctc_weight"], blank_index=0)

    def forced(idx, tokens):
        return O.beam_search(enc[idx], lens[idx], sd, CFG, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], BOS, EOS,
                             beam_size=1, temperature=1.0, using_eos_threshold=False, length_normalization=True,
                             prefix="Transformer.", lm=olm, ctc=octc, forced=tokens)

    check_beam("switchboard beam60 lm+ctc", [list(h) + [EOS] for h in hyps], scores.cpu().view(-1, 1),
               [list(h) + [EOS] for h in gb["hyps"]], gb["scores"].view(-1, 1), forced)


HPARAMS = """
d_model: 256
output_neurons: 2000
bos_index: 1
eos_index: 2
blank_index: 0
normalizer: !new:speechbrain.processing.features.InputNormalization
    norm_type: global
compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: 16000
    n_fft: 400
    n_mels: 80
CNN: !new:speechbrain.lobes.models.convolution.ConvolutionFrontEnd
    input_shape: (8, 10, 80)
    num_blocks: 3
    num_layers_per_block: 1
    out_channels: (64, 64, 64)
    kernel_sizes: (5, 5, 1)
    strides: (2, 2, 1)
    residuals: (False, False, True)
Transformer: !new:speechbrain.lobes.models.transformer.TransformerASR.TransformerASR
    input_size: 1280
    tgt_vocab: !ref <output_neurons>
    d_model: !ref <d_model>
    nhead: 4
    num_encoder_layers: 12
    num_decoder_layers: 6
    d_ffn: 2048
    dropout: 0.1
    activation: !name:torch.nn.GELU
    encoder_module: transformer
    attention_type: regularMHA
    normalize_before: True
    causal: False
ctc_lin: !new:speechbrain.nnet.linear.Linear
    input_size: !ref <d_model>
    n_neurons: !ref <output_neurons>
seq_lin: !new:speechbrain.nnet.linear.Linear
    input_size: !ref <d_model>
    n_neurons: !ref <output_neurons>
lm_model: !new:speechbrain.lobes.models.transformer.TransformerLM.TransformerLM
    vocab: !ref <output_neurons>
    d_model: 264
    d_embedding: 128
    nhead: 12
    num_encoder_layers: 12
    num_decoder_layers: 0
    d_ffn: 1024
    dropout: 0.0
    activation: !name:torch.nn.ReLU
    normalize_before: False
transformerlm_scorer: !new:speechbrain.decoders.scorer.TransformerLMScorer
    language_model: !ref <lm_model>
    temperature: 1.0
ctc_scorer: !new:speechbrain.decoders.scorer.CTCScorer
    eos_index: !ref <eos_index>
    blank_index: !ref <blank_index>
    ctc_fc: !ref <ctc_lin>
scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <transformerlm_scorer>, !ref <ctc_scorer>]
    weights:
        transformerlm: 0.3
        ctc: 0.3
    scorer_beam_scale: 0.3
decoder: !new:speechbrain.decoders.S2STransformerBeamSearcher
    modules: [!ref <Transformer>, !ref <seq_lin>]
    bos_index: !ref <bos_index>
    eos_index: !ref <eos_index>
    min_decode_ratio: 0.0
    max_decode_ratio: 0.05
    beam_size: 60
    using_eos_threshold: False
    eos_threshold: 1.5
    temperature: 1.0
    length_normalization: True
    scorer: !ref <scorer>
Tencoder: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
    transformer: !ref <Transformer>
encoder: !new:speechbrain.nnet.containers.LengthsCapableSequential
    input_shape: [null, null, 80]
    compute_features: !ref <compute_features>
    normalize: !ref <normalizer>
    cnn: !ref <CNN>
    transformer_encoder: !ref <Tencoder>
tokenizer: null
asr_model: !new:torch.nn.ModuleList
    - [!ref <CNN>, !ref <Transformer>, !ref <seq_lin>, !ref <ctc_lin>]
modules:
    normalizer: !ref <normalizer>
    encoder: !ref <encoder>
    decoder: !ref <decoder>
    lm_model: !ref <lm_model>
pretrainer: !new:speechbrain.utils.parameter_transfer.Pretrainer
    loadables:
        normalizer: !ref <normalizer>
        asr: !ref <asr_model>
        lm: !ref <lm_model>
    paths:
        asr: <save_dir>/asr.ckpt
        lm: <save_dir>/lm.ckpt
"""


def test_from_hparams_recipe_layout(dev, fx, sd, lm, tmp_path):
    """A pretrained-model directory in transformer.yaml's layout (3-block CNN, Transformer, ctc_lin, seq_lin, the
    d_embedding TransformerLM, ScorerBuilder with scorer_beam_scale) loads through from_hparams into the mirrors and
    transcribes like the same modules wired directly"""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
    model, sd_lm = lm
    tmp = write_pretrained_dir(tmp_path, HPARAMS, dict(asr=module_list_ckpt(sd), lm=sd_lm, normalizer=normalizer_ckpt(sd)))
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": str(dev)})
    dec = loaded.mods["decoder"]
    assert isinstance(dec.lm_scorer.lm, TransformerLM) and dec.lm_scorer.lm.d_embedding == 128
    assert torch.equal(dec.lm_scorer.lm.embedding_proj.w.weight.cpu(), sd_lm["embedding_proj.w.weight"])
    assert (dec.lm_weight, dec.ctc_weight, dec.beam_size) == (0.3, 0.3, 60)
    m = build_mirror(CFG, sd)
    direct = EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=_searcher(m, model, 60, 0.05)),
                               hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})
    wav, lens = case_wav(fx["asr"])
    _, t1 = loaded.transcribe_batch(wav, lens)
    _, t2 = direct.transcribe_batch(wav, lens)
    print("from_hparams tokens", t1)
    assert t1 == t2 and len(t1) == 4 and sum(len(t) for t in t1) > 0
