"""-m gpu tests of the Loquacious Conformers (conformer_activation=torch.nn.GELU, RelPosMHAXL at head width 64; d_model 256,
512, 768 and 1024 with 4, 8, 12 and 16 heads; GELU decoders over 1024 or 5120 tokens; blank 3, bos 1, eos 2).

Kernel level: the depthwise conv + LayerNorm + GELU of the convolution module through sbk_dwconv_act_test against a float64
reference, on every instantiation the launcher picks (K = 31 with 1, 2 or 4 channels per thread, runtime K, chunked).

Model level, on seeded weights (utils/seeded_init.LOQUACIOUS_*), against the reference outputs in tests/golden/loquacious.pt
(generator: tools/make_loquacious_golden.py) and the fp32 CPU oracle of loquacious_oracle.py recomputed here (it equals the
reference to 1e-5 on every fixture entry, test_loquacious_golden.py): encoder states of every fixture case at the
Conformer's 1e-3 bar, 48 greedy steps and the recipe's beam 80 + CTC 0.3 search on the full-depth xlarge, batch invariance
and bit-identical reruns, and streaming against the masked Dynamic Chunk mode."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import loquacious_oracle as LO  # noqa: E402
from parity import (BEAM_TOL, check_alone_vs_batch, check_beam, check_encoder, check_greedy, check_summary,  # noqa: E402,F401
                    dev, module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir)

ENC_BAR = 1e-3
DW_BAR = 9e-4  # the Swish kernel's bar in test_gpu_encoder_kernels.py
BOS, EOS, BLANK = LO.BOS, LO.EOS, LO.BLANK
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loquacious.pt")

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ depthwise conv + GELU
def _dwconv_ref(x, taps, bias, ln_g, ln_b, chunk, eps=1e-5):
    """float64 GELU(LayerNorm(Conv1d_K(x) + bias)), zero padding outside [0, T); chunk > 0: inputs at or past the end of the
    output frame's chunk count as zero"""
    import torch.nn.functional as F
    B, T, D = x.shape
    K = taps.shape[-1]
    pad = (K - 1) // 2
    x, taps, bias = x.double(), taps.double(), bias.double()
    t = torch.arange(T, device=x.device)
    end = (t // chunk + 1) * chunk if chunk > 0 else torch.full_like(t, T + pad)
    xp = F.pad(x, (0, 0, pad, pad))
    h = bias.view(1, 1, D).expand(B, T, D).clone()
    for k in range(K):
        ok = (t + k - pad < end).view(1, T, 1)
        h = h + torch.where(ok, xp[:, k:k + T], torch.zeros((), dtype=x.dtype, device=x.device)) * taps[:, 0, k]
    return F.gelu(F.layer_norm(h, (D,), ln_g.double(), ln_b.double(), eps))


def _dwconv_dev(x, taps, bias, ln_g, ln_b, chunk, act):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    B, T, D = x.shape
    out = torch.full((B, T, D), float("nan"), dtype=torch.float16, device=x.device)
    check(lib().sbk_dwconv_act_test(ptr(x), B, T, D, taps.shape[-1], ptr(taps), ptr(bias), ptr(ln_g), ptr(ln_b), chunk, act,
                                    ptr(out), stream_ptr(x.device)), "sbk_dwconv_act_test")
    return out


@pytest.mark.parametrize("chunk", [0, 16])
@pytest.mark.parametrize("T", [1, 16, 17, 251])
@pytest.mark.parametrize("K", [31, 15])
@pytest.mark.parametrize("D", [256, 512, 768, 1024])
def test_dwconv_gelu_kernel(dev, D, K, T, chunk):
    """GELU after the LayerNorm on a ragged B = 3 batch (padded frames hold other values: they are inputs); a rerun is
    bit-identical and act 0 equals sbk_dwconv_test (Swish)"""
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    g = torch.Generator().manual_seed(D * 7 + K * 1009 + T + chunk)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    x = r(3, T, D)
    for b, frac in enumerate((1.0, 0.7, 0.4)):
        n = max(1, int(frac * T))
        x[b, n:] = 0.25 * r(T - n, D) - 0.1
    taps = r(D, 1, K) * (1.4 / K ** 0.5)
    bias, ln_g, ln_b = 0.1 * r(D), 1.0 + 0.1 * r(D), 0.05 * r(D)
    x, taps, bias, ln_g, ln_b = [t.to(dev).contiguous() for t in (x, taps, bias, ln_g, ln_b)]
    out = _dwconv_dev(x, taps, bias, ln_g, ln_b, chunk, 1)
    ref = _dwconv_ref(x, taps, bias, ln_g, ln_b, chunk)
    o = out.double()
    err = float(((o - ref).abs() / (ref.abs() + ref.pow(2).mean().sqrt())).max())
    print(f"MEASURE dwconv GELU D={D} K={K} T={T} chunk={chunk}: max |d|/(|ref|+rms) {err:.3e} (bar {DW_BAR})")
    assert torch.isfinite(o).all() and err <= DW_BAR
    assert torch.equal(out, _dwconv_dev(x, taps, bias, ln_g, ln_b, chunk, 1)), "rerun differs"
    swish = torch.empty_like(out)
    check(lib().sbk_dwconv_test(ptr(x), 3, T, D, K, ptr(taps), ptr(bias), ptr(ln_g), ptr(ln_b), chunk, ptr(swish),
                                stream_ptr(dev)), "sbk_dwconv_test")
    assert torch.equal(_dwconv_dev(x, taps, bias, ln_g, ln_b, chunk, 0), swish)


def test_dwconv_act_rejects_unknown(dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    x = torch.zeros(16, 256, device=dev)
    taps = torch.zeros(256, 1, 31, device=dev)
    v = torch.ones(256, device=dev)
    out = torch.zeros(16, 256, dtype=torch.float16, device=dev)
    assert lib().sbk_dwconv_act_test(ptr(x), 1, 16, 256, 31, ptr(taps), ptr(v), ptr(v), ptr(v), 0, 2, ptr(out),
                                     stream_ptr(dev)) != 0


def test_dwconv_gelu_is_the_erf_form(dev):
    """with LayerNorm gain 0 every output is act(ln_b[c]) exactly, so the kernel's activation is read directly: at
    pre-activations in [-3, 3] (where the erf and tanh forms of GELU differ by up to 4e-4, tens of fp16 ulps below -1.5)
    the GELU output is the fp16 rounding of the erf form within 1 ulp and is not the tanh form's; act 0 is SiLU"""
    import torch.nn.functional as F
    D, T = 256, 16
    pre = torch.linspace(-3.0, 3.0, D, dtype=torch.float64)
    x = torch.randn(1, T, D, generator=torch.Generator().manual_seed(1)).to(dev)
    taps = torch.zeros(D, 1, 31, device=dev)
    bias, ln_g, ln_b = torch.zeros(D, device=dev), torch.zeros(D, device=dev), pre.float().to(dev)
    for act, fn in ((1, F.gelu), (0, F.silu)):
        out = _dwconv_dev(x, taps, bias, ln_g, ln_b, 0, act)[0].cpu().double()
        want = fn(pre.float().double())
        ulp = (want.abs().clamp_min(6.1e-5).log2().floor() - 10).exp2()  # fp16 spacing at |want|
        assert ((out - want).abs() <= ulp).all(), (act, float(((out - want).abs() / ulp).max()))
    tanh_form = F.gelu(pre, approximate="tanh")
    gelu_out = _dwconv_dev(x, taps, bias, ln_g, ln_b, 0, 1)[0, 0].cpu().double()
    far = pre < -1.5
    assert ((gelu_out[far] - tanh_form[far]).abs() > 4 * (tanh_form[far].abs().log2().floor() - 10).exp2()).any()


def test_create_rejects_unknown_activation(dev):
    """sbk_asr_create refuses a conformer_activation other than 0 (Swish) and 1 (GELU), and GELU outside the Conformer"""
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC, seeded_asr_state
    cfg = LO.reduced(LO.sizes()["loquacious_small"])
    sd = LO.state(cfg)
    with pytest.raises(NotImplementedError):
        AsrEngine(dict(cfg, conformer_activation="tanh_gelu"), sd, device=str(dev))
    bf = dict(BRANCHFORMER_CTC, num_encoder_layers=1, conformer_activation="gelu")
    with pytest.raises(RuntimeError, match="Conformer encoder only"):
        AsrEngine(bf, seeded_asr_state(bf, 0), device=str(dev), parts=("fbank", "cnn", "encoder"))


# ------------------------------------------------------------------------------------------------ model level
@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN)


@pytest.fixture(scope="module")
def wav():
    return LO.waveforms()


def _engine(cfg, dev):
    from speechbrain_b200.engine import AsrEngine
    return AsrEngine(dict(cfg, conformer_activation="gelu"), LO.state(cfg), device=str(dev))


def _enc_case(tag, cfg, rec, wav, dev, dynchunk=None):
    """wav -> encoder states on the device (AsrEngine; with dynchunk the masked Dynamic Chunk mode) against the fixture's
    summary and the oracle"""
    w, lens = wav
    eng = _engine(cfg, dev)
    if dynchunk is not None:
        eng.set_dynchunk(*dynchunk)
    enc = eng.encode_wav(w.to(dev), lens.to(dev)).cpu()
    T = enc.shape[1]
    s = rec["enc"]
    check_summary(f"{tag} encoder", enc, s["frame_norm"], s["sample_idx"], s["sample_rows"], ENC_BAR)
    check_encoder(tag, enc, LO.encode(cfg, LO.state(cfg), w, lens, dynchunk), [round(float(x) * T) for x in lens], ENC_BAR)
    return eng


@pytest.mark.parametrize("name", ["loquacious_small", "loquacious_base", "loquacious_large", "loquacious_xlarge"])
def test_encoder_reduced(dev, fx, wav, name):
    _enc_case(name, LO.reduced(LO.sizes()[name]), fx["reduced"][name], wav, dev)


def test_encoder_dynchunk(dev, fx, wav):
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_LARGE
    _enc_case("large dynchunk", LO.reduced(LOQUACIOUS_LARGE), fx["dynchunk"], wav, dev, tuple(fx["dynchunk"]["chunk"]))


def test_encoder_rope(dev, fx, wav):
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_SMALL
    _enc_case("small rope", LO.reduced(LOQUACIOUS_SMALL, attention_type="RoPEMHA"), fx["rope"], wav, dev)


@pytest.fixture(scope="module")
def xlarge(fx, wav):
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_XLARGE
    w, lens = wav
    return dict(cfg=LOQUACIOUS_XLARGE, enc=LO.encode(LOQUACIOUS_XLARGE, LO.state(LOQUACIOUS_XLARGE), w, lens), fx=fx)


def test_xlarge_encoder_and_greedy(dev, xlarge, wav):
    """the full 18 + 6 layer xlarge: wav -> encoder states against the fixture and the oracle, 48 greedy steps against the
    reference's; a rerun is bit-identical and the first utterance alone equals its rows in the batch"""
    cfg, g = xlarge["cfg"], xlarge["fx"]["xlarge"]
    eng = _engine(cfg, dev)
    w, lens = wav[0].to(dev), wav[1].to(dev)

    def greedy(x, ln):
        pred, score, enc, _ = eng.transcribe_greedy_dev(x, ln, LO.STEPS, BOS, EOS, want_enc=True)
        return enc, pred, score
    enc, pred, score = greedy(w, lens)
    torch.cuda.synchronize()
    enc = enc.cpu()
    T = enc.shape[1]
    s = g["enc"]
    check_summary("xlarge encoder", enc, s["frame_norm"], s["sample_idx"], s["sample_rows"], ENC_BAR)
    check_encoder("xlarge", enc, xlarge["enc"], [round(float(x) * T) for x in wav[1]], ENC_BAR)
    check_greedy("xlarge", pred.cpu(), score.cpu(), g["greedy_tokens"], g["greedy_margin"], g["greedy_chosen_lp"], stop_at=EOS)
    check_alone_vs_batch(greedy, w, lens, 1e-5, relative=True)


@pytest.mark.parametrize("which", ["beam", "beam_eos"])
def test_xlarge_beam80_ctc(dev, xlarge, wav, which):
    """the recipe's test search (beam 80, CTC 0.3 with blank 3, temperature 1.15, using_eos_threshold) on the oracle's
    encoder states of the fixture case's utterances against the reference fixture (parity.check_beam); a rerun is
    identical.  "beam": the full xlarge on utterances 0 and 3 with the seeded weights as they are; "beam_eos": the reduced
    xlarge on all four utterances with seq_lin's EOS bias raised, where the best hypotheses differ between utterances"""
    gb = xlarge["fx"][which]
    utts = gb["utts"]
    if which == "beam":
        cfg, enc = xlarge["cfg"], xlarge["enc"][utts]
    else:
        cfg = LO.reduced(xlarge["cfg"])
        enc = LO.encode(cfg, LO.state(cfg), wav[0], wav[1])[utts]
        assert len({tuple(h) for h in gb["hyps"]}) > 1
    sd = dict(LO.state(cfg))
    lens = wav[1][utts]
    _, lin, _, bs = LO.search_modules(cfg, (gb["steps"] + 0.5) / enc.shape[1], gb)
    with torch.no_grad():
        lin.w.bias[EOS] += gb["eos_bias"]
    sd["seq_lin.w.bias"] = lin.w.bias.detach().clone()
    hyps, _, scores, _ = bs(enc.to(dev), lens.to(dev))
    scores = scores.cpu().view(-1, 1)
    h2, _, s2, _ = bs(enc.to(dev), lens.to(dev))
    assert h2 == hyps and torch.equal(s2.cpu().view(-1, 1), scores), "rerun differs"
    check_beam(f"xlarge {which} {gb['beam']}", [list(h) + [EOS] for h in hyps], scores,
               [list(h) + [EOS] for h in gb["hyps"]], gb["scores"].view(-1, 1),
               lambda idx, tokens: LO.beam(cfg, sd, enc[idx], lens[idx], dict(gb, beam=1), forced=tokens))


def test_gelu_engine_differs_from_swish(dev, wav):
    """the engine built from engine_cfg() follows conformer_activation: the same weights as a Swish model give other
    encoder states"""
    cfg = LO.reduced(LO.sizes()["loquacious_base"])
    tr = LO.mirror(cfg)
    src = torch.randn(2, 60, 640, generator=torch.Generator().manual_seed(5)).to(dev)
    gelu = tr.encode(src).cpu()
    tr.conformer_activation = "swish"
    tr.invalidate_engines()
    swish = tr.encode(src).cpu()
    assert rel(swish, gelu) > 1e-2


@pytest.mark.parametrize("att,cs,lc", [("RelPosMHAXL", 16, 2), ("RoPEMHA", 8, None)])
def test_streaming_equals_masked(dev, att, cs, lc):
    """encode_streaming with GELU equals the masked Dynamic Chunk mode, as test_gpu_streaming.py checks for Swish"""
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = LO.mirror(dict(LO.sizes()["loquacious_large"], num_encoder_layers=3, num_decoder_layers=1, attention_type=att))
    B, T = 2, 14 * cs + 5
    src = torch.randn(B, T, 640, generator=torch.Generator().manual_seed(cs)).to(dev)
    dc = DynChunkTrainConfig(cs, lc)
    full = tr.encode(src, None, dynchunktrain_config=dc)
    ctx = tr.make_streaming_context(dc)
    out = torch.cat([tr.encode_streaming(src[:, t:t + cs].contiguous(), ctx) for t in range(0, T, cs)], dim=1)
    r = rel(out.cpu(), full.cpu())
    print(f"[stream GELU {att} ({cs}, {lc})] rel vs masked {r:.2e}")
    assert out.shape == full.shape and r < 3e-4


# the released model's inference layout with the recipe's entries (conformer_xlarge.yaml): the activation defined once and
# reused as conformer_activation, the recipe's token indices, CTC scorer and test search
INFERENCE_YAML = """
d_model: {d_model}
nhead: {nhead}
num_encoder_layers: {num_encoder_layers}
num_decoder_layers: {num_decoder_layers}
d_ffn: {d_ffn}
output_neurons: {vocab}
blank_index: 3
pad_index: 0
bos_index: 1
eos_index: 2
min_decode_ratio: 0.0
max_decode_ratio: {ratio}
test_beam_size: 80
ctc_weight_decode: 0.3
scorer_beam_scale: 0.3
activation: !name:torch.nn.GELU
normalizer: !new:speechbrain.processing.features.InputNormalization
    norm_type: global
compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: 16000
    n_fft: 400
    n_mels: 80
CNN: !new:speechbrain.lobes.models.convolution.ConvolutionFrontEnd
    input_shape: (8, 10, 80)
    num_blocks: 2
    num_layers_per_block: 1
    out_channels: (64, 32)
    kernel_sizes: (3, 3)
    strides: (2, 2)
    residuals: (False, False)
Transformer: !new:speechbrain.lobes.models.transformer.TransformerASR.TransformerASR
    input_size: 640
    tgt_vocab: !ref <output_neurons>
    d_model: !ref <d_model>
    nhead: !ref <nhead>
    num_encoder_layers: !ref <num_encoder_layers>
    num_decoder_layers: !ref <num_decoder_layers>
    d_ffn: !ref <d_ffn>
    dropout: 0.1
    conformer_activation: !ref <activation>
    activation: !ref <activation>
    encoder_module: conformer
    attention_type: RelPosMHAXL
    normalize_before: True
    causal: False
ctc_lin: !new:speechbrain.nnet.linear.Linear
    input_size: !ref <d_model>
    n_neurons: !ref <output_neurons>
seq_lin: !new:speechbrain.nnet.linear.Linear
    input_size: !ref <d_model>
    n_neurons: !ref <output_neurons>
ctc_scorer: !new:speechbrain.decoders.scorer.CTCScorer
    eos_index: !ref <eos_index>
    blank_index: !ref <blank_index>
    ctc_fc: !ref <ctc_lin>
scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <ctc_scorer>]
    weights:
        ctc: !ref <ctc_weight_decode>
    scorer_beam_scale: !ref <scorer_beam_scale>
decoder: !new:speechbrain.decoders.S2STransformerBeamSearcher
    modules: [!ref <Transformer>, !ref <seq_lin>]
    bos_index: !ref <bos_index>
    eos_index: !ref <eos_index>
    min_decode_ratio: !ref <min_decode_ratio>
    max_decode_ratio: !ref <max_decode_ratio>
    beam_size: !ref <test_beam_size>
    temperature: 1.15
    using_eos_threshold: True
    scorer: !ref <scorer>
encoder: !new:speechbrain.nnet.containers.LengthsCapableSequential
    input_shape: [null, null, 80]
    compute_features: !ref <compute_features>
    normalize: !ref <normalizer>
    cnn: !ref <CNN>
    transformer_encoder: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
        transformer: !ref <Transformer>
tokenizer: null
asr_model: !new:torch.nn.ModuleList
    - [!ref <CNN>, !ref <Transformer>, !ref <seq_lin>, !ref <ctc_lin>]
modules:
    normalizer: !ref <normalizer>
    encoder: !ref <encoder>
    decoder: !ref <decoder>
pretrainer: !new:speechbrain.utils.parameter_transfer.Pretrainer
    loadables:
        normalizer: !ref <normalizer>
        asr: !ref <asr_model>
    paths:
        asr: <save_dir>/asr.ckpt
"""


def test_from_hparams_local_directory(dev, wav, tmp_path):
    """the xlarge's inference layout (d_model 1024, 16 heads; 2 encoder and 1 decoder layer keep the checkpoint small) with
    `activation: !name:torch.nn.GELU` reused as `conformer_activation: !ref <activation>`, blank 3 / bos 1 / eos 2 and the
    beam 80 + CTC 0.3 test search loads through EncoderDecoderASR.from_hparams from a local directory; the loaded
    Transformer is a GELU Conformer holding the checkpoint, and transcribe_batch gives the tokens of the same modules
    constructed directly, 10 steps per utterance"""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.lobes.features import Fbank
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.processing.features import InputNormalization
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_XLARGE
    cfg = LO.reduced(LOQUACIOUS_XLARGE)
    sd = LO.state(cfg)
    ratio = (LO.BEAM["steps"] + 0.5) / 251
    yaml = INFERENCE_YAML.format(ratio=ratio, **{k: cfg[k] for k in ("d_model", "nhead", "num_encoder_layers",
                                                                   "num_decoder_layers", "d_ffn", "vocab")})
    tmp = write_pretrained_dir(tmp_path, yaml, dict(asr=module_list_ckpt(sd), normalizer=normalizer_ckpt(sd)))
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": str(dev)})
    dec = loaded.mods["decoder"]
    assert dec.model.conformer_activation == "gelu" and dec.model.engine_cfg()["conformer_activation"] == "gelu"
    assert torch.equal(dec.fc.w.weight.cpu(), sd["seq_lin.w.weight"])
    assert dec.ctc_scorer.blank_index == BLANK and dec.ctc_weight == 0.3 and (dec.bos_index, dec.eos_index) == (BOS, EOS)
    tr, _, _, bs = LO.search_modules(cfg, ratio)
    norm = InputNormalization(norm_type="global")
    norm.glob_mean, norm.glob_std, norm.count = sd["normalize.glob_mean"], sd["normalize.glob_std"], 1
    norm.eval()
    cnn = ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1, out_channels=(64, 32),
                              kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
    cnn.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("CNN.")})
    enc = LengthsCapableSequential(compute_features=Fbank(sample_rate=16000, n_fft=400, n_mels=80), normalize=norm, cnn=cnn)
    direct = EncoderDecoderASR(modules=dict(encoder=enc, transformer=tr, decoder=bs),
                               hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})
    w, lens = wav
    _, t1 = loaded.transcribe_batch(w, lens)
    _, t2 = direct.transcribe_batch(w, lens)
    print(f"MEASURE loquacious from_hparams tokens {t1}")
    assert t1 == t2 and len(t1) == 4 and sum(len(t) for t in t1) > 0
