"""-m gpu tests of the d_model 640 Conformer of the Libriheavy and People's Speech conformer_large recipes (14 layers, 8 heads
of 80 with RelPosMHAXL; 6 decoder layers with a GELU FFN over 5000 tokens, or a Swish FFN over 5120 tokens).

Kernel level: the encoder attention and the decode-step attention at head width 80 against the float64 references of
encoder_kernels_oracle.py / decoder_kernels_oracle.py, on the inputs and bars of test_gpu_encoder_kernels.py and
test_gpu_decoder_kernels.py (whose case functions run here with head width 80).

Model level, on seeded weights (utils/seeded_init.CONFORMER_640 / CONFORMER_640_PEOPLES), against the reference outputs in
tests/golden/conformer640.pt (generator: tools/make_conformer640_golden.py) and against the fp32 CPU oracle of
conformer640_oracle.py recomputed here (it equals the reference to 1e-5 on every fixture entry, test_conformer640_oracle.py):
4 x 10 s ragged [1.0, 0.9, 0.6, 0.3] waveforms -> encoder states (all frames and each utterance's valid frames, rel-L2 <=
ENC_BAR), 48 greedy steps and teacher-forced decode() on 48 positions, Libriheavy's beam 66 + TransformerLM 0.6 + CTC 0.4
and People's Speech's beam 10 + CTC 0.3 for 24 steps (parity.check_beam), a 1.3 s utterance, and both
recipes' inference layouts loaded through EncoderDecoderASR.from_hparams from a local directory.

ENC_BAR: the oracle with every GEMM operand rounded to fp16 sits at about 5e-4 of the fp32 oracle on this input
(test_conformer640_oracle.py::test_fp16_operand_error_estimate), so the Conformer's 1e-3 bar holds at d_model 640."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conformer640_oracle as CO  # noqa: E402
import test_gpu_decoder_kernels as DKT  # noqa: E402
import test_gpu_encoder_kernels as EKT  # noqa: E402
from mirrors import build_mirror, seeded  # noqa: E402
from parity import (BEAM_TOL, check_alone_vs_batch, check_beam, check_encoder, check_greedy, check_summary,  # noqa: E402,F401
                    dev, lm_scorer_state, module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir)

ENC_BAR = 1e-3
DEC_BAR = 2e-3  # teacher-forced decode(), rel-L2 (measured 4.4e-4)
BOS, EOS = CO.BOS, CO.EOS
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conformer640.pt")

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ kernels at head width 80
@pytest.mark.parametrize("T", [1, 17, 63, 64, 65, 251, 1000])
@pytest.mark.parametrize("relpos", [True, False])
def test_attention80_full_context(dev, relpos, T):
    EKT.test_attention_full_context(dev, 80, relpos, T)


@pytest.mark.parametrize("T", [1036, 1037, 2500])
def test_attention80_relpos_long(dev, T):
    EKT.test_attention_relpos_long(dev, 80, T)


@pytest.mark.parametrize("T", [251, 300])
@pytest.mark.parametrize("chunk,left", EKT.WINDOWS)
@pytest.mark.parametrize("relpos", [False, True])
def test_attention80_dynamic_chunk(dev, relpos, chunk, left, T):
    EKT.test_attention_dynamic_chunk(dev, 80, relpos, chunk, left, T)


def test_attention80_built_alone(dev):
    """80 is built with and without RelPosMHAXL; 48, 96 and RelPosMHAXL at 128 still are not."""
    import ctypes

    from speechbrain_b200._lib import lib, ptr, stream_ptr
    T, H = 16, 2
    qkv = torch.zeros(T, 3 * H * 128, dtype=torch.float16, device=dev)
    out = torch.zeros(T, H * 128, dtype=torch.float16, device=dev)
    uv = torch.zeros(H * 128, device=dev)
    P = torch.zeros(T, H * 128, dtype=torch.float16, device=dev)
    call = lambda dh, rp: lib().sbk_encoder_attention_test(ptr(qkv), 1, T, H, dh, None, rp, ptr(uv), ptr(uv), ptr(P),  # noqa: E731
                                                           ctypes.c_float(0.1), 0, -1, ptr(out), stream_ptr(dev))
    assert call(80, 1) == 0 and call(80, 0) == 0
    assert call(48, 1) != 0 and call(96, 1) != 0 and call(96, 0) != 0 and call(128, 1) != 0


@pytest.mark.parametrize("mode", DKT.SELF_MODES)
def test_decode_self_attention80(dev, mode):
    DKT.test_self_attention(dev, 80, mode)


def test_decode_cross_attention80(dev):
    """row-major cross K/V (the head-major layout is built for head width 64), up to 2560 frames"""
    DKT.test_cross_attention(dev, 80, "row")


# ------------------------------------------------------------------------------------------------ model level
@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN)


def _case(cfg, fx_recipe):
    """seeded weights, the waveforms, the oracle's encoder states and greedy search (CPU), and the reference fixture"""
    sd = seeded(cfg)
    wav, lens = CO.waveforms()
    enc = CO.encode(cfg, sd, wav, lens)
    _, _, logits = CO.greedy(cfg, sd, enc, lens)
    return dict(cfg=cfg, sd=sd, wav=wav, lens=lens, enc=enc, T=enc.shape[1], greedy_logits=logits, fx=fx_recipe)


@pytest.fixture(scope="module")
def libriheavy(fx):
    from speechbrain_b200.utils.seeded_init import CONFORMER_640
    return _case(CONFORMER_640, fx["libriheavy"])


@pytest.fixture(scope="module")
def peoples(fx):
    from speechbrain_b200.utils.seeded_init import CONFORMER_640_PEOPLES
    return _case(CONFORMER_640_PEOPLES, fx["peoples"])


def _check_summary(tag, x, summ, bar):
    """the fixture names the row norms row_norm"""
    check_summary(tag, x, summ["row_norm"], summ["sample_idx"], summ["sample_rows"], bar)


@pytest.mark.parametrize("recipe", ["libriheavy", "peoples"])
def test_wav_to_encoder_and_greedy(dev, recipe, request):
    """wav -> Fbank -> CNN -> encoder -> 48 greedy steps on the device vs the reference fixture and the oracle; a rerun is
    bit-identical and the first utterance alone equals its rows in the batch to 1e-5"""
    from speechbrain_b200.engine import AsrEngine
    case = request.getfixturevalue(recipe)
    g = case["fx"]
    eng = AsrEngine(case["cfg"], case["sd"], device=str(dev))
    wav, lens = case["wav"].to(dev), case["lens"].to(dev)
    def greedy(w, ln):
        pred, score, enc, _ = eng.transcribe_greedy_dev(w, ln, CO.STEPS, BOS, EOS, want_enc=True)
        return enc, pred, score
    enc, pred, score = greedy(wav, lens)
    torch.cuda.synchronize()
    enc = enc.cpu()
    _check_summary(f"{recipe} encoder", enc, g["enc"], ENC_BAR)
    check_encoder(recipe, enc, case["enc"], [round(float(x) * case["T"]) for x in case["lens"]], ENC_BAR)
    check_greedy(recipe, pred.cpu(), score.cpu(), g["greedy_tokens"], g["greedy_margin"], g["greedy_chosen_lp"], stop_at=EOS)
    check_alone_vs_batch(greedy, wav, lens, 1e-5, relative=True)
    if "short" in g:  # one 1.3 s utterance (T = 33)
        w1, l1 = CO.waveforms(seed=13, L=20800, lens=[1.0])
        _, _, e1, _ = eng.transcribe_greedy_dev(w1.to(dev), l1.to(dev), 4, BOS, EOS, want_enc=True)
        r = rel(e1.cpu(), g["short"]["enc"])
        print(f"MEASURE {recipe} 1.3 s utterance encoder vs reference rel-L2 {r:.3e}")
        assert r <= ENC_BAR


@pytest.mark.parametrize("recipe", ["libriheavy", "peoples"])
def test_decode_teacher_forced(dev, recipe, request):
    """TransformerASR.decode() (the mirror, built with the recipe's decoder activation) on 48 positions of the oracle's
    encoder states vs the reference fixture and the oracle; covers the Swish FFN on both projection back ends"""
    case = request.getfixturevalue(recipe)
    cfg = case["cfg"]
    tr = build_mirror(cfg, case["sd"]).tr
    assert tr.decoder_activation == cfg["decoder_activation"]
    tgt = CO.teacher_tokens(cfg)
    enc_len = torch.round(case["lens"] * case["T"]).int()
    ref = CO.decode(cfg, case["sd"], tgt, case["enc"], enc_len)
    for rows in (64, 1):  # weight streaming, then the wgmma projections
        tr._decoder_engine(dev).set_decoder_tc_min_rows(rows)
        out, _ = tr.decode(tgt.to(dev), case["enc"].to(dev), enc_len.to(dev))
        out = out.cpu()
        r = rel(out, ref)
        print(f"MEASURE {recipe} decode() tc_min_rows={rows} rel-L2 vs oracle {r:.3e}")
        assert torch.isfinite(out).all() and r <= DEC_BAR
        _check_summary(f"{recipe} decode() tc_min_rows={rows}", out, case["fx"]["decode"], DEC_BAR)
    tr._decoder_engine(dev).set_decoder_tc_min_rows(64)


def searcher(m, beam, lm_weight, ctc_weight, max_decode_ratio):
    """the recipes' test search on the mirror m: [TransformerLM, CTC] (Libriheavy) or [CTC] (People's Speech)"""
    scorers = dict(transformerlm=lm_weight, ctc=ctc_weight) if lm_weight else dict(ctc=ctc_weight)
    kwargs = dict(min_decode_ratio=0.0, beam_size=beam, temperature=1.15, using_eos_threshold=False, length_normalization=True)
    return m.searcher(kwargs, max_decode_ratio, scorers=scorers)


@pytest.mark.parametrize("recipe", ["libriheavy", "peoples"])
def test_beam_search(dev, recipe, request):
    """the recipe's test search (Libriheavy: beam 66, TransformerLM 0.6, CTC 0.4 on utterances 0 and 3; People's Speech:
    beam 10, CTC 0.3) for 24 steps on the oracle's encoder states vs the reference fixture: best scores within 3e-2, and a
    best hypothesis that differs from the reference's must score, by the oracle walked along its tokens, within 3e-2 of its
    own score and no worse than the reference's best (parity.check_beam); the n-best list against the oracle's"""
    case = request.getfixturevalue(recipe)
    cfg, sd, gb = case["cfg"], case["sd"], case["fx"]["beam"]
    utts = gb["utts"]
    bs = searcher(build_mirror(cfg, sd), gb["beam"], gb["lm_weight"], gb["ctc_weight"], (gb["steps"] + 0.5) / case["T"])
    enc, lens = case["enc"][utts], case["lens"][utts]
    hyps, _, scores, _ = bs(enc.to(dev), lens.to(dev))
    scores = scores.cpu().view(-1, 1)
    h2, _, s2, _ = bs(enc.to(dev), lens.to(dev))
    assert h2 == hyps and torch.equal(s2.cpu().view(-1, 1), scores), "rerun differs"
    # the fixture keeps the reference's best hypotheses and scores; its n-best list is the oracle's
    check_beam(f"{recipe} beam {gb['beam']}", [list(h) + [EOS] for h in hyps], scores, [list(h) + [EOS] for h in gb["hyps"]],
               gb["scores"].view(-1, 1), lambda idx, tokens: CO.beam(cfg, sd, enc[idx], lens[idx], dict(gb, beam=1), forced=tokens))
    bs.return_topk, bs.topk = True, gb["beam"]
    _, _, nbest, _ = bs(enc.to(dev), lens.to(dev))
    _, _, ref_s, _ = CO.beam(cfg, sd, enc, lens, gb, return_topk=True, topk=gb["beam"])
    nbest_err = (nbest.cpu() - ref_s).abs().max().item()
    print(f"MEASURE {recipe} beam {gb['beam']}: max |n-best - oracle| {nbest_err:.2e}")
    assert nbest_err < BEAM_TOL


INFERENCE_YAML = """
d_model: 640
output_neurons: {vocab}
bos_index: 1
eos_index: 2
blank_index: 0
activation: !name:{activation}
normalizer: !new:speechbrain.processing.features.InputNormalization
    norm_type: global
compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: 16000
    n_fft: 512
    n_mels: 80
    win_length: 32
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
    nhead: 8
    num_encoder_layers: 14
    num_decoder_layers: 6
    d_ffn: 2048
    dropout: 0.1
    activation: !ref <activation>
    conformer_activation: !name:speechbrain.nnet.activations.Swish
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
{lm_block}decoder: !new:speechbrain.decoders.S2STransformerBeamSearcher
    modules: [!ref <Transformer>, !ref <seq_lin>]
    bos_index: !ref <bos_index>
    eos_index: !ref <eos_index>
    min_decode_ratio: 0.0
    max_decode_ratio: {ratio}
    beam_size: {beam}
    temperature: 1.15
    using_eos_threshold: False
    length_normalization: True
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
        asr: !ref <asr_model>{lm_loadable}
    paths:
        asr: <save_dir>/asr.ckpt{lm_path}
"""
LM_BLOCK = """lm_model: !new:speechbrain.lobes.models.transformer.TransformerLM.TransformerLM
    vocab: !ref <output_neurons>
    d_model: 768
    nhead: 12
    num_encoder_layers: 12
    num_decoder_layers: 0
    d_ffn: 3072
    dropout: 0.0
    activation: !name:torch.nn.GELU
    normalize_before: False
transformerlm_scorer: !new:speechbrain.decoders.scorer.TransformerLMScorer
    language_model: !ref <lm_model>
    temperature: 1.15
scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <transformerlm_scorer>, !ref <ctc_scorer>]
    weights:
        ctc: 0.4
        transformerlm: 0.6
"""
CTC_BLOCK = """scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <ctc_scorer>]
    weights:
        ctc: 0.3
"""


@pytest.mark.parametrize("recipe", ["libriheavy", "peoples"])
def test_from_hparams_local_directory(dev, recipe, request, tmp_path):
    """Each recipe's inference layout (Libriheavy: beam 66 with the [TransformerLM, CTC] ScorerBuilder; People's Speech:
    beam 10 with CTC and `activation: !name:speechbrain.nnet.activations.Swish`) loads through EncoderDecoderASR.from_hparams
    from a local directory, the checkpoints land in the mirrors, and transcribe_batch gives the tokens of the same modules
    constructed directly, 24 steps per utterance"""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    case = request.getfixturevalue(recipe)
    cfg, sd = case["cfg"], case["sd"]
    lm = recipe == "libriheavy"
    beam, ratio = (66, 0.6, 0.4) if lm else (10, 0.0, 0.3), (24 + 0.5) / case["T"]
    yaml = INFERENCE_YAML.format(
        vocab=cfg["vocab"], ratio=ratio, beam=beam[0],
        activation="speechbrain.nnet.activations.Swish" if cfg["decoder_activation"] == "swish" else "torch.nn.GELU",
        lm_block=LM_BLOCK if lm else CTC_BLOCK, lm_loadable="\n        lm: !ref <lm_model>" if lm else "",
        lm_path="\n        lm: <save_dir>/lm.ckpt" if lm else "")
    ckpts = dict(asr=module_list_ckpt(sd), normalizer=normalizer_ckpt(sd), **(dict(lm=lm_scorer_state(cfg["vocab"])) if lm else {}))
    tmp = write_pretrained_dir(tmp_path, yaml, ckpts)
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": str(dev)})
    assert torch.equal(loaded.mods["decoder"].fc.w.weight.cpu(), sd["seq_lin.w.weight"])
    m = build_mirror(cfg, sd)
    bs = searcher(m, beam[0], beam[1], beam[2], ratio)
    assert loaded.mods["decoder"].model.decoder_activation == m.tr.decoder_activation == cfg["decoder_activation"]
    direct = EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=bs),
                               hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})
    wav, lens = case["wav"], case["lens"]
    _, t1 = loaded.transcribe_batch(wav, lens)
    _, t2 = direct.transcribe_batch(wav, lens)
    print(f"MEASURE {recipe} from_hparams tokens {t1}")
    assert t1 == t2 and len(t1) == 4 and sum(len(t) for t in t1) > 0


def test_streaming_rejected_at_head_width_80(dev):
    """the streaming ring is not built at head width 80: make_streaming_context raises before any device work"""
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = TransformerASR(tgt_vocab=50, input_size=640, d_model=640, nhead=8, num_encoder_layers=1, num_decoder_layers=1,
                        encoder_module="conformer", attention_type="RelPosMHAXL", normalize_before=True, causal=False)
    before = torch.cuda.memory_allocated(dev)
    with pytest.raises(NotImplementedError):
        tr.make_streaming_context(DynChunkTrainConfig(chunk_size=16, left_context_size=2))
    with pytest.raises(NotImplementedError):
        tr.encode_streaming(torch.zeros(1, 16, 640, device=dev), None)
    assert torch.cuda.memory_allocated(dev) == before and not tr._slots
