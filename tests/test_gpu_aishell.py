"""-m gpu tests of the AISHELL-1 Transformer recipe's device path: the 256-channel 2-block front-end kernels (conv1 per frame,
conv2 as a wgmma implicit GEMM with the LayerNorm in its epilogue) against the float64 oracle (tests/aishell_oracle.py), the
whole pipeline (Fbank -> CMVN -> CNN -> 12 regularMHA layers of 4 heads of 64 -> greedy decode) and the recipe's beam-10 +
CTC 0.4 test search against the reference outputs in tests/golden/aishell_transformer.pt, a from_hparams round trip of the
recipe's module layout, and the refusal of the 2-block channel pairs that are not built.

Front-end bar: rel-L2 <= 5e-4 (the 3-block front-end's: fp16 act1 and conv2 operands).  Encoder bar: rel-L2 <= 1e-3.
Greedy: tokens identical up to the first decision whose reference top-1/top-2 margin is below 5e-3 (parity.check_greedy).
Beam: hypotheses identical, scores within 5e-2."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import (case_wav, check_alone_vs_batch, check_encoder, check_greedy, check_summary, dev,  # noqa: E402,F401
                    module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir)
import aishell_oracle as AO  # noqa: E402
from mirrors import build_mirror, seeded  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CNN_BAR = 5e-4
ENC_BAR = 1e-3

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "aishell_transformer.pt"))


@pytest.fixture(scope="module")
def sd(fx):
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER
    return seeded(AISHELL_TRANSFORMER, fx["weight_seed"])


def _mirror(sd):
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER
    return build_mirror(AISHELL_TRANSFORMER, sd)


def _launches():
    from speechbrain_b200 import _lib
    return _lib.lib().sbk_launch_count()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T0", [3, 5, 6, 1001])
def test_front_end_kernels_vs_fp64_oracle(dev, sd, B, T0):
    """3 frames is the shortest input the reflect padding accepts (T1 = 2); 5 and 6 give odd and even T1 at the time edge
    (T2 = 2 with the last conv2 frame reading the reflected row, or not); 1001 is 10 s (T2 = 251: 42 CTAs of 6 frames per
    utterance, the last one with 5)."""
    cnn = _mirror(sd).cnn.to(dev)
    g = torch.Generator().manual_seed(2000 + 10 * T0 + B)
    feats = torch.randn(B, T0, 80, generator=g) * 2.0
    out = cnn(feats.to(dev)).cpu()
    ref = AO.cnn(feats.double(), sd)
    err = rel(out.double(), ref)
    print(f"256-channel front-end B={B} T0={T0} -> {tuple(out.shape)}: rel-L2 {err:.2e}, "
          f"max abs {(out.double() - ref).abs().max():.2e}")
    assert out.shape == ref.shape and torch.isfinite(out).all() and err <= CNN_BAR
    assert torch.equal(out, cnn(feats.to(dev)).cpu())
    one = cnn(feats[-1:].to(dev)).cpu()  # batch independence
    assert torch.equal(one[0], out[-1])


def test_front_end_rejects_too_short_before_any_launch(dev, sd):
    cnn = _mirror(sd).cnn.to(dev)
    cnn(torch.randn(1, 3, 80, device=dev))  # the engine exists before the count starts
    n0 = _launches()
    with pytest.raises(RuntimeError, match="reflect"):
        cnn(torch.randn(1, 2, 80, device=dev))
    assert _launches() == n0


@pytest.mark.parametrize("channels", [(128, 32), (256, 128), (64, 64)])
def test_unbuilt_channel_pairs_refused_before_any_launch(dev, sd, channels):
    """The C ABI states the built 2-block pairs: any other is refused at creation, before any device work."""
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER, seeded_asr_state
    cfg = dict(AISHELL_TRANSFORMER, cnn_channels=channels, input_size=20 * channels[1], num_encoder_layers=1,
               num_decoder_layers=1)
    state = seeded_asr_state(cfg, 0)
    torch.cuda.synchronize()
    n0 = _launches()
    with pytest.raises(RuntimeError, match="not built"):
        AsrEngine(cfg, state, device=dev, parts=("fbank", "cnn", "encoder"))
    assert _launches() == n0


def _engine(sd, dev):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER
    return AsrEngine(AISHELL_TRANSFORMER, sd, device=dev)


def test_pipeline_cnn_encoder_and_greedy(dev, fx, sd):
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER as cfg
    g = fx["large"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        ref = AO.encode(AO.wav_to_cnn(wav, lens, sd, cfg), lens, sd, cfg)
    check_summary("aishell oracle enc", ref, g["enc"]["frame_norm"], g["enc"]["sample_idx"], g["enc"]["sample_rows"], 1e-5)
    m = _mirror(sd)
    cnn = m.front_end().to(dev)(wav.to(dev), lens.to(dev)).cpu().flatten(2)
    check_summary("aishell cnn", cnn, g["cnn"]["frame_norm"], g["cnn"]["sample_idx"], g["cnn"]["sample_rows"], CNN_BAR)
    eng = _engine(sd, dev)
    S = g["greedy_tokens"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), lens.to(dev), S, 1, 2, want_enc=True)
    torch.cuda.synchronize()
    check_encoder("aishell", enc.cpu(), ref, g["abs_len"], ENC_BAR)
    check_summary("aishell enc", enc.cpu(), g["enc"]["frame_norm"], g["enc"]["sample_idx"], g["enc"]["sample_rows"], ENC_BAR)
    check_greedy("aishell", pred.cpu(), None, g["greedy_tokens"], g["greedy_margin"], chosen_lp=None)
    check_alone_vs_batch(lambda w, ln: eng.encode_wav(w.to(dev), ln.to(dev)), wav, lens, 1e-5)


def _searcher(m, max_decode_ratio):
    """train_ASR_transformer.yaml's test search on the mirror m: beam 10, no EOS threshold, length normalisation, CTC 0.4"""
    kwargs = dict(min_decode_ratio=0.0, beam_size=10, using_eos_threshold=False, length_normalization=True)
    return m.searcher(kwargs, max_decode_ratio, scorers=dict(ctc=0.4))


def test_beam10_ctc_matches_reference(dev, fx, sd):
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER as cfg
    g, gb = fx["large"], fx["beam10"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        enc = AO.encode(AO.wav_to_cnn(wav, lens, sd, cfg), lens, sd, cfg)
    hyps, _, scores, _ = _searcher(_mirror(sd), gb["max_decode_ratio"])(enc.to(dev), lens.to(dev))
    print(f"[aishell beam10 ctc] hyps equal {hyps == gb['hyps']}; score err {(scores.cpu() - gb['scores']).abs().max():.2e}")
    assert hyps == gb["hyps"]
    assert (scores.cpu() - gb["scores"]).abs().max() < 5e-2


HPARAMS = """
d_model: 256
output_neurons: 5000
bos_index: 1
eos_index: 2
blank_index: 0
normalize: !new:speechbrain.processing.features.InputNormalization
    norm_type: global
compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: 16000
    n_fft: 400
    n_mels: 80
CNN: !new:speechbrain.lobes.models.convolution.ConvolutionFrontEnd
    input_shape: (8, 10, 80)
    num_blocks: 2
    num_layers_per_block: 1
    out_channels: (256, 256)
    kernel_sizes: (3, 3)
    strides: (2, 2)
    residuals: (False, False)
Transformer: !new:speechbrain.lobes.models.transformer.TransformerASR.TransformerASR
    input_size: 5120
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
ctc_scorer: !new:speechbrain.decoders.scorer.CTCScorer
    eos_index: !ref <eos_index>
    blank_index: !ref <blank_index>
    ctc_fc: !ref <ctc_lin>
scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <ctc_scorer>]
    weights:
        ctc: 0.40
decoder: !new:speechbrain.decoders.S2STransformerBeamSearcher
    modules: [!ref <Transformer>, !ref <seq_lin>]
    bos_index: !ref <bos_index>
    eos_index: !ref <eos_index>
    min_decode_ratio: 0.0
    max_decode_ratio: 1.0
    beam_size: 10
    using_eos_threshold: False
    length_normalization: True
    scorer: !ref <scorer>
Tencoder: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
    transformer: !ref <Transformer>
encoder: !new:speechbrain.nnet.containers.LengthsCapableSequential
    input_shape: [null, null, 80]
    compute_features: !ref <compute_features>
    normalize: !ref <normalize>
    cnn: !ref <CNN>
    transformer_encoder: !ref <Tencoder>
tokenizer: null
asr_model: !new:torch.nn.ModuleList
    - [!ref <CNN>, !ref <Transformer>, !ref <seq_lin>, !ref <ctc_lin>]
modules:
    CNN: !ref <CNN>
    Transformer: !ref <Transformer>
    seq_lin: !ref <seq_lin>
    ctc_lin: !ref <ctc_lin>
    normalize: !ref <normalize>
    encoder: !ref <encoder>
    decoder: !ref <decoder>
pretrainer: !new:speechbrain.utils.parameter_transfer.Pretrainer
    loadables:
        normalizer: !ref <normalize>
        asr: !ref <asr_model>
    paths:
        asr: <save_dir>/asr.ckpt
"""


def test_from_hparams_local_directory_round_trip(dev, fx, sd, tmp_path):
    """A pretrained-model directory with train_ASR_transformer.yaml's module layout (the 256-channel CNN, the Transformer
    encoder at d_model 256, seq_lin, ctc_lin, the beam-10 + CTC 0.4 test search) loads through from_hparams, the
    checkpoints land in the mirrors, and it transcribes like the same modules wired directly."""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    tmp = write_pretrained_dir(tmp_path, HPARAMS, dict(asr=module_list_ckpt(sd), normalizer=normalizer_ckpt(sd)))
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": str(dev)})
    m = _mirror(sd)
    direct = EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=_searcher(m, 1.0)),
                               hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})
    assert torch.equal(loaded.mods["decoder"].fc.w.weight.cpu(), sd["seq_lin.w.weight"])
    assert torch.equal(loaded.mods["CNN"].convblock_1.convs.conv_0.conv.weight.cpu(),
                       sd["CNN.convblock_1.convs.conv_0.conv.weight"])
    wav, lens = case_wav(fx["large"])
    w1, t1 = loaded.transcribe_batch(wav, lens)
    w2, t2 = direct.transcribe_batch(wav, lens)
    print("from_hparams tokens", [len(t) for t in t1])
    assert t1 == t2 and len(t1) == 4 and sum(len(t) for t in t1) > 0
