"""Branchformer encoder (TransformerASR(encoder_module="branchformer"), Branchformer.py:92-410), no GPU needed: the CPU oracle
against the reference outputs stored in tests/golden/branchformer.pt (generator: tools/make_branchformer_golden.py), the
mirror's state_dict layout, the constructor / encode errors, a from_hparams directory in the layout of the LibriSpeech
Branchformer seq2seq recipe, and the fp16-operand error the device encoder can be expected to show."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import case_wav, check_summary, module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir  # noqa: E402
import branchformer_oracle as BO  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "branchformer.pt"))


def _oracle_encode(cfg, sd, case, q=None):
    return BO.wav_to_states(*case_wav(case), sd, cfg, q=q)


@pytest.mark.parametrize("case", ["large", "short", "ctc"])
def test_oracle_matches_reference(fx, case):
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC, BRANCHFORMER_LARGE
    cfg = BRANCHFORMER_CTC if case == "ctc" else BRANCHFORMER_LARGE
    sd = BO.state(cfg, fx)
    with torch.no_grad():
        enc = _oracle_encode(cfg, sd, fx[case])
    if case == "short":
        r = rel(enc, fx[case]["enc_out"])
        print(f"[{case}] oracle vs reference encoder rel-L2 {r:.2e}")
        assert r <= 1e-6
    else:  # the fixture keeps the per-frame norms and sampled rows instead of the whole states
        c = fx[case]
        check_summary(f"{case} oracle", enc, c["frame_norm"], c["sample_idx"], c["sample_rows"], 1e-6)
    if case == "ctc":
        lp = torch.log_softmax(torch.nn.functional.linear(enc, sd["ctc_lin.w.weight"], sd["ctc_lin.w.bias"]), -1)
        assert rel(lp, fx["ctc"]["log_probs"]) <= 1e-6


def _mirror(cfg, **kw):
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    args = dict(tgt_vocab=cfg["vocab"], input_size=640, d_model=cfg["d_model"], nhead=cfg["nhead"],
                num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=cfg["num_decoder_layers"], d_ffn=cfg["d_ffn"],
                activation=torch.nn.GELU, branchformer_activation=torch.nn.GELU, encoder_module="branchformer",
                csgu_linear_units=cfg["csgu_linear_units"], kernel_size=cfg["kernel_size"], attention_type="RelPosMHAXL",
                normalize_before=True, causal=False)
    args.update(kw)
    return TransformerASR(**args)


@pytest.mark.parametrize("which", ["large", "ctc"])
def test_state_dict_layout_matches_reference(fx, which):
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC, BRANCHFORMER_LARGE
    tr = _mirror(BRANCHFORMER_CTC if which == "ctc" else BRANCHFORMER_LARGE)
    ours = [(k, tuple(v.shape)) for k, v in tr.state_dict().items()]
    ref = [(k, tuple(s)) for k, s in fx["keys_" + which]]
    assert sorted(ours) == sorted(ref), set(ours) ^ set(ref)


def test_constructor_rejects_what_is_not_built():
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC
    cfg = dict(BRANCHFORMER_CTC, num_encoder_layers=1)
    _mirror(cfg, branchformer_activation=torch.nn.ReLU, gate_activation=torch.nn.Identity, kernel_size=15)
    _mirror(cfg, branchformer_activation=None, gate_activation=None)
    for kw in (dict(attention_type="regularMHA"), dict(attention_type="hypermixing"), dict(attention_type="RoPEMHA"),
               dict(use_linear_after_conv=True), dict(gate_activation=torch.nn.Sigmoid), dict(gate_activation=torch.nn.GELU),
               dict(branchformer_activation=torch.nn.SiLU), dict(kernel_size=30), dict(kernel_size=33),
               dict(csgu_linear_units=2404), dict(csgu_linear_units=2401)):
        with pytest.raises(NotImplementedError):
            _mirror(cfg, **kw)


def test_encode_errors():
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC
    tr = _mirror(dict(BRANCHFORMER_CTC, num_encoder_layers=1))
    with pytest.raises(AssertionError):
        tr.encode(torch.zeros(1, 40, 640), dynchunktrain_config=DynChunkTrainConfig(8, 2))
    with pytest.raises(RuntimeError, match="reflect padding"):  # T <= (K - 1) / 2: the reference's F.pad fails
        tr.encode(torch.zeros(1, 15, 640))
    with pytest.raises(NotImplementedError):
        tr.make_streaming_context(DynChunkTrainConfig(8, 2))
    with pytest.raises(NotImplementedError):
        tr.encode_streaming(torch.zeros(1, 8, 640), None)


YAML = """
sample_rate: 16000
n_fft: 512
n_mels: 80
win_length: 32
d_model: 512
nhead: 8
num_encoder_layers: 2
num_decoder_layers: 1
csgu_linear_units: 3072
csgu_kernel_size: 31
transformer_dropout: 0.1
activation: !name:torch.nn.GELU
output_neurons: 60
blank_index: 0
bos_index: 1
eos_index: 2
min_decode_ratio: 0.0
max_decode_ratio: 1.0
test_beam_size: 4
ctc_weight_decode: 0.40

normalizer: !new:speechbrain.processing.features.InputNormalization
    norm_type: global

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
    dropout: !ref <transformer_dropout>
    activation: !ref <activation>
    branchformer_activation: !ref <activation>
    encoder_module: branchformer
    csgu_linear_units: !ref <csgu_linear_units>
    kernel_size: !ref <csgu_kernel_size>
    attention_type: RelPosMHAXL
    normalize_before: True
    causal: False

ctc_lin: !new:speechbrain.nnet.linear.Linear
    input_size: !ref <d_model>
    n_neurons: !ref <output_neurons>

seq_lin: !new:speechbrain.nnet.linear.Linear
    input_size: !ref <d_model>
    n_neurons: !ref <output_neurons>

tokenizer: !new:sentencepiece.SentencePieceProcessor

compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: !ref <sample_rate>
    n_fft: !ref <n_fft>
    n_mels: !ref <n_mels>
    win_length: !ref <win_length>

ctc_scorer: !new:speechbrain.decoders.scorer.CTCScorer
    eos_index: !ref <eos_index>
    blank_index: !ref <blank_index>
    ctc_fc: !ref <ctc_lin>

scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <ctc_scorer>]
    weights:
        ctc: !ref <ctc_weight_decode>

decoder: !new:speechbrain.decoders.S2STransformerBeamSearcher
    modules: [!ref <Transformer>, !ref <seq_lin>]
    bos_index: !ref <bos_index>
    eos_index: !ref <eos_index>
    min_decode_ratio: !ref <min_decode_ratio>
    max_decode_ratio: !ref <max_decode_ratio>
    beam_size: !ref <test_beam_size>
    temperature: 1.15
    using_eos_threshold: False
    length_normalization: True
    scorer: !ref <scorer>

Tencoder: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
    transformer: !ref <Transformer>

encoder: !new:speechbrain.nnet.containers.LengthsCapableSequential
    input_shape: [null, null, !ref <n_mels>]
    compute_features: !ref <compute_features>
    normalize: !ref <normalizer>
    cnn: !ref <CNN>
    transformer_encoder: !ref <Tencoder>

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
        tokenizer: !ref <tokenizer>
    paths:
        asr: !ref <save_dir>/asr.ckpt
"""


def test_from_hparams_branchformer_recipe_layout(tmp_path):
    import sentencepiece as spm

    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_LARGE, seeded_asr_state
    cfg = dict(BRANCHFORMER_LARGE, num_encoder_layers=2, num_decoder_layers=1, vocab=60)
    sd = seeded_asr_state(cfg, 0)
    tmp = write_pretrained_dir(tmp_path, YAML, dict(asr=module_list_ckpt(sd), normalizer=normalizer_ckpt(sd)))
    with open(os.path.join(tmp, "corpus.txt"), "w") as f:
        words = ["branch", "former", "gating", "spatial", "conv", "reflect", "merge", "attention", "encoder", "decoder"]
        for i in range(400):
            f.write(" ".join(words[(i * 7 + j * 3) % len(words)] for j in range(9)) + f" {i % 13}\n")
    spm.SentencePieceTrainer.train(input=os.path.join(tmp, "corpus.txt"), model_prefix=os.path.join(tmp, "tok"), vocab_size=60,
                                   model_type="bpe", bos_id=1, eos_id=2, unk_id=0, pad_id=-1, minloglevel=2)
    os.rename(os.path.join(tmp, "tok.model"), os.path.join(tmp, "tokenizer.ckpt"))
    asr = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    tr = asr.transformer
    assert tr.encoder_module == "branchformer" and tr.csgu_linear_units == 3072 and asr.mods["decoder"].model is tr
    key = "encoder.layers.1.convolution_branch.csgu.conv.conv.weight"
    assert torch.equal(tr.state_dict()[key], sd["Transformer." + key])
    assert torch.equal(tr.state_dict()["encoder.layers.0.merge_proj.weight"], sd["Transformer.encoder.layers.0.merge_proj.weight"])
    assert tr.engine_cfg()["encoder_module"] == "branchformer"


def test_fp16_operand_error_estimate(fx):
    """The oracle with every GEMM operand (and the CSGU input) rounded to fp16 on the Branchformer-L input: the encoder
    error the device can be expected to show against the reference.  It is 1.0e-3 (the Conformer-L sits well below its 1e-3
    bar): the 18 layers add to the residual stream without a LayerNorm in between, so the rounding of every layer's
    operands accumulates (5e-4 after layer 1).  That is why the device encoder bar for the Branchformer is 1.5e-3
    (test_gpu_branchformer.py); this test pins the estimate that bar rests on."""
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_LARGE
    sd = BO.state(BRANCHFORMER_LARGE, fx)
    with torch.no_grad():
        enc = _oracle_encode(BRANCHFORMER_LARGE, sd, fx["large"], q=lambda t: t.half().float())
        ref = _oracle_encode(BRANCHFORMER_LARGE, sd, fx["large"])  # = the reference (test_oracle_matches_reference)
    lens = fx["large"]["abs_len"]
    per_utt = [rel(enc[b, :int(lens[b])], ref[b, :int(lens[b])]) for b in range(ref.shape[0])]
    r = rel(enc, ref)
    print(f"fp16-operand oracle vs reference: encoder rel-L2 {r:.2e}, valid frames per utterance "
          f"{['%.2e' % x for x in per_utt]}")
    assert r <= 1.2e-3 and max(per_utt) <= 1.2e-3
