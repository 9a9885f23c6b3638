"""HyperConformer encoder (TransformerASR(attention_type="hypermixing"), Conformer.py:451-499 with nnet/hypermixing.py), no GPU
needed: the CPU oracle against the reference outputs stored in tests/golden/hyperconformer.pt (generator:
tools/make_hyperconformer_golden.py), the mirror's state_dict layout, the constructor / encode errors, a from_hparams
directory in the layout of the LibriSpeech hyperconformer_22M recipe, and the fp16-operand error the device encoder can be
expected to show."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import case_wav, check_summary, module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir  # noqa: E402
import hyperconformer_oracle as HO  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "hyperconformer.pt"))


def _state(fx):
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M, scale_hypernet, seeded_asr_state
    return scale_hypernet(seeded_asr_state(HYPERCONFORMER_22M, fx["weight_seed"]), fx["hypernet_gain"])


def test_oracle_matches_reference(fx):
    """Frame norms and the full short-utterance states to 1e-6; the sampled full rows to 2e-6 (fp32 summation-order noise of
    individual channels: 1.2e-6 against the reference's einsum / bmm order)."""
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    sd = _state(fx)
    with torch.no_grad():
        enc = HO.wav_to_states(*case_wav(fx["main"]), sd, HYPERCONFORMER_22M)
        short = HO.wav_to_states(*case_wav(fx["short"]), sd, HYPERCONFORMER_22M)
    m = fx["main"]
    r_norm, _ = check_summary("hyperconformer_22M oracle", enc, m["frame_norm"], m["sample_idx"], m["sample_rows"], 2e-6)
    r_short = rel(short, fx["short"]["enc_out"])
    print(f"oracle vs reference: short utterance {r_short:.2e}")
    assert r_norm <= 1e-6 and r_short <= 1e-6


def _mirror(**kw):
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M as cfg
    args = dict(tgt_vocab=cfg["vocab"], input_size=640, d_model=cfg["d_model"], nhead=cfg["nhead"],
                num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=cfg["num_decoder_layers"], d_ffn=cfg["d_ffn"],
                activation=torch.nn.GELU, encoder_module="conformer", attention_type="hypermixing", normalize_before=True,
                causal=False)
    args.update(kw)
    return TransformerASR(**args)


def test_state_dict_layout_matches_reference(fx):
    ours = [(k, tuple(v.shape)) for k, v in _mirror().state_dict().items()]
    ref = [(k, tuple(s)) for k, s in fx["keys"]]
    assert sorted(ours) == sorted(ref), set(ours) ^ set(ref)


def test_shapes_table_matches_reference_parameters(fx):
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M as cfg
    from speechbrain_b200.utils.shapes import transformer_asr_shapes
    s = transformer_asr_shapes(cfg["vocab"], 640, cfg["d_model"], cfg["nhead"], cfg["num_encoder_layers"],
                               cfg["num_decoder_layers"], cfg["d_ffn"], 31, "hypermixing")
    ref = {k: tuple(v) for k, v in fx["keys"] if not k.endswith(".pe")}
    assert s == ref, set(s.items()) ^ set(ref.items())


def test_constructor_rejects_what_is_not_built():
    _mirror(num_encoder_layers=1, num_decoder_layers=1)
    _mirror(num_encoder_layers=1, d_model=512, nhead=8, d_ffn=2048)  # Conformer-L width: e = 64, k = 256
    for kw in (dict(d_model=144, nhead=8, d_ffn=1024),                   # hyperconformer_8M.yaml: head width 18
               dict(d_model=144, nhead=8, d_ffn=576),
               dict(d_model=256, nhead=8, d_ffn=1000),                   # k = 125
               dict(d_model=256, nhead=8, d_ffn=4096),                   # k = 512
               dict(d_model=288, nhead=8, d_ffn=1024),                   # head width 36
               dict(encoder_module="branchformer", csgu_linear_units=1536),  # the HyperBranchformer
               dict(output_hidden_states=True)):
        with pytest.raises(NotImplementedError):
            _mirror(**dict(dict(num_encoder_layers=1), **kw))


def test_encode_errors():
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _mirror(num_encoder_layers=1, num_decoder_layers=1)
    with pytest.raises(NotImplementedError):
        tr.encode(torch.zeros(1, 40, 640), dynchunktrain_config=DynChunkTrainConfig(8, 2))
    with pytest.raises(RuntimeError, match="3000"):  # the reference fails to broadcast its 3000-row table
        tr.encode(torch.zeros(1, 3001, 640))
    with pytest.raises(NotImplementedError):
        tr.make_streaming_context(DynChunkTrainConfig(8, 2))
    with pytest.raises(NotImplementedError):
        tr.encode_streaming(torch.zeros(1, 8, 640), None)


def test_reference_rejects_3001_frames(fx):
    assert fx["t3001_error"] == "RuntimeError"
    sd = _state(fx)
    with pytest.raises(RuntimeError):
        HO.encode(torch.zeros(1, 3001, 640), None, sd, dict(num_encoder_layers=1), "Transformer.")


def test_hypermixing_masks_padded_frames_and_uses_every_frame(fx):
    """Properties of the oracle's HyperMixing the device tests lean on: the values of padded frames do not reach valid
    frames, a padded frame's output is the LayerNorm's beta, and every valid frame changes every other frame's output."""
    sd = _state(fx)
    p = "Transformer.encoder.layers.0.mha_layer."
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 40, 256, generator=g)
    kpm = torch.zeros(2, 40, dtype=torch.bool)
    kpm[1, 25:] = True
    y = HO.hypermixing(x, sd, p, kpm)
    x2 = x.clone()
    x2[1, 25:] = 100.0 * torch.randn(15, 256, generator=g)
    y2 = HO.hypermixing(x2, sd, p, kpm)
    assert torch.equal(y[:, :25], y2[:, :25]) and torch.equal(y[0], y2[0])
    assert torch.allclose(y[1, 25:], sd[p + "layer_norm.bias"].expand(15, 256), atol=1e-6)
    x3 = x.clone()
    x3[0, 7] += 0.5
    y3 = HO.hypermixing(x3, sd, p, kpm)
    assert float((y3[0] - y[0]).abs().amax(dim=-1).min()) > 1e-4


YAML = """
sample_rate: 16000
n_fft: 400
n_mels: 80
d_model: 256
nhead: 8
num_encoder_layers: 2
num_decoder_layers: 1
d_ffn: 1024
transformer_dropout: 0.1
attention_type: hypermixing
encoder_module: conformer
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
    d_ffn: !ref <d_ffn>
    dropout: !ref <transformer_dropout>
    activation: !ref <activation>
    encoder_module: !ref <encoder_module>
    attention_type: !ref <attention_type>
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


def test_from_hparams_hyperconformer_recipe_layout(tmp_path):
    import sentencepiece as spm

    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M, seeded_asr_state
    cfg = dict(HYPERCONFORMER_22M, num_encoder_layers=2, num_decoder_layers=1, vocab=60)
    sd = seeded_asr_state(cfg, 0)
    tmp = write_pretrained_dir(tmp_path, YAML, dict(asr=module_list_ckpt(sd), normalizer=normalizer_ckpt(sd)))
    with open(os.path.join(tmp, "corpus.txt"), "w") as f:
        words = ["hyper", "mixing", "token", "conformer", "linear", "time", "network", "weights", "encoder", "decoder"]
        for i in range(400):
            f.write(" ".join(words[(i * 7 + j * 3) % len(words)] for j in range(9)) + f" {i % 13}\n")
    spm.SentencePieceTrainer.train(input=os.path.join(tmp, "corpus.txt"), model_prefix=os.path.join(tmp, "tok"), vocab_size=60,
                                   model_type="bpe", bos_id=1, eos_id=2, unk_id=0, pad_id=-1, minloglevel=2)
    os.rename(os.path.join(tmp, "tok.model"), os.path.join(tmp, "tokenizer.ckpt"))
    asr = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    tr = asr.transformer
    assert tr.attention_type == "hypermixing" and asr.mods["decoder"].model is tr
    key = "encoder.layers.1.mha_layer.hyper.w2_gen.fc2_weights"
    assert torch.equal(tr.state_dict()[key], sd["Transformer." + key])
    assert tr.engine_cfg()["attention_type"] == "hypermixing"


def test_fp16_operand_error_estimate(fx):
    """The oracle with every product's operands rounded to fp16 on the HyperConformer-22M input: the encoder error the device
    can be expected to show against the reference.  It is 3.2e-3 over all frames and up to 4.9e-3 over one utterance's
    valid frames, not <= 1e-3: the FFN / convolution modules alone give 1.4e-3 (ten layers of d_model 256 whose hypernetwork
    outputs are large), and HyperMixing alone 2.4e-3, because y = W2 GELU(H)^T sums k = 128 terms of magnitude |H| ~ 1e3
    into a per-frame value that its LayerNorm then rescales to unit size, so the rounding of G and W2 is amplified by that
    cancellation.  The device encoder bar is therefore 7.5e-3 (test_gpu_hyperconformer.py), 1.5x the worst estimate; this
    test pins the estimate that bar rests on."""
    from speechbrain_b200.utils.seeded_init import HYPERCONFORMER_22M
    sd = _state(fx)
    with torch.no_grad():
        enc = HO.wav_to_states(*case_wav(fx["main"]), sd, HYPERCONFORMER_22M, q=lambda t: t.half().float())
        ref = HO.wav_to_states(*case_wav(fx["main"]), sd, HYPERCONFORMER_22M)
    lens = fx["main"]["abs_len"]
    per_utt = [rel(enc[b, :int(lens[b])], ref[b, :int(lens[b])]) for b in range(ref.shape[0])]
    r = rel(enc, ref)
    print(f"fp16-operand oracle vs reference: encoder rel-L2 {r:.2e}, valid frames per utterance "
          f"{['%.2e' % x for x in per_utt]}")
    assert r <= 4e-3 and max(per_utt) <= 5.5e-3
