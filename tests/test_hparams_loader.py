"""from_hparams / HyperPyYAML-subset loader / Pretrainer mirror (SURVEY 8f N1): an inference ``hyperparams.yaml`` written
the way speechbrain/asr-conformer-transformerlm-librispeech writes it -- ``speechbrain.*`` dotted names, ``!ref`` aliases,
``pretrainer`` with loadables -- is loaded from a LOCAL directory into this package's mirrors, the checkpoints land in the
modules, and (GPU test) the interface transcribes like the directly constructed one."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import module_list_ckpt, normalizer_ckpt, write_pretrained_dir  # noqa: E402

YAML = """
# Feature parameters
sample_rate: 16000
n_fft: 512
n_mels: 80
win_length: 32

# Transformer
d_model: 512
nhead: 8
num_encoder_layers: {n_enc}
num_decoder_layers: {n_dec}
d_ffn: 2048
transformer_dropout: 0.1
activation: !name:torch.nn.GELU
output_neurons: {vocab}

blank_index: 0
bos_index: 1
eos_index: 2
min_decode_ratio: 0.0
max_decode_ratio: 1.0
test_beam_size: 4
lm_weight: 0.60
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
    encoder_module: conformer
    attention_type: RoPEMHA
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
    max_decode_ratio: {max_ratio}
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

# training-only entries of a recipe file must not be touched by the lazy loader
speed_perturb: !new:speechbrain.augment.time_domain.SpeedPerturb
    orig_freq: !ref <sample_rate>

pretrainer: !new:speechbrain.utils.parameter_transfer.Pretrainer
    loadables:
        normalizer: !ref <normalizer>
        asr: !ref <asr_model>
        tokenizer: !ref <tokenizer>
    paths:
        asr: !ref <save_dir>/asr.ckpt
"""


def _make_dir(tmp, n_enc=1, n_dec=1, vocab=60, max_ratio=0.2):
    """A pretrained-model directory: hyperparams.yaml + asr.ckpt (reference key layout: ModuleList index prefixes) +
    normalizer.ckpt + tokenizer.ckpt (a tiny sentencepiece model trained here)."""
    import sentencepiece as spm

    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    cfg = dict(CONFORMER_LARGE, num_encoder_layers=n_enc, num_decoder_layers=n_dec, vocab=vocab)
    sd = seeded_asr_state(cfg, 0)
    txt = os.path.join(tmp, "corpus.txt")
    with open(txt, "w") as f:
        words = ["speech", "brain", "blackwell", "tensor", "memory", "conformer", "encoder", "decoder", "beam", "search", "greedy",
                 "filterbank", "mel", "frame", "token", "kernel", "cluster", "barrier", "stream", "graph", "hypothesis", "score"]
        for i in range(400):
            f.write(" ".join(words[(i * 7 + j * 3) % len(words)] for j in range(9)) + f" {i % 13}\n")
    spm.SentencePieceTrainer.train(input=txt, model_prefix=os.path.join(tmp, "tok"), vocab_size=vocab, model_type="bpe",
                                   bos_id=1, eos_id=2, unk_id=0, pad_id=-1, minloglevel=2)
    os.rename(os.path.join(tmp, "tok.model"), os.path.join(tmp, "tokenizer.ckpt"))
    write_pretrained_dir(tmp, YAML.format(n_enc=n_enc, n_dec=n_dec, vocab=vocab, max_ratio=max_ratio),
                         dict(asr=module_list_ckpt(sd), normalizer=normalizer_ckpt(sd)))
    return cfg, sd


def test_from_hparams_builds_and_loads(tmp_path):
    from speechbrain_b200.decoders.seq2seq import S2STransformerBeamSearcher
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    tmp = str(tmp_path)
    cfg, sd = _make_dir(tmp)
    asr = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    assert isinstance(asr.mods["encoder"], LengthsCapableSequential) and isinstance(asr.mods["decoder"], S2STransformerBeamSearcher)
    tr, dec = asr.transformer, asr.mods["decoder"]
    assert dec.model is tr and dec.beam_size == 4 and dec.ctc_weight == pytest.approx(0.4)
    # the checkpoint landed in the mirrors (asr.ckpt -> ModuleList [CNN, Transformer, seq_lin, ctc_lin]; normalizer; tokenizer)
    assert torch.equal(tr.state_dict()["encoder.layers.0.mha_layer.in_proj_weight"], sd["Transformer.encoder.layers.0.mha_layer.in_proj_weight"])
    assert torch.equal(asr.cnn.state_dict()["convblock_1.convs.conv_0.conv.weight"], sd["CNN.convblock_1.convs.conv_0.conv.weight"])
    assert torch.equal(dec.fc.w.weight, sd["seq_lin.w.weight"]) and torch.equal(dec.ctc_scorer.ctc_fc.w.bias, sd["ctc_lin.w.bias"])
    assert torch.equal(asr.normalize.glob_mean, sd["normalize.glob_mean"]) and asr.normalize.count == 1
    assert asr.tokenizer.get_piece_size() == 60 and asr.tokenizer.decode_ids([5, 6]) is not None
    assert asr.fbank.n_fft == 512 and asr.fbank.win_length == 512 and asr.hparams["tokenizer"] is asr.tokenizer


def test_hparams_subset_semantics():
    from speechbrain_b200.utils.hparams import load_hyperpyyaml
    hp = load_hyperpyyaml("a: 3\nb: !ref <a> * 2 + 1\nc: !ref <d>/x.ckpt\nd: /tmp\nt: (1, 2)\n"
                          "lin: !new:speechbrain.nnet.linear.Linear\n    input_size: !ref <a>\n    n_neurons: 4\n"
                          "two: [!ref <lin>, !ref <lin>]\ncp: !copy <lin>\nf: !name:torch.nn.functional.relu\n"
                          "bad: !new:speechbrain.nnet.RNN.LSTM\n    hidden_size: 3\n", overrides={"a": 5})
    assert hp["a"] == 5 and hp["b"] == 11 and hp["c"] == "/tmp/x.ckpt" and hp["t"] == (1, 2)
    assert hp["two"][0] is hp["lin"] and hp["two"][1] is hp["lin"] and hp["cp"] is not hp["lin"]
    assert hp["lin"].w.in_features == 5 and hp["f"] is torch.nn.functional.relu
    with pytest.raises(NotImplementedError):
        hp["bad"]


@pytest.mark.gpu
def test_from_hparams_transcribes_like_direct_construction(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import bench
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    tmp = str(tmp_path)
    cfg, sd = _make_dir(tmp, n_enc=2, n_dec=2, vocab=60, max_ratio=0.2)
    asr = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    g = torch.Generator().manual_seed(11)
    wav = torch.randn(3, 32000, generator=g)
    lens = torch.tensor([1.0, 0.8, 0.6])
    words, toks = asr.transcribe_batch(wav, lens)
    ref = bench.build_product_asr(cfg, sd, torch.device("cuda:0"), decoder="beam", beam=4, ctc=True)
    ref.mods["decoder"].max_decode_ratio = 0.2
    w2, t2 = ref.transcribe_batch(wav, lens)
    print("from_hparams tokens", toks, "words", words)
    assert toks == t2 and len(words) == 3 and all(isinstance(w, str) for w in words)
