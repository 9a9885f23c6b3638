"""-m gpu tests of the Transformer recipes' device path: the 3-block front-end kernels against the fp32 oracle
(tests/transformer_oracle.py), the whole pipeline (Fbank -> CMVN -> CNN -> 12 regularMHA layers of 4 heads of 128 -> greedy
decode) against the reference outputs in tests/golden/transformer.pt, and the head_dim-128 decoder attention (self and
cross) through the teacher-forced decode (weight-streaming and wgmma decode paths) against the oracle, the recipe's
beam-10 test search with the CTC and TransformerLM scorers (the lineage-indexed beam step) against the reference, and a
from_hparams round trip of the recipe's module layout.

Front-end bar: rel-L2 <= 5e-4 (3.0e-4 measured: fp16 act1 and block-2 operands).  Encoder bar: rel-L2 <= 1e-3 (the
Conformer's).  Greedy: tokens identical up to the first decision whose reference top-1/top-2 margin is below 5e-3
(parity.check_greedy; the fixture keeps no chosen log-probs).  Beam: hypotheses identical, scores within 5e-2 (the rule of test_gpu_kernels.py's CTC+LM
beam test)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import (case_wav, check_alone_vs_batch, check_encoder, check_greedy, check_summary, dev,  # noqa: E402,F401
                    lm_scorer, module_list_ckpt, normalizer_ckpt, rel, write_pretrained_dir)
import transformer_oracle as TO  # noqa: E402
from mirrors import build_mirror, seeded  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ENC_BAR = 1e-3

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "transformer.pt"))


@pytest.fixture(scope="module")
def sd(fx):
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE
    return seeded(TRANSFORMER_LARGE, fx["weight_seed"])


def _mirror(sd):
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE
    return build_mirror(TRANSFORMER_LARGE, sd)


def _front_end(sd, dev):
    return _mirror(sd).cnn.to(dev)


@pytest.mark.parametrize("B,T0", [(2, 1001), (3, 1003), (1, 1002), (2, 5), (1, 6), (1, 7), (4, 37)])
def test_front_end_kernel_vs_oracle(dev, sd, B, T0):
    """T0 = 1001 is 10 s; 1003 / 1002 give T2 = 251 with a different tail tile; 5 frames is the shortest input the
    reference's 5x5 reflect padding accepts."""
    cnn = _front_end(sd, dev)
    g = torch.Generator().manual_seed(1000 + T0)
    feats = torch.randn(B, T0, 80, generator=g) * 2.0
    out = cnn(feats.to(dev)).cpu()
    ref = TO.cnn3(feats, sd)
    err = rel(out, ref)
    print(f"front-end B={B} T0={T0} -> {tuple(out.shape)}: rel-L2 {err:.2e}, max abs {(out - ref).abs().max():.2e}")
    assert out.shape == ref.shape and torch.isfinite(out).all() and err <= 5e-4
    assert torch.equal(out, cnn(feats.to(dev)).cpu())
    one = cnn(feats[-1:].to(dev)).cpu()  # batch independence
    assert torch.equal(one[0], out[-1])


def test_front_end_rejects_too_short(dev, sd):
    cnn = _front_end(sd, dev)
    with pytest.raises(RuntimeError, match="reflect"):
        cnn(torch.randn(1, 4, 80, device=dev))


def _engine(sd, dev, parts=("fbank", "cnn", "encoder", "decoder")):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE
    return AsrEngine(TRANSFORMER_LARGE, sd, device=dev, parts=parts)


def test_transformer_large_encoder_and_greedy(dev, fx, sd):
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE as cfg
    g = fx["large"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        ref = TO.encode(TO.wav_to_cnn(wav, lens, sd, cfg), lens, sd, cfg)
    check_summary("transformer_large oracle", ref, g["enc"]["frame_norm"], g["enc"]["sample_idx"], g["enc"]["sample_rows"], 1e-5)
    eng = _engine(sd, dev)
    S = g["greedy_tokens"].shape[1]
    pred, score, enc, done = eng.transcribe_greedy_dev(wav.to(dev), lens.to(dev), S, 1, 2, want_enc=True)
    torch.cuda.synchronize()
    check_encoder("transformer_large", enc.cpu(), ref, g["abs_len"], ENC_BAR)
    # the fixture keeps no chosen log-probs: tokens only
    check_greedy("transformer_large", pred.cpu(), None, g["greedy_tokens"], g["greedy_margin"], chosen_lp=None)
    check_alone_vs_batch(lambda w, ln: eng.encode_wav(w.to(dev), ln.to(dev)), wav, lens, 1e-5)


@pytest.mark.parametrize("n", [3, 72])
def test_head_dim_128_decoder_attention_teacher_forced(dev, sd, n):
    """TransformerASR.decode (self- and cross-attention at 4 heads of 128) against the oracle's decoder, on ragged
    encoder states: 3 rows run the weight-streaming decode path, 72 rows (>= 64) the wgmma one."""
    from oracle import asr_oracle as O
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE as cfg
    tr = _mirror(sd).tr
    g = torch.Generator().manual_seed(7 + n)
    T, S = 97, 11
    enc = torch.randn(n, T, 512, generator=g)
    tgt = torch.randint(3, 5000, (n, S), generator=g)
    tgt[:, 0] = 1
    enc_len = torch.randint(1, T + 1, (n,), generator=g).int()
    enc_len[0] = T
    out, _ = tr.to(dev).decode(tgt.to(dev), enc.to(dev), enc_len.to(dev))
    ref = O.decode(tgt, enc, enc_len, sd, cfg, "Transformer.")
    ref = ref[0] if isinstance(ref, tuple) else ref
    err = rel(out.cpu(), ref)
    print(f"decode head_dim 128: rel-L2 {err:.2e}")
    assert torch.isfinite(out).all() and err <= 2e-3


def _searcher(m, beam, max_decode_ratio, lm):
    """transformer.yaml's test search on the mirror m: beam, temperature 1.15, no EOS threshold, CTC 0.4 + TransformerLM
    0.6 (in that order)"""
    kwargs = dict(min_decode_ratio=0.0, beam_size=beam, temperature=1.15, using_eos_threshold=False, length_normalization=True)
    return m.searcher(kwargs, max_decode_ratio, scorers=dict(ctc=0.4, transformerlm=0.6), lm=lm)


def test_beam10_ctc_lm_matches_reference(dev, fx, sd):
    """The recipe's test search at beam 10 (40 live hypotheses: the beam step's lineage-indexed self-attention and the
    cross-attention at head width 128) on the reference's encoder states, recomputed by the oracle."""
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE as cfg
    g, gb = fx["large"], fx["beam10"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        enc = TO.encode(TO.wav_to_cnn(wav, lens, sd, cfg), lens, sd, cfg)
    assert gb["lm_seed"] == 1
    bs = _searcher(_mirror(sd), gb["kwargs"]["beam_size"], gb["max_decode_ratio"], lm_scorer())
    hyps, _, scores, _ = bs(enc.to(dev), lens.to(dev))
    print(f"[transformer_large beam10 ctc+lm] hyps equal {hyps == gb['hyps']}; score err "
          f"{(scores.cpu() - gb['scores']).abs().max():.2e}")
    assert hyps == gb["hyps"]
    assert (scores.cpu() - gb["scores"]).abs().max() < 5e-2


HPARAMS = """
d_model: 512
output_neurons: 5000
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
    d_model: 128
    nhead: 2
    num_encoder_layers: 2
    num_decoder_layers: 0
    d_ffn: 256
    dropout: 0.0
    activation: !name:torch.nn.GELU
    normalize_before: False
ctc_scorer: !new:speechbrain.decoders.scorer.CTCScorer
    eos_index: !ref <eos_index>
    blank_index: !ref <blank_index>
    ctc_fc: !ref <ctc_lin>
transformerlm_scorer: !new:speechbrain.decoders.scorer.TransformerLMScorer
    language_model: !ref <lm_model>
    temperature: 1.15
scorer: !new:speechbrain.decoders.scorer.ScorerBuilder
    full_scorers: [!ref <ctc_scorer>, !ref <transformerlm_scorer>]
    weights:
        ctc: 0.4
        transformerlm: 0.6
decoder: !new:speechbrain.decoders.S2STransformerBeamSearcher
    modules: [!ref <Transformer>, !ref <seq_lin>]
    bos_index: !ref <bos_index>
    eos_index: !ref <eos_index>
    min_decode_ratio: 0.0
    max_decode_ratio: 0.05
    beam_size: 10
    temperature: 1.15
    using_eos_threshold: False
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


def test_from_hparams_local_directory_round_trip(dev, fx, sd, tmp_path):
    """A pretrained-model directory with transformer.yaml's module layout (3-block CNN, Transformer encoder, ctc_lin,
    seq_lin, TransformerLM, beam search with the CTC and LM scorers) loads through from_hparams, the checkpoints land in the
    mirrors, and it transcribes like the same modules wired directly."""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    lm = TransformerLM(vocab=5000, d_model=128, nhead=2, num_encoder_layers=2, num_decoder_layers=0, d_ffn=256, dropout=0.0,
                       activation=torch.nn.GELU, normalize_before=False)
    lm.load_state_dict(seeded_state_dict(lm, seed=1))
    tmp = write_pretrained_dir(tmp_path, HPARAMS, dict(asr=module_list_ckpt(sd), lm=lm.state_dict(), normalizer=normalizer_ckpt(sd)))
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": str(dev)})
    # direct construction of the same layout
    m = _mirror(sd)
    direct = EncoderDecoderASR(modules=dict(encoder=m.front_end(), transformer=m.tr, decoder=_searcher(m, 10, 0.05, lm)),
                               hparams=dict(tokenizer=None, transformer_beam_search=True), run_opts={"device": str(dev)})
    assert torch.equal(loaded.mods["decoder"].fc.w.weight.cpu(), sd["seq_lin.w.weight"])
    wav, lens = case_wav(fx["large"])
    w1, t1 = loaded.transcribe_batch(wav, lens)
    w2, t2 = direct.transcribe_batch(wav, lens)
    print("from_hparams tokens", t1)
    assert t1 == t2 and len(t1) == 4 and sum(len(t) for t in t1) > 0
