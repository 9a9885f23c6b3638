"""-m gpu tests of the device CTC beam search (speechbrain_b200.decoders.ctc.CTCBeamSearcher, csrc/ctc_beam.cu) against
the reference CTCBeamSearcher's hypotheses stored in tests/golden/ctc_beam.pt and against the NumPy oracle
(tests/ctc_beam_oracle.py), plus EncoderASR with the searcher (Branchformer CTC recipe, a sentencepiece model, from_hparams).

Comparison rule: at every rank whose reference score is at least 1e-3 away from both neighbours the texts and
text_frames are identical; inside a closer group ours is one of the group's texts.  Scores agree to 1e-4 + 1e-6 |score|
(the device folds merged scores with the same float32 formula as np.logaddexp, with CUDA's expf / log1pf)."""
import functools
import os
import sys
import warnings

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401
import branchformer_oracle as BO  # noqa: E402
import ctc_beam_oracle as CO  # noqa: E402
from mirrors import build_mirror  # noqa: E402
from test_ctc_beam_golden import CASES  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECIPE = dict(blank_index=0, beam_size=100, beam_prune_logp=-12.0, token_prune_min_logp=-1.2, prune_history=False)
DEFAULTS = dict(blank_index=0, topk=5)


def _tuples(hyps):
    return CO.as_tuples(hyps)


def check_hyps(tag, ref, ours, score_tol=True):
    """ref, ours: [[(text, text_frames, score)]] -> number of near-tie ranks met."""
    assert len(ref) == len(ours), tag
    near = 0
    for b, (hr, ho) in enumerate(zip(ref, ours)):
        assert len(hr) == len(ho), (tag, b, len(hr), len(ho))
        sc = [float(h[2]) for h in hr]
        for r, (x, y) in enumerate(zip(hr, ho)):
            gap = min([abs(sc[r] - sc[q]) for q in (r - 1, r + 1) if 0 <= q < len(sc)] or [np.inf])
            if gap >= 1e-3:
                assert (x[0], [tuple(f) for f in x[1]]) == (y[0], [tuple(f) for f in y[1]]), (tag, b, r, x[0], y[0])
            else:
                near += 1
                group = [h[0] for h in hr if abs(float(h[2]) - sc[r]) < 1e-3]
                assert y[0] in group, (tag, b, r, y[0], group)
            if score_tol:
                assert abs(float(y[2]) - sc[r]) <= 1e-4 + 1e-6 * abs(sc[r]), (tag, b, r, float(y[2]), sc[r])
    return near


def _oracle(lp, lens, vocab, params):
    kw = {k: v for k, v in params.items() if k != "blank_index"}
    return CO.as_tuples(CO.decode(lp, lens, vocab, params["blank_index"], **kw))


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0]["name"] for c in CASES])
def test_device_matches_reference_and_oracle(dev, idx):
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    c, lp, lens, vocab = CASES[idx]
    s = CTCBeamSearcher(vocab_list=vocab, **c["params"])
    ours = _tuples(s(lp.to(dev), lens.to(dev)))
    n1 = check_hyps(c["name"] + " vs reference", c["hyps"], ours)
    n2 = check_hyps(c["name"] + " vs oracle", _oracle(lp, lens, vocab, c["params"]), ours)
    print(f"[{c['name']}] equal to the reference and the oracle (near-tie ranks {n1}, {n2}); best {[h[0][0][:30] for h in ours if h]}")


def test_exact_ties_keep_position_order(dev):
    """Bit-identical scores between different texts: the survivors and their order follow the candidate position (the
    reference's stable heapq.nlargest), so here texts, frames and scores must equal the oracle's and the reference's exactly."""
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    c, lp, lens, vocab = next(x for x in CASES if x[0]["name"] == "ties")
    ours = _tuples(CTCBeamSearcher(vocab_list=vocab, **c["params"])(lp.to(dev), lens.to(dev)))
    assert ours == _oracle(lp, lens, vocab, c["params"])
    assert [[(h[0], [tuple(f) for f in h[1]]) for h in hs] for hs in c["hyps"]] == [[(h[0], h[1]) for h in hs] for hs in ours]


@pytest.mark.parametrize("setting", ["recipe", "defaults"])
def test_batch32_and_long_utterance(dev, setting):
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    params = RECIPE if setting == "recipe" else DEFAULTS
    s = CTCBeamSearcher(vocab_list=CO.CHAR_VOCAB, **params)
    lp = CO.synthetic_log_probs(201, 32, 251, 31)
    lens = torch.linspace(1.0, 0.3, 32)
    check_hyps(f"32x251 {setting}", _oracle(lp, lens, CO.CHAR_VOCAB, params), _tuples(s(lp.to(dev), lens.to(dev))))
    lp = CO.synthetic_log_probs(202, 1, 3000, 31)
    lens = torch.ones(1)
    ours = _tuples(s(lp.to(dev), lens.to(dev)))
    check_hyps(f"T=3000 {setting}", _oracle(lp, lens, CO.CHAR_VOCAB, params), ours)
    assert len(ours[0][0][0]) > 500


def test_batch_invariance_and_reruns(dev):
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    c, lp, lens, vocab = CASES[0]
    s = CTCBeamSearcher(vocab_list=vocab, **dict(c["params"], topk=10))
    full = _tuples(s(lp.to(dev), lens.to(dev)))
    assert full == _tuples(s(lp.to(dev), lens.to(dev)))   # reruns: identical texts, frames and score bits
    for b in (0, 3, 7):
        assert _tuples(s(lp[b:b + 1].to(dev), lens[b:b + 1].to(dev)))[0] == full[b]
    # the same utterance inside a batch padded with other utterances (longer beams elsewhere, more candidates per frame)
    pad = torch.cat([CO.synthetic_log_probs(7, 2, 251, 31), lp[3:4]], 0)
    assert _tuples(s(pad.to(dev), torch.tensor([1.0, 1.0, float(lens[3])]).to(dev)))[2] == full[3]


def test_input_validation(dev):
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    s = CTCBeamSearcher(vocab_list=CO.CHAR_VOCAB, **RECIPE)
    lp = CO.synthetic_log_probs(5, 2, 20, 31)
    with pytest.raises(RuntimeError, match="CUDA"):
        s(lp, torch.ones(2))
    with pytest.raises(ValueError, match="float32"):
        s(lp.double().to(dev), torch.ones(2))
    with pytest.raises(ValueError):
        CTCBeamSearcher(vocab_list=CO.CHAR_VOCAB, blank_index=0, beam_size=257)
    with pytest.raises(ValueError, match="8192"):
        CTCBeamSearcher(vocab_list=["x"] * 8193, blank_index=0, prune_history=False)(torch.zeros(1, 2, 8193, device=dev))
    with pytest.raises(ValueError, match="blank_index"):
        CTCBeamSearcher(vocab_list=CO.CHAR_VOCAB, blank_index=31)(lp.to(dev))
    with pytest.raises(NotImplementedError):
        s(lp.to(dev), torch.ones(2), lm_start_state=object())
    # log-probs wider than vocab_list: the reference warns and drops the extra columns
    short = CO.CHAR_VOCAB[:25]
    s2 = CTCBeamSearcher(vocab_list=short, **RECIPE)
    lp = CO.synthetic_log_probs(5, 2, 20, 31, active=list(range(25)))   # arg-max always inside vocab_list
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        ours = _tuples(s2(lp.to(dev), torch.ones(2).to(dev)))
    assert any("Vocab size mismatch" in str(x.message) for x in w)
    check_hyps("vocab 25 of 31", _oracle(lp, torch.ones(2), short, RECIPE), ours)
    # a frame whose arg-max lies outside vocab_list and no other token passes: the reference fails (max of nothing)
    bad = torch.full((1, 3, 31), -30.0)
    bad[0, :, 30] = 0.0
    with pytest.raises(ValueError):
        s2(bad.to(dev))


# ------------------------------------------------------------------------------------------- EncoderASR
class _LabelEncoder:
    """The ind2lab part of a CTCTextEncoder (what EncoderASR reads the beam searcher's vocab_list from)."""

    def __init__(self, labels):
        self.ind2lab = dict(enumerate(labels))

    def decode_ids(self, ids):
        return "".join(self.ind2lab[i] for i in ids)


def _branchformer_ctc_asr(dev, decoding_function, hparams_extra):
    from speechbrain_b200.inference.ASR import EncoderASR
    from speechbrain_b200.utils.seeded_init import BRANCHFORMER_CTC as cfg
    fx = torch.load(os.path.join(GOLDEN, "branchformer.pt"))
    m = build_mirror(cfg, BO.state(cfg, fx))
    enc = m.front_end(m.ctc_lin)
    hp = dict(tokenizer=_LabelEncoder(CO.CHAR_VOCAB), decoding_function=decoding_function, **hparams_extra)
    c = fx["ctc"]
    B, L = c["wav_shape"]
    g = torch.Generator().manual_seed(c["wav_seed"])
    wav = torch.randn(B, L, generator=g)
    for b in range(B):
        wav[b, int(round(float(c["wav_lens"][b]) * L)):] = 0
    return EncoderASR(modules=dict(encoder=enc), hparams=hp, run_opts={"device": str(dev)}), wav, c["wav_lens"]


@pytest.mark.parametrize("setting", ["recipe", "defaults"])
def test_encoder_asr_branchformer_ctc_beam(dev, setting):
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    params = RECIPE if setting == "recipe" else DEFAULTS
    asr, wav, lens = _branchformer_ctc_asr(dev, CTCBeamSearcher, dict(test_beam_search=dict(params)))
    assert isinstance(asr.decoding_function, CTCBeamSearcher) and asr.decoding_function.beam_size == params.get("beam_size", 100)
    words, hyps = asr.transcribe_batch(wav, lens)
    lp = asr.encode_batch(wav, lens).cpu()
    ours = _tuples(hyps)
    assert words == [h[0][0] for h in ours]
    check_hyps(f"EncoderASR {setting} vs oracle on the device log-posteriors", _oracle(lp, lens, CO.CHAR_VOCAB, params), ours)
    ref = next(c for c, _, _, _ in CASES if c["name"] == f"branchformer_{setting}")["hyps"]
    # the reference ran on its own log-posteriors (device ones differ by up to 2e-2): texts under the near-tie rule
    check_hyps(f"EncoderASR {setting} vs reference", ref, ours, score_tol=False)
    print(f"[EncoderASR branchformer {setting}] {words}")


def test_encoder_asr_rejects_other_tokenizers_and_keeps_greedy(dev):
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher, ctc_greedy_decode
    asr, wav, lens = _branchformer_ctc_asr(dev, functools.partial(ctc_greedy_decode, blank_id=0), {})
    assert not asr.beam_search
    with pytest.raises(ValueError, match="sentencepiece or CTCTextEncoder"):
        type(asr)(modules=dict(asr.mods), hparams=dict(tokenizer=None, decoding_function=CTCBeamSearcher))


SPM_YAML = """
n_mels: 80
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
    tgt_vocab: 60
    d_model: 512
    nhead: 8
    num_encoder_layers: 2
    num_decoder_layers: 2
    d_ffn: 2048
    activation: !name:torch.nn.GELU
    encoder_module: conformer
    attention_type: RoPEMHA
    normalize_before: True
    causal: False
ctc_lin: !new:speechbrain.nnet.linear.Linear
    input_size: 512
    n_neurons: 60
seq_lin: !new:speechbrain.nnet.linear.Linear
    input_size: 512
    n_neurons: 60
log_softmax: !new:speechbrain.nnet.activations.Softmax
    apply_log: True
tokenizer: !new:sentencepiece.SentencePieceProcessor
compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: 16000
    n_fft: 512
    n_mels: 80
    win_length: 32
Tencoder: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
    transformer: !ref <Transformer>
encoder: !new:speechbrain.nnet.containers.LengthsCapableSequential
    input_shape: [null, null, !ref <n_mels>]
    compute_features: !ref <compute_features>
    normalize: !ref <normalizer>
    cnn: !ref <CNN>
    transformer_encoder: !ref <Tencoder>
    ctc_lin: !ref <ctc_lin>
    log_softmax: !ref <log_softmax>
decoding_function: !name:speechbrain.decoders.ctc.CTCBeamSearcher
test_beam_search:
    blank_index: 0
    beam_size: 10
    topk: 3
asr_model: !new:torch.nn.ModuleList
    - [!ref <CNN>, !ref <Transformer>, !ref <seq_lin>, !ref <ctc_lin>]
modules:
    encoder: !ref <encoder>
pretrainer: !new:speechbrain.utils.parameter_transfer.Pretrainer
    loadables:
        normalizer: !ref <normalizer>
        asr: !ref <asr_model>
        tokenizer: !ref <tokenizer>
    paths:
        asr: <save_dir>/asr.ckpt
"""


def test_encoder_asr_sentencepiece_and_from_hparams(dev, tmp_path):
    from test_hparams_loader import _make_dir

    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    from speechbrain_b200.inference.ASR import EncoderASR
    tmp = str(tmp_path)
    _make_dir(tmp, n_enc=2, n_dec=2, vocab=60)
    with open(os.path.join(tmp, "ctc.yaml"), "w") as f:
        f.write(SPM_YAML.replace("<save_dir>", tmp))
    asr = EncoderASR.from_hparams(source=tmp, hparams_file="ctc.yaml", run_opts={"device": str(dev)})
    s = asr.decoding_function
    assert isinstance(s, CTCBeamSearcher) and s.is_spm and s.beam_size == 10 and s.topk == 3 and len(s.vocab_list) == 60
    g = torch.Generator().manual_seed(11)
    wav = torch.randn(3, 32000, generator=g)
    lens = torch.tensor([1.0, 0.8, 0.6])
    words, hyps = asr.transcribe_batch(wav, lens)
    lp = asr.encode_batch(wav, lens).cpu()
    params = dict(blank_index=0, beam_size=10, topk=3)
    check_hyps("spm EncoderASR vs oracle", _oracle(lp, lens, s.vocab_list, params), _tuples(hyps))
    # direct construction with the same modules and hyperparameters
    direct = EncoderASR(modules=dict(asr.mods), hparams=dict(tokenizer=asr.tokenizer, decoding_function=CTCBeamSearcher,
                                                             test_beam_search=dict(params)), run_opts={"device": str(dev)})
    w2, h2 = direct.transcribe_batch(wav, lens)
    assert w2 == words and _tuples(h2) == _tuples(hyps)
    print(f"[spm EncoderASR] {words}")
