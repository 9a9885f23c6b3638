"""-m gpu tests of the device CTC prefix beam search (speechbrain_b200.decoders.ctc.CTCPrefixBeamSearcher,
csrc/ctc_prefix_beam.cu) against the reference CTCPrefixBeamSearcher's hypotheses stored in tests/golden/ctc_prefix_beam.pt
and against the NumPy oracle (tests/ctc_prefix_beam_oracle.py), plus EncoderASR with the searcher (Branchformer CTC
recipe, a sentencepiece model through from_hparams).

Comparison rule: texts and text_frames identical at every rank; scores within 1e-8 or two float32 ulps of the score.  The
scores are float64 on both sides, but the reference folds p_nb + p and p_b + p in float32 (NumPy 2 casts the Python float
to the float32 log-prob), where CUDA's expf / log1pf may differ from the host libm by one float32 ulp.  Folding the
float64 sums in float32 instead moves the scores by more than that on most fixture cases."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401
import ctc_beam_oracle as CO  # noqa: E402
from test_ctc_prefix_beam_golden import CASES, oracle  # noqa: E402

pytestmark = pytest.mark.gpu
RECIPE = dict(blank_index=0, beam_size=100, beam_prune_logp=-12.0, token_prune_min_logp=-1.2, prune_history=False)
DEFAULTS = dict(blank_index=0, topk=5)


def tuples(hyps):
    return [[(h.text, [(w, (int(a), int(b))) for w, (a, b) in h.text_frames], h.score) for h in hs] for hs in hyps]


def check(tag, ref, ours):
    """Identical texts and frames at every rank, scores within max(1e-8, 2 float32 ulps) -> the worst score difference."""
    assert len(ref) == len(ours), tag
    worst = 0.0
    for b, (hr, ho) in enumerate(zip(ref, ours)):
        assert [(h[0], [(w, tuple(f)) for w, f in h[1]]) for h in hr] == [(h[0], h[1]) for h in ho], (tag, b)
        for r, (x, y) in enumerate(zip(hr, ho)):
            d = 0.0 if float(x[2]) == float(y[2]) else abs(float(x[2]) - float(y[2]))   # -inf scores too
            assert d <= max(1e-8, 2 * float(np.spacing(np.float32(abs(float(x[2])))))), (tag, b, r, x[2], y[2])
            worst = max(worst, d)
    return worst


def run(dev, vocab, params, lp, lens):
    from speechbrain_b200.decoders.ctc import CTCPrefixBeamSearcher
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return tuples(CTCPrefixBeamSearcher(vocab_list=vocab, **params)(lp.to(dev), lens.to(dev)))


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0]["name"] for c in CASES])
def test_device_matches_reference(dev, idx):
    c, lp, lens, vocab = CASES[idx]
    ours = run(dev, vocab, c["params"], lp, lens)
    worst = check(c["name"], c["hyps"], ours)
    assert all(isinstance(h[2], float) for hs in ours for h in hs)
    print(f"[{c['name']}] identical texts and frames; worst score difference {worst:.2e}")


def test_exact_ties_keep_order(dev):
    c, lp, lens, vocab = next(x for x in CASES if x[0]["name"] == "ties")
    ours = run(dev, vocab, c["params"], lp, lens)
    assert [[(h[0], [(w, tuple(f)) for w, f in h[1]], h[2]) for h in hs] for hs in c["hyps"]] == ours


@pytest.mark.parametrize("setting", ["recipe", "defaults"])
def test_batch32_and_long_utterance(dev, setting):
    params = RECIPE if setting == "recipe" else DEFAULTS
    lp = CO.synthetic_log_probs(401, 32, 251, 31)
    lens = torch.linspace(1.0, 0.6, 32)
    check(f"32x251 {setting}", oracle(lp, lens, CO.CHAR_VOCAB, params), run(dev, CO.CHAR_VOCAB, params, lp, lens))
    lp = CO.synthetic_log_probs(402, 1, 3000, 31)
    lens = torch.ones(1)
    ours = run(dev, CO.CHAR_VOCAB, params, lp, lens)
    check(f"T=3000 {setting}", oracle(lp, lens, CO.CHAR_VOCAB, params), ours)
    assert len(ours[0][0][0]) > 500


def test_batch_invariance_and_reruns(dev):
    c, lp, lens, vocab = CASES[0]
    params = dict(c["params"], topk=10)
    full = run(dev, vocab, params, lp, lens)
    assert full == run(dev, vocab, params, lp, lens)   # reruns: identical texts, frames and score bits
    for b in (0, 3, 7):
        assert run(dev, vocab, params, lp[b:b + 1], lens[b:b + 1])[0] == full[b]
    pad = torch.cat([CO.synthetic_log_probs(7, 2, 251, 31), lp[3:4]], 0)
    assert run(dev, vocab, params, pad, torch.tensor([1.0, 1.0, float(lens[3])]))[2] == full[3]


def test_input_validation(dev):
    from speechbrain_b200.decoders.ctc import CTCPrefixBeamSearcher
    s = CTCPrefixBeamSearcher(vocab_list=CO.CHAR_VOCAB, **RECIPE)
    lp = CO.synthetic_log_probs(5, 2, 20, 31)
    with pytest.raises(ValueError, match="float32"):
        s(lp.double().to(dev), torch.ones(2))
    with pytest.raises(ValueError, match="8192"):
        CTCPrefixBeamSearcher(vocab_list=["x"] * 8193, blank_index=0)(torch.zeros(1, 2, 8193, device=dev))
    with pytest.raises(ValueError, match="blank_index"):
        CTCPrefixBeamSearcher(vocab_list=CO.CHAR_VOCAB, blank_index=31)(lp.to(dev))
    # a frame whose arg-max lies outside vocab_list and no other token passes: no candidate, every beam steps to -inf
    bad = torch.full((1, 3, 31), -30.0)
    bad[0, :, 30] = 0.0
    short = CO.CHAR_VOCAB[:25]
    check("no candidate", oracle(bad, torch.ones(1), short, RECIPE), run(dev, short, RECIPE, bad, torch.ones(1)))


@pytest.mark.parametrize("setting", ["recipe", "defaults"])
def test_encoder_asr_branchformer_prefix_beam(dev, setting):
    from test_gpu_ctc_beam import _branchformer_ctc_asr

    from speechbrain_b200.decoders.ctc import CTCPrefixBeamSearcher
    params = RECIPE if setting == "recipe" else DEFAULTS
    asr, wav, lens = _branchformer_ctc_asr(dev, CTCPrefixBeamSearcher, dict(test_beam_search=dict(params)))
    assert isinstance(asr.decoding_function, CTCPrefixBeamSearcher)
    words, hyps = asr.transcribe_batch(wav, lens)
    lp = asr.encode_batch(wav, lens).cpu()
    ours = tuples(hyps)
    assert words == [h[0][0] for h in ours]
    check(f"EncoderASR {setting} vs oracle on the device log-posteriors", oracle(lp, lens, CO.CHAR_VOCAB, params), ours)
    print(f"[EncoderASR branchformer prefix {setting}] {words}")


def test_encoder_asr_sentencepiece_from_hparams(dev, tmp_path):
    from test_gpu_ctc_beam import SPM_YAML
    from test_hparams_loader import _make_dir

    from speechbrain_b200.decoders.ctc import CTCPrefixBeamSearcher
    from speechbrain_b200.inference.ASR import EncoderASR
    tmp = str(tmp_path)
    _make_dir(tmp, n_enc=2, n_dec=2, vocab=60)
    yaml = SPM_YAML.replace("<save_dir>", tmp).replace("speechbrain.decoders.ctc.CTCBeamSearcher",
                                                       "speechbrain.decoders.CTCPrefixBeamSearcher")
    with open(os.path.join(tmp, "ctc.yaml"), "w") as f:
        f.write(yaml)
    asr = EncoderASR.from_hparams(source=tmp, hparams_file="ctc.yaml", run_opts={"device": str(dev)})
    s = asr.decoding_function
    assert isinstance(s, CTCPrefixBeamSearcher) and s.is_spm and s.beam_size == 10 and s.topk == 3
    g = torch.Generator().manual_seed(11)
    wav = torch.randn(3, 32000, generator=g)
    lens = torch.tensor([1.0, 0.8, 0.6])
    words, hyps = asr.transcribe_batch(wav, lens)
    lp = asr.encode_batch(wav, lens).cpu()
    params = dict(blank_index=0, beam_size=10, topk=3)
    check("spm EncoderASR vs oracle", oracle(lp, lens, s.vocab_list, params), tuples(hyps))
    direct = EncoderASR(modules=dict(asr.mods), hparams=dict(tokenizer=asr.tokenizer, decoding_function=CTCPrefixBeamSearcher,
                                                             test_beam_search=dict(params)), run_opts={"device": str(dev)})
    w2, h2 = direct.transcribe_batch(wav, lens)
    assert w2 == words and tuples(h2) == tuples(hyps)
    print(f"[spm EncoderASR prefix] {words}")
