"""CPU checks of the CTC prefix beam-search fixture (tests/golden/ctc_prefix_beam.pt, generator
tools/make_ctc_prefix_beam_golden.py): the NumPy oracle (tests/ctc_prefix_beam_oracle.py) equals the reference
CTCPrefixBeamSearcher's stored hypotheses on every case -- texts, text_frames and float64 score bits; the emulated CPython
set order equals real sets; the searcher's constructor and argument checks; the YAML names."""
import os
import random
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import ctc_beam_oracle as CO  # noqa: E402
import ctc_prefix_beam_oracle as PO  # noqa: E402
from make_ctc_prefix_beam_golden import case_inputs, oracle, vocab_of  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_cases():
    """[(fixture entry, log_probs, wav_lens, vocab)] with the inputs regenerated and checked against the stored checksum."""
    out = []
    for c in torch.load(os.path.join(GOLDEN, "ctc_prefix_beam.pt"))["cases"]:
        lp, lens = case_inputs(c)
        assert float(lp.double().abs().sum()) == c["checksum"], c["name"]
        out.append((c, lp, lens, vocab_of(c["vocab"])))
    return out


CASES = load_cases()


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0]["name"] for c in CASES])
def test_oracle_equals_reference(idx):
    c, lp, lens, vocab = CASES[idx]
    assert oracle(lp, lens, vocab, c["params"]) == [[(t, [(w, tuple(f)) for w, f in fr], s) for t, fr, s in hs]
                                                    for hs in c["hyps"]]


def test_fixture_covers_the_issue_cases():
    by = {c["name"]: c for c, _, _, _ in CASES}
    assert max(max(v) for v in by["recipe"]["live"] if v) == 100                     # the beam fills
    assert by["defaults"]["params"] == dict(blank_index=0, topk=5)                   # history pruning, -10 / -5
    assert all(len(h) > 1 for h in by["defaults"]["hyps"][:4])
    assert all(n == 0 for v in by["t1"]["live"] for n in v[1:])
    assert [len(v) for v in by["t1"]["live"]] == [1, 0, 0]                           # T = 1, a 0-frame utterance
    assert by["blank_last"]["params"]["blank_index"] == 30
    assert CASES[[c["name"] for c, _, _, _ in CASES].index("wide")][1].shape[2] == 40
    tied = [h[2] for hs in by["ties"]["hyps"] for h in hs]
    assert len(tied) > len(set(tied))                                                 # exact float ties between texts


def _real_order(above, am, nv):
    s = set(np.array(above, dtype=np.int64)) | {np.int64(am)}
    return [int(v) for v in s & set(range(nv))]


@pytest.mark.parametrize("V", [31, 257, 5000, 8192])
def test_candidate_order_matches_cpython_sets(V):
    rng = random.Random(V)
    non_ascending = 0
    for _ in range(2000):
        k = rng.choice([0, 1, 2, 3, 4, 5, 8, 13, 30, 64, 200])
        above = sorted(rng.sample(range(V), min(k, V)))
        am = rng.randrange(V) if rng.random() < 0.3 or not above else rng.choice(above)
        nv = V if rng.random() < 0.7 else rng.randrange(1, V + 1)
        got = PO.candidate_order(above, am, nv)
        assert got == _real_order(above, am, nv), (V, above, am, nv)
        non_ascending += got != sorted(got)
    if V > 31:
        assert non_ascending > 0
    assert PO.candidate_order([3, 10, 17, 4099], 3, 5000) == [3, 17, 10, 4099]


def test_range_set_iterates_in_ascending_order():
    """candidate_order walks set(range(n)) in ascending order: every v sits in slot v for every n up to 8192."""
    s = PO.PySetEmu()
    for n in range(8192):
        s.add(n)
        if n in (0, 30, 256, 4999, 8191):
            assert list(s) == list(range(n + 1))


def test_constructor_and_arguments():
    from speechbrain_b200.decoders.ctc import CTCBaseSearcher, CTCBeamSearcher, CTCPrefixBeamSearcher
    s = CTCPrefixBeamSearcher(blank_index=0, vocab_list=CO.CHAR_VOCAB)
    assert isinstance(s, CTCBaseSearcher) and not isinstance(s, CTCBeamSearcher)
    assert (s.beam_size, s.beam_prune_logp, s.token_prune_min_logp, s.prune_history, s.topk, s.space_index) == \
        (100, -10.0, -5.0, True, 1, 1)
    assert s.blank_skip_threshold == 0.0 and not s.is_spm
    assert CTCPrefixBeamSearcher(blank_index=0, vocab_list=CO.spm_vocab(60, 0)).is_spm
    with pytest.raises(NotImplementedError, match="KenLM"):
        CTCPrefixBeamSearcher(blank_index=0, vocab_list=CO.CHAR_VOCAB, kenlm_model_path="lm.arpa")
    with pytest.raises(ValueError, match="beam_size"):
        CTCPrefixBeamSearcher(blank_index=0, vocab_list=CO.CHAR_VOCAB, beam_size=257)
    with pytest.raises(RuntimeError, match="CUDA"):
        s(CO.synthetic_log_probs(5, 2, 20, 31), torch.ones(2))
    with pytest.raises(NotImplementedError, match="lm_start_state"):
        s(CO.synthetic_log_probs(5, 2, 20, 31), torch.ones(2), lm_start_state=object())
    # pieces with whitespace are hashed per part: a history key of any text is supported
    CTCPrefixBeamSearcher(blank_index=0, vocab_list=["<b>", "a b", " ", "c"], prune_history=True)


def test_yaml_names_resolve():
    from speechbrain_b200.decoders.ctc import CTCPrefixBeamSearcher
    from speechbrain_b200.utils.hparams import resolve_name
    assert resolve_name("speechbrain.decoders.CTCPrefixBeamSearcher") is CTCPrefixBeamSearcher
    assert resolve_name("speechbrain.decoders.ctc.CTCPrefixBeamSearcher") is CTCPrefixBeamSearcher
