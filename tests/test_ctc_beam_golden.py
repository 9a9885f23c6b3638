"""CPU checks of the CTC beam-search fixture (tests/golden/ctc_beam.pt, generator tools/make_ctc_beam_golden.py): the
NumPy oracle (tests/ctc_beam_oracle.py) equals the reference CTCBeamSearcher's stored hypotheses on every case -- texts
and text_frames identical, scores bit-equal -- and the searcher mirror's constructor keeps the reference's semantics."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ctc_beam_oracle as CO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def fixture_cases():
    """(case entry, log_probs, wav_lens, vocab) for every fixture case, inputs regenerated and checksummed."""
    fx = torch.load(os.path.join(GOLDEN, "ctc_beam.pt"))
    bf = torch.load(os.path.join(GOLDEN, "branchformer.pt"))["ctc"]
    spm = CO.spm_vocab(5000, 0)
    out = []
    for c in fx["cases"]:
        if "gen" in c:
            g = dict(c["gen"])
            lp = CO.synthetic_log_probs(g.pop("seed"), g.pop("B"), g.pop("T"), g.pop("V"), **g)
        elif "tied" in c:
            lp = CO.tied_log_probs(**c["tied"])
        else:
            lp = bf["log_probs"].float()
        assert abs(float(lp.double().abs().sum()) - c["checksum"]) <= 1e-9 * c["checksum"], c["name"]
        out.append((c, lp, torch.tensor(c["lens"], dtype=torch.float32), CO.CHAR_VOCAB if c["vocab"] == "char" else spm))
    return out


CASES = fixture_cases()


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0]["name"] for c in CASES])
def test_oracle_equals_reference(idx):
    c, lp, lens, vocab = CASES[idx]
    kw = {k: v for k, v in c["params"].items() if k != "blank_index"}
    ora = CO.as_tuples(CO.decode(lp, lens, vocab, c["params"]["blank_index"], **kw))
    for b, (hr, ho) in enumerate(zip(c["hyps"], ora)):
        assert len(hr) == len(ho)
        for r, (x, y) in enumerate(zip(hr, ho)):
            assert (x[0], [tuple(f) for f in x[1]]) == (y[0], y[1]), (c["name"], b, r)
            assert np.float32(x[2]) == np.float32(y[2]), (c["name"], b, r)


def test_fixture_exercises_the_search():
    by = {c["name"]: c for c, _, _, _ in CASES}
    assert max(max(v) for v in by["recipe"]["live"]) == 100 and sum(map(sum, by["recipe"]["merges"])) > 0
    assert sum(map(sum, by["spm"]["merges"])) > 0 and sum(map(sum, by["branchformer_defaults"]["merges"])) > 0
    assert by["t1"]["hyps"][1] == [("", [], 0.0)]                        # the 0-frame utterance
    assert [int(x) for x in (251 * torch.tensor(by["recipe"]["lens"])).numpy().astype(int)][1] == 225   # truncation
    assert any(len(h) > 1 for h in by["defaults"]["hyps"])                # topk 5
    tied = by["ties"]["hyps"][0]                                           # exact ties decided by position order
    assert len(tied) == 10 and len({h[2] for h in tied}) < len(tied)


def test_frame_lengths_truncate_like_the_reference():
    assert CO.frame_lengths(251, torch.tensor([0.9, 1.0, 0.0]), 3) == [225, 251, 0]
    assert CO.frame_lengths(10, torch.tensor([1.5, -0.2]), 2) == [10, 8]   # used as a slice bound


def test_searcher_constructor_semantics():
    from speechbrain_b200.decoders.ctc import CTCBeamSearcher
    s = CTCBeamSearcher(blank_index=0, vocab_list=CO.CHAR_VOCAB, beam_size=100, beam_prune_logp=-12, token_prune_min_logp=-1.2,
                        prune_history=False)
    assert not s.is_spm and s.space_index == 1 and s.blank_skip_threshold == 0.0 and s.topk == 1
    info = s._info.numpy()
    assert info[0, 0] == 1 and info[1, 0] == 3 and info[2].tolist() == [0, 2, 1]   # blank, space, plain "E"
    sp = CTCBeamSearcher(blank_index=0, vocab_list=CO.spm_vocab(64, 0))
    assert sp.is_spm and sp._info[1].tolist() == [2, 1, 0]                          # bare "▁": word start, empty string
    assert sp._info[10, 1] == 3 and sp._info[3, 1] == 3                             # duplicated "b": one string id
    with pytest.raises(NotImplementedError):
        CTCBeamSearcher(blank_index=0, vocab_list=CO.CHAR_VOCAB, kenlm_model_path="lm.bin")
    with pytest.raises(ValueError):
        CTCBeamSearcher(blank_index=0, vocab_list=CO.CHAR_VOCAB, beam_size=257)
    with pytest.raises(RuntimeError, match="CUDA"):
        s(torch.zeros(1, 3, 31), torch.ones(1))
