"""CPU checks of the transducer beam-search fixture (tests/golden/transducer_beam.pt, generator
tools/make_transducer_beam_golden.py): the fp32 oracle (tests/transducer_beam_oracle.py) equals the reference
TransducerBeamSearcher on every case -- identical n-best tokens, scores within 1e-5 -- its replay of its own pops changes
nothing, and the constructor refuses what the device search does not build before any device work."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import transducer_beam_oracle as BO  # noqa: E402
import transducer_oracle as TO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
FX = torch.load(os.path.join(ROOT, "tests", "golden", "transducer_beam.pt"))


def case_inputs(case):
    import make_transducer_beam_golden as MB
    W, tn, blank = MB.case_inputs(case)
    assert abs(float(tn.double().abs().sum()) - case["checksum"]) <= 1e-9 * case["checksum"], case["name"]
    return W, tn, blank


def run_case(case):
    W, tn, blank = case_inputs(case)
    return BO.BeamOracle(W).batch(tn, blank, case["beam"], case["nbest"], case["sb"], case["eb"]), W, tn, blank


@pytest.mark.parametrize("case", FX["cases"], ids=[c["name"] for c in FX["cases"]])
def test_oracle_equals_reference(case):
    (best, score, nb, nbs, rows), _, _, _ = run_case(case)
    assert nb == case["tokens"]
    for a, b in zip(nbs, case["scores"]):
        assert len(a) == len(b) and all(abs(x - y) <= 1e-5 for x, y in zip(a, b))
    assert [r["pops"] for r in rows] == case["pops"]
    assert abs(float(score) - case["score"]) <= 1e-5 * max(1.0, abs(case["score"]))


def test_replay_of_own_pops_agrees():
    case = next(c for c in FX["cases"] if c["name"] == "t17")
    W, tn, blank = case_inputs(case)
    O = BO.BeamOracle(W)
    for b in range(tn.shape[0]):
        walk = O.search(tn[b], blank, case["beam"], case["nbest"], case["sb"], case["eb"])
        rep = O.search(tn[b], blank, case["beam"], case["nbest"], case["sb"], case["eb"], replay=walk["trace"])
        assert rep["issues"] == [] and rep["hyps"] == walk["hyps"] and rep["scores"] == walk["scores"]
        assert [x[0] for x in rep["raw"]] == [r["score"] for r in walk["trace"]]


def test_fixture_covers_the_recipes():
    names = {c["name"]: c for c in FX["cases"]}
    assert names["librispeech"]["beam"] == 10 and names["librispeech"]["T"] == 251
    assert names["commonvoice_nbest"]["nbest"] == names["commonvoice_nbest"]["beam"] == 4
    assert any(c["T"] == 1 for c in FX["cases"]) and any(c["T"] == 17 for c in FX["cases"])
    assert FX["e2e"]["beam"] == 10 and len(FX["e2e"]["tokens"]) == 4
    # no frame of the fixture comes near the pop cap (4 * beam_size)
    assert all(c["max_pops_per_frame"] <= c["beam"] for c in FX["cases"] + [FX["e2e"]])


def _modules(V=512, H=512, J=512, blank=0):
    from speechbrain_b200.nnet.embedding import Embedding
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.RNN import LSTM
    from speechbrain_b200.nnet.transducer.transducer_joint import Transducer_joint
    emb = Embedding(num_embeddings=V, consider_as_one_hot=True, blank_id=blank)
    dec = [emb, LSTM(input_size=V - 1, hidden_size=H), Linear(input_size=H, n_neurons=J, bias=False)]
    return dec, Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU), [Linear(input_size=J, n_neurons=V, bias=False)]


def test_constructor_selects_beam_search():
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    dec, joint, lin = _modules()
    s = TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=10, nbest=1, state_beam=2.3, expand_beam=2.3)
    assert s.searcher == s.transducer_beam_search_decode and s.builds == 0
    g = TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=1, nbest=1)
    assert g.searcher == g.transducer_greedy_decode
    s = TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=32, nbest=32, lm_module=torch.nn.Identity(),
                               lm_weight=0.0)
    assert s.searcher == s.transducer_beam_search_decode and s.builds == 0


def test_constructor_refusals_before_device_work():
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    dec, joint, lin = _modules()
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=4, nbest=5)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=10, nbest=1, lm_module=torch.nn.Identity(),
                               lm_weight=0.5)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=33, nbest=1)
    with pytest.raises(ValueError):
        TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=10, nbest=1, lm_weight=0.5)
    small, joint, lin8 = _modules(V=8, H=64, J=64)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(small, joint, lin8, blank_id=0, beam_size=10, nbest=1)
    s = TransducerBeamSearcher(small, joint, lin8, blank_id=0, beam_size=8, nbest=1)
    assert s.builds == 0


def test_read_trace_layout():
    K = 3
    tr = torch.full((1, 4, 6 + 2 * K), -1, dtype=torch.int32)
    lp = torch.tensor([-0.5, -1.0, -2.0])
    tr[0, 0, :6] = torch.tensor([0, 2, 1, 1, 0b101, 0], dtype=torch.int32)
    tr[0, 0, 5] = torch.tensor([-3.25]).view(torch.int32)
    tr[0, 0, 6:6 + K] = torch.tensor([7, 0, 4], dtype=torch.int32)
    tr[0, 0, 6 + K:] = lp.view(torch.int32)
    (r,) = BO.BeamOracle.read_trace(tr, 0, K)
    assert r == dict(frame=2, hyp=1, ended=1, kept=0b101, score=-3.25, tokens=[7, 0, 4], logp=lp.tolist())
