"""CPU checks of the transducer greedy-search fixture (tests/golden/transducer.pt, generator tools/make_transducer_golden.py):
the fp32 oracle (tests/transducer_oracle.py) equals the reference TransducerBeamSearcher on every case -- tokens identical,
score to 1e-6 -- and the mirrors keep the reference's state_dict keys and constructor checks."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import transducer_oracle as TO  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
FX = torch.load(os.path.join(ROOT, "tests", "golden", "transducer.pt"))


def case_inputs(case):
    J, H, V = TO.RECIPE_SIZES[case["recipe"]]
    blank = 0 if case["blank"] == "first" else V - 1
    W = TO.seeded_weights(case["seed"], J, H, V, blank)
    tn = TO.seeded_tn(case["seed"] + 1000, case["B"], case["T"], W)
    if case.get("suppress_blank"):
        W["transducer_lin.w.weight"][blank] = -50.0 / J ** 0.5
        tn = tn.abs()
    assert abs(float(tn.double().abs().sum()) - case["checksum"]) <= 1e-9 * case["checksum"], case["name"]
    return W, tn, blank


@pytest.mark.parametrize("case", FX["cases"], ids=[c["name"] for c in FX["cases"]])
def test_oracle_equals_reference(case):
    W, tn, blank = case_inputs(case)
    O = TO.Oracle(W)
    if "chunk" in case:   # chunked reference calls with the carried state == one oracle walk
        hyps, _, rows = O.batch(tn, blank, case["m"])
        assert hyps == case["tokens"]
        p, h, c = (torch.stack([r["state"][i] for r in rows]) for i in range(3))
        for got, ref in zip((p.norm(dim=-1), h.norm(dim=-1), c.norm(dim=-1)), case["state_norms"]):
            torch.testing.assert_close(got, ref.reshape(-1).float(), rtol=1e-5, atol=1e-6)
        return
    hyps, score, rows = O.batch(tn, blank, case["m"])
    assert hyps == case["tokens"]
    assert abs(float(score) - case["score"]) <= 1e-6 * max(1.0, abs(case["score"]))
    if case.get("suppress_blank"):
        assert all(len(h) == (case["m"] + 1) * case["T"] for h in hyps)


def test_fixture_has_varied_emissions():
    total = {0: 0, 1: 0, 2: 0}
    for c in FX["cases"]:
        for k, v in c["emission_hist"].items():
            total[k] += v
    assert all(v > 0 for v in total.values()), total
    assert any(c["m"] == 0 for c in FX["cases"]) and any(c["T"] == 1 for c in FX["cases"])


def test_state_dict_keys_match_reference():
    from speechbrain_b200.nnet.embedding import Embedding
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.RNN import LSTM
    mods = {"emb": Embedding(num_embeddings=1000, consider_as_one_hot=True, blank_id=0),
            "dec": LSTM(input_shape=[None, None, 999], hidden_size=512, num_layers=1),
            "proj_dec": Linear(input_size=512, n_neurons=640, bias=False),
            "transducer_lin": Linear(input_size=640, n_neurons=1000, bias=False)}
    for p, m in mods.items():
        assert sorted(m.state_dict()) == FX["keys"][p], p


@pytest.mark.parametrize("blank", [0, 3, 9])
def test_one_hot_embedding_matches_reference_construction(blank):
    from speechbrain_b200.nnet.embedding import Embedding
    e = Embedding(num_embeddings=10, consider_as_one_hot=True, blank_id=blank)
    assert e.embedding_dim == 9
    assert torch.equal(e.Embedding.weight, TO.one_hot_embedding(10, blank))


def test_lstm_without_input_size_raises_both_error_types():
    from speechbrain_b200.nnet.RNN import LSTM
    with pytest.raises(ValueError):
        LSTM(hidden_size=3)
    with pytest.raises(NotImplementedError):
        LSTM(hidden_size=3)


def test_constructor_checks():
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.nnet.embedding import Embedding
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.RNN import LSTM
    from speechbrain_b200.nnet.transducer.transducer_joint import Transducer_joint
    emb = Embedding(num_embeddings=512, consider_as_one_hot=True, blank_id=0)
    dec = [emb, LSTM(input_size=511, hidden_size=512), Linear(input_size=512, n_neurons=512, bias=False)]
    lin = [Linear(input_size=512, n_neurons=512, bias=False)]
    joint = Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU)
    s = TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=1, nbest=1)
    assert s.searcher == s.transducer_greedy_decode and s.builds == 0
    with pytest.raises(ValueError):
        TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=1, lm_weight=0.3)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec, joint, lin, blank_id=0, beam_size=4)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec[:2], joint, lin, blank_id=0, beam_size=1)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec, joint, [Linear(input_size=512, n_neurons=512, bias=True)], blank_id=0, beam_size=1)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher([emb, LSTM(input_size=511, hidden_size=512, num_layers=2), dec[2]], joint, lin, blank_id=0,
                               beam_size=1)
    with pytest.raises(NotImplementedError):
        Transducer_joint(joint="concat", nonlinearity=torch.nn.GELU)
    with pytest.raises(NotImplementedError):
        Transducer_joint(joint="sum")   # LeakyReLU, the reference default
    with pytest.raises(NotImplementedError):
        Transducer_joint(joint="sum", nonlinearity=lambda: torch.nn.GELU(approximate="tanh"))


def test_hparams_resolve_transducer_mirrors():
    from speechbrain_b200.utils.hparams import load_hyperpyyaml
    hp = load_hyperpyyaml("emb: !new:speechbrain.nnet.embedding.Embedding\n    num_embeddings: 8\n"
                          "    consider_as_one_hot: True\n    blank_id: 0\n"
                          "dec: !new:speechbrain.nnet.RNN.LSTM\n    input_shape: [null, null, 7]\n    hidden_size: 64\n"
                          "    num_layers: 1\n    re_init: True\n"
                          "Tjoint: !new:speechbrain.nnet.transducer.transducer_joint.Transducer_joint\n    joint: sum\n"
                          "    nonlinearity: !name:torch.nn.GELU\n")
    assert hp["dec"].rnn.input_size == 7 and hp["emb"].embedding_dim == 7 and hp["Tjoint"].joint == "sum"
