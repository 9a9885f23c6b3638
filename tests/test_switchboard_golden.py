"""CPU tests of the Switchboard transformer.yaml recipe's mirrors against tests/golden/switchboard.pt (generator:
tools/make_switchboard_golden.py, which runs the reference): the fp32 LM oracle (tests/switchboard_oracle.py) reproduces
the reference's TransformerLM.forward, the mirrors expose the reference's state_dict keys and shapes, TransformerLM
accepts d_embedding only for the Switchboard LM's shape, and the other LM head widths still raise."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import switchboard_oracle as SO  # noqa: E402

from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM  # noqa: E402
from speechbrain_b200.utils.seeded_init import SWITCHBOARD_LM, SWITCHBOARD_TRANSFORMER, seeded_state_dict  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "switchboard.pt"))


def _lm(**kw):
    return TransformerLM(**dict(SWITCHBOARD_LM, activation=torch.nn.ReLU, **kw))


def test_lm_oracle_equals_reference(fx):
    g = fx["lm"]
    sd = seeded_state_dict(_lm(), seed=g["seed"])
    tokens, lens = g["tokens"], g["lengths"]
    valid = torch.arange(tokens.shape[1]).unsqueeze(0) < lens.unsqueeze(1)
    assert tokens.shape[0] >= 6 and ((tokens == 0) & valid).sum() >= 3
    with torch.no_grad():
        logits = SO.lm_forward(tokens, sd)
    assert logits.shape == (tokens.shape[0], tokens.shape[1], 2000) and torch.isfinite(logits).all()
    assert (logits.logsumexp(-1) - g["logsumexp"]).abs().max() < 1e-4
    top_v, top_i = logits.topk(8, dim=-1)
    assert (top_v - g["top_values"]).abs().max() < 1e-4
    sure = (g["top_values"][..., 0] - g["top_values"][..., 1]) >= 5e-3
    assert torch.equal(top_i[..., 0][sure], g["top_ids"][..., 0][sure].long())
    idx = g["sample_idx"].long()
    sample = logits[idx[:, 0], idx[:, 1]]
    assert float((sample - g["sample_logits"]).norm() / g["sample_logits"].norm()) < 1e-5


def test_state_dict_keys_match_reference(fx):
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    assert sorted((k, tuple(v.shape)) for k, v in _lm().state_dict().items()) == sorted(fx["keys"]["lm"])
    c = SWITCHBOARD_TRANSFORMER
    tr = TransformerASR(input_size=c["input_size"], tgt_vocab=c["vocab"], d_model=c["d_model"], nhead=c["nhead"],
                        num_encoder_layers=c["num_encoder_layers"], num_decoder_layers=c["num_decoder_layers"],
                        d_ffn=c["d_ffn"], activation=torch.nn.GELU, encoder_module="transformer",
                        attention_type="regularMHA", normalize_before=True, causal=False,
                        positional_encoding="fixed_abs_sine")
    assert sorted((k, tuple(v.shape)) for k, v in tr.state_dict().items()) == sorted(fx["keys"]["transformer"])
    ec = tr.engine_cfg()
    assert (ec["cnn_channels"], ec["cnn_blocks"], ec["input_size"]) == ((64, 64), 3, 1280)


def test_lm_engine_config():
    assert _lm().engine_cfg() == dict(d_model=264, nhead=12, num_encoder_layers=12, d_ffn=1024, activation="relu")


@pytest.mark.parametrize("kw", [dict(d_embedding=64), dict(d_embedding=None), dict(d_embedding=264),
                                dict(nhead=11, d_model=264), dict(d_model=256, nhead=4),
                                dict(d_model=768, nhead=12, d_embedding=128), dict(normalize_before=True)])
def test_d_embedding_only_for_the_switchboard_shape(kw):
    with pytest.raises(NotImplementedError):
        _lm(**kw)


@pytest.mark.parametrize("d_model,nhead", [(264, 8), (264, 6), (288, 12), (384, 12), (512, 16), (640, 8)])
def test_other_head_widths_raise(d_model, nhead):
    with pytest.raises(NotImplementedError):
        TransformerLM(vocab=100, d_model=d_model, nhead=nhead, num_encoder_layers=1, d_ffn=256)
