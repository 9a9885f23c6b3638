"""CPU tests of the Loquacious Conformers (conformer_activation=torch.nn.GELU): the oracle of loquacious_oracle.py against
the reference outputs in tests/golden/loquacious.pt (generator: tools/make_loquacious_golden.py), the mirror's
state_dict keys against the reference's for all four recipe sizes, and which Conformer activations TransformerASR
accepts."""
import functools
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import loquacious_oracle as LO  # noqa: E402
from parity import check_summary  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loquacious.pt")
BAR = 1e-5  # the fp32 oracle against the fp32 reference


@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN)


def _mirror(cfg, **kw):
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    args = dict(input_size=cfg["input_size"], tgt_vocab=cfg["vocab"], d_model=cfg["d_model"], nhead=cfg["nhead"],
                num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=cfg["num_decoder_layers"],
                d_ffn=cfg["d_ffn"], activation=torch.nn.GELU, encoder_module="conformer", attention_type="RelPosMHAXL",
                normalize_before=True, causal=False, conformer_activation=torch.nn.GELU)
    args.update(kw)
    return TransformerASR(**args)


@functools.lru_cache(maxsize=1)
def _wav():
    return LO.waveforms()


def _check_enc(tag, cfg, rec, dynchunk=None):
    wav, lens = _wav()
    enc = LO.encode(cfg, LO.state(cfg), wav, lens, dynchunk)
    s = rec["enc"]
    check_summary(tag, enc, s["frame_norm"], s["sample_idx"], s["sample_rows"], BAR)


@pytest.mark.parametrize("name", ["loquacious_small", "loquacious_base", "loquacious_large", "loquacious_xlarge"])
def test_oracle_reduced(fx, name):
    """2 encoder layers of every size: the GELU oracle equals the reference"""
    _check_enc(name, LO.reduced(LO.sizes()[name]), fx["reduced"][name])


def test_oracle_dynchunk_and_rope(fx):
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_LARGE, LOQUACIOUS_SMALL
    _check_enc("large dynchunk", LO.reduced(LOQUACIOUS_LARGE), fx["dynchunk"], tuple(fx["dynchunk"]["chunk"]))
    _check_enc("small rope", LO.reduced(LOQUACIOUS_SMALL, attention_type="RoPEMHA"), fx["rope"])


def test_swish_oracle_differs(fx):
    """the fixture tells the activations apart: the Swish encoder misses it by far more than the bar"""
    cfg = LO.reduced(LO.sizes()["loquacious_base"])
    wav, lens = _wav()
    from oracle import asr_oracle as O
    feats = O.full_pipeline_features(wav, lens, LO.state(cfg), dict(cfg, win_length=25))
    enc = O.encode(feats, lens, LO.state(cfg), cfg, LO.PREFIX)
    s = fx["reduced"]["loquacious_base"]["enc"]
    idx = s["sample_idx"].long()
    err = float((enc[idx[:, 0], idx[:, 1]] - s["sample_rows"]).norm() / s["sample_rows"].norm())
    assert err > 1e-2, err


@pytest.mark.parametrize("name", ["loquacious_small", "loquacious_base", "loquacious_large", "loquacious_xlarge"])
def test_state_dict_keys(fx, name):
    """the mirror of each full-size recipe has the reference's keys and shapes"""
    cfg = LO.sizes()[name]
    got = [(k, tuple(v.shape)) for k, v in _mirror(cfg).state_dict().items()]
    assert sorted(got) == sorted(tuple(x) for x in fx["keys"][name])


def test_gelu_accepted():
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_XLARGE
    small = dict(LOQUACIOUS_XLARGE, num_encoder_layers=1, num_decoder_layers=1)
    for att in ("RelPosMHAXL", "RoPEMHA"):
        tr = _mirror(small, attention_type=att)
        assert tr.conformer_activation == "gelu" and tr.engine_cfg()["conformer_activation"] == "gelu"


@pytest.mark.parametrize("act", ["tanh_gelu", "Tanh", "ReLU", "LeakyReLU", "GELU_subclass", "Mish"])
def test_other_activations_rejected(act):
    from speechbrain_b200.utils.seeded_init import LOQUACIOUS_SMALL
    small = dict(LOQUACIOUS_SMALL, num_encoder_layers=1, num_decoder_layers=1)
    fn = {"tanh_gelu": functools.partial(torch.nn.GELU, approximate="tanh"),
          "GELU_subclass": type("GELU", (torch.nn.GELU,), {})}.get(act) or getattr(torch.nn, act)
    with pytest.raises(NotImplementedError, match="conformer_activation"):
        _mirror(small, conformer_activation=fn)


def test_swish_engine_cfg_unchanged():
    """a Swish Conformer's engine config is what it was before the activation became a setting, plus the new key"""
    from speechbrain_b200.nnet.activations import Swish
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE
    cfg = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=1)
    for act in (None, Swish, torch.nn.SiLU):
        ec = _mirror(cfg, attention_type="RoPEMHA", conformer_activation=act).engine_cfg()
        assert ec.pop("conformer_activation") == "swish"
        assert ec == dict(n_fft=400, hop=160, win=400, n_mels=80, cnn_channels=(64, 32), cnn_blocks=2, input_size=640,
                          d_model=512, nhead=8, num_encoder_layers=1, num_decoder_layers=1, d_ffn=2048, vocab=5000,
                          kernel_size=31, attention_type="RoPEMHA", decoder_activation="gelu", max_length=2500,
                          encoder_module="conformer", csgu_linear_units=3072, branchformer_activation="gelu")


def test_recipe_sizes():
    """seeded_init's configs carry the recipes' sizes, vocabularies and Fbank"""
    from speechbrain_b200.utils import seeded_init as S
    got = {n: (c["d_model"], c["nhead"], c["num_encoder_layers"], c["num_decoder_layers"], c["d_ffn"], c["vocab"], c["n_fft"])
           for n, c in LO.sizes().items()}
    assert got == {"loquacious_small": (256, 4, 12, 6, 1024, 1024, 400), "loquacious_base": (512, 8, 12, 6, 2048, 5120, 400),
                   "loquacious_large": (768, 12, 14, 6, 3072, 5120, 400),
                   "loquacious_xlarge": (1024, 16, 18, 6, 3072, 5120, 400)}
    assert (S.LOQUACIOUS_BLANK, S.LOQUACIOUS_BOS, S.LOQUACIOUS_EOS, S.LOQUACIOUS_PAD) == (3, 1, 2, 0)
