"""-m gpu tests of what sbk_asr_create rejects (csrc/asr_weights.cu): a state_dict with a required tensor missing, or with
one of the wrong element count, fails with an error that names the key, for every part of a model and every encoder family;
the optional tensors stay optional; a failed create leaves the process able to create."""
import os
import pytest
import sys
import torch

from speechbrain_b200.engine import AsrEngine
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, TRANSFORMER_LARGE, seeded_asr_state, seeded_tensor
from speechbrain_b200.utils.shapes import transformer_lm_shapes

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401

pytestmark = pytest.mark.gpu
LM = dict(d_model=128, nhead=2, num_encoder_layers=1, d_ffn=256)
SMALL = dict(d_model=128, nhead=2, d_ffn=256, num_encoder_layers=1, num_decoder_layers=1, vocab=50, max_length=64)
CONFIGS = {
    "conformer_rope": dict(CONFORMER_LARGE, **SMALL),
    "conformer_relpos": dict(CONFORMER_LARGE, **SMALL, attention_type="RelPosMHAXL"),
    "hyperconformer": dict(CONFORMER_LARGE, **SMALL, attention_type="hypermixing"),
    "branchformer": dict(CONFORMER_LARGE, **SMALL, attention_type="RelPosMHAXL", encoder_module="branchformer",
                         csgu_linear_units=64),
    "transformer": dict(TRANSFORMER_LARGE, **SMALL),  # with the 3-block front-end
    "lm": dict(CONFORMER_LARGE, **SMALL, lm=LM),
}
CONFIGS["hyperconformer"]["nhead"] = 4  # HyperMixing heads of 32 channels
LAYER = "Transformer.encoder.layers.0."
# (configuration, a tensor its loader requires)
REQUIRED = [
    ("conformer_rope", "CNN.convblock_1.convs.conv_0.conv.weight"),  # 2-block front-end
    ("transformer", "CNN.convblock_2.reduce_conv.conv.conv.weight"),  # 3-block front-end
    ("conformer_rope", LAYER + "convolution_module.bottleneck.0.weight"),
    ("conformer_rope", LAYER + "mha_layer.in_proj_weight"),
    ("conformer_relpos", LAYER + "mha_layer.linear_pos.weight"),
    ("hyperconformer", LAYER + "mha_layer.hyper.w2_gen.fc2_weights"),
    ("branchformer", LAYER + "convolution_branch.csgu.conv.conv.weight"),
    ("branchformer", LAYER + "merge_proj.bias"),
    ("transformer", LAYER + "self_att.att.in_proj_bias"),
    ("transformer", "Transformer.encoder.norm.norm.weight"),
    ("conformer_rope", "Transformer.decoder.layers.0.multihead_attn.att.in_proj_weight"),
    ("conformer_rope", "Transformer.decoder.norm.norm.bias"),
    ("conformer_rope", "seq_lin.w.bias"),
    ("conformer_rope", "ctc_lin.w.bias"),
    ("lm", "lm.encoder.layers.0.self_att.att.in_proj_weight"),
    ("lm", "lm.output_proj.layers.2.w.weight"),
]


def _state(name):
    cfg = CONFIGS[name]
    sd = seeded_asr_state(cfg, 0)
    if "lm" in cfg:
        for k, shp in transformer_lm_shapes(cfg["vocab"], LM["d_model"], LM["nhead"], LM["num_encoder_layers"], LM["d_ffn"]).items():
            sd["lm." + k] = seeded_tensor(1, "lm." + k, shp)
    return sd


def _create(name, sd, dev):
    parts = ("fbank", "cnn", "encoder", "decoder") + (("lm",) if "lm" in CONFIGS[name] else ())
    return AsrEngine(CONFIGS[name], sd, device=dev, parts=parts)


@pytest.mark.parametrize("name,key", REQUIRED)
def test_missing_tensor_is_named(dev, name, key):
    sd = _state(name)
    del sd[key]
    with pytest.raises(RuntimeError, match="missing weight") as err:
        _create(name, sd, dev)
    assert f"'{key}'" in str(err.value)


@pytest.mark.parametrize("name,key", REQUIRED)
def test_wrong_element_count_is_named(dev, name, key):
    sd = _state(name)
    n = sd[key].numel()
    sd[key] = torch.zeros(n + 1)
    with pytest.raises(RuntimeError, match=f"has {n + 1} elements, expected {n}") as err:
        _create(name, sd, dev)
    assert f"'{key}'" in str(err.value)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_optional_tensors_may_be_absent(dev, name):
    sd = _state(name)
    for k in ("seq_lin.w.weight", "seq_lin.w.bias", "ctc_lin.w.weight", "ctc_lin.w.bias", "normalize.glob_mean",
              "normalize.glob_std"):
        del sd[k]
    eng = _create(name, sd, dev)
    cfg = CONFIGS[name]
    src = torch.randn(2, 40, cfg["input_size"], generator=torch.Generator().manual_seed(0)).to(dev)
    assert torch.isfinite(eng.encode_from_cnn(src)).all()


def test_create_after_a_failed_create(dev):
    sd = _state("lm")
    src = torch.randn(2, 40, CONFIGS["lm"]["input_size"], generator=torch.Generator().manual_seed(0)).to(dev)
    ref = _create("lm", sd, dev).encode_from_cnn(src)
    bad = dict(sd)
    del bad["lm.encoder.norm.norm.weight"]  # one of the last tensors the loader reads
    with pytest.raises(RuntimeError, match="lm.encoder.norm.norm.weight"):
        _create("lm", bad, dev)
    assert torch.equal(_create("lm", sd, dev).encode_from_cnn(src), ref)
