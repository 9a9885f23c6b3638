"""CPU tests of the Transformer recipes' front-end and encoder mirrors against tests/golden/transformer.pt (generator:
tools/make_transformer_golden.py, which runs the reference): the fp32 oracle (tests/transformer_oracle.py) reproduces the
reference's stored outputs, the mirrors expose the reference's state_dict keys, and the configurations that are not
built still raise."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import case_wav, check_summary, rel  # noqa: E402
import transformer_oracle as TO  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "transformer.pt"))


def test_oracle_equals_reference(fx):
    from speechbrain_b200.utils.seeded_init import TRANSFORMER_LARGE as cfg, seeded_asr_state
    sd = seeded_asr_state(cfg, fx["weight_seed"])
    g = fx["large"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        cnn = TO.wav_to_cnn(wav, lens, sd, cfg)
        enc = TO.encode(cnn, lens, sd, cfg)
    assert cnn.shape == (4, 251, 20, 64) and enc.shape == (4, 251, 512)
    for name, x in (("cnn", cnn.flatten(2)), ("enc", enc)):
        check_summary(f"transformer_large oracle {name}", x, g[name]["frame_norm"], g[name]["sample_idx"], g[name]["sample_rows"], 1e-5)
    s = fx["short"]
    w5, l5 = case_wav(s)
    assert rel(TO.wav_to_cnn(w5, l5, sd, cfg), s["cnn"]) <= 1e-5


def test_state_dict_keys_match_reference(fx):
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    cnn = ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=3, num_layers_per_block=1, out_channels=(64, 64, 64),
                              kernel_sizes=(5, 5, 1), strides=(2, 2, 1), residuals=(False, False, True))
    assert [(k, tuple(v.shape)) for k, v in cnn.state_dict().items()] == fx["keys"]["cnn"]
    tr = TransformerASR(input_size=1280, tgt_vocab=5000, d_model=512, nhead=4, num_encoder_layers=12, num_decoder_layers=6,
                        d_ffn=2048, activation=torch.nn.GELU, encoder_module="transformer", attention_type="regularMHA",
                        normalize_before=True, causal=False, positional_encoding="fixed_abs_sine")
    assert sorted((k, tuple(v.shape)) for k, v in tr.state_dict().items()) == sorted(fx["keys"]["transformer"])


@pytest.mark.parametrize("kw", [
    dict(attention_type="RelPosMHAXL"), dict(attention_type="RoPEMHA"), dict(attention_type="hypermixing"),
    dict(normalize_before=False), dict(causal=True), dict(d_model=512, nhead=16), dict(positional_encoding=None)])
def test_transformer_encoder_unbuilt_configurations_raise(kw):
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    args = dict(input_size=1280, tgt_vocab=5000, d_model=512, nhead=4, num_encoder_layers=2, num_decoder_layers=1,
                d_ffn=2048, activation=torch.nn.GELU, encoder_module="transformer", attention_type="regularMHA",
                normalize_before=True, causal=False)
    args.update(kw)
    with pytest.raises(NotImplementedError):
        TransformerASR(**args)


def test_branchformer_and_conformer_with_regular_mha_raise():
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    for module in ("branchformer", "conformer"):
        with pytest.raises(NotImplementedError):
            TransformerASR(input_size=640, tgt_vocab=5000, d_model=512, nhead=8, num_encoder_layers=2, num_decoder_layers=1,
                           encoder_module=module, attention_type="regularMHA", normalize_before=True, causal=False)


@pytest.mark.parametrize("kw", [
    dict(kernel_sizes=(5, 5, 3)), dict(strides=(2, 2, 2)), dict(residuals=(False, False, False)),
    dict(out_channels=(64, 64, 128)), dict(num_layers_per_block=2)])
def test_other_three_block_front_ends_raise(kw):
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    args = dict(input_shape=(8, 10, 80), num_blocks=3, num_layers_per_block=1, out_channels=(64, 64, 64),
                kernel_sizes=(5, 5, 1), strides=(2, 2, 1), residuals=(False, False, True))
    args.update(kw)
    with pytest.raises(NotImplementedError):
        ConvolutionFrontEnd(**args)
