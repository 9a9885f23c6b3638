"""CPU tests of the AISHELL-1 Transformer recipe's front-end and encoder mirrors against tests/golden/aishell_transformer.pt
(generator: tools/make_aishell_golden.py, which runs the reference): the oracle (tests/aishell_oracle.py) reproduces the
reference's stored outputs, the mirrors expose the reference's state_dict keys, the encoder alone picks the 256-channel
front-end for its 5120-wide input, and the 2-block configurations that are not built still raise."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import case_wav, check_summary, rel  # noqa: E402
import aishell_oracle as AO  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CNN_KW = dict(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1, out_channels=(256, 256), kernel_sizes=(3, 3),
              strides=(2, 2), residuals=(False, False))
TR_KW = dict(input_size=5120, tgt_vocab=5000, d_model=256, nhead=4, num_encoder_layers=12, num_decoder_layers=6, d_ffn=2048,
             activation=torch.nn.GELU, encoder_module="transformer", attention_type="regularMHA", normalize_before=True,
             causal=False)


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "aishell_transformer.pt"))


def test_oracle_equals_reference(fx):
    from speechbrain_b200.utils.seeded_init import AISHELL_TRANSFORMER as cfg, seeded_asr_state
    sd = seeded_asr_state(cfg, fx["weight_seed"])
    g = fx["large"]
    wav, lens = case_wav(g)
    with torch.no_grad():
        cnn = AO.wav_to_cnn(wav, lens, sd, cfg)
        enc = AO.encode(cnn, lens, sd, cfg)
    assert cnn.shape == (4, 251, 20, 256) and enc.shape == (4, 251, 256)
    for name, x in (("cnn", cnn.flatten(2)), ("enc", enc)):
        check_summary(f"aishell oracle {name}", x, g[name]["frame_norm"], g[name]["sample_idx"], g[name]["sample_rows"], 1e-5)
    s = fx["short"]
    w3, l3 = case_wav(s)
    assert rel(AO.wav_to_cnn(w3, l3, sd, cfg), s["cnn"]) <= 1e-5


def test_state_dict_keys_match_reference(fx):
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    cnn = ConvolutionFrontEnd(**CNN_KW)
    assert [(k, tuple(v.shape)) for k, v in cnn.state_dict().items()] == fx["keys"]["cnn"]
    tr = TransformerASR(**TR_KW, positional_encoding="fixed_abs_sine")
    assert sorted((k, tuple(v.shape)) for k, v in tr.state_dict().items()) == sorted(fx["keys"]["transformer"])


def test_encoder_alone_pairs_with_the_256_channel_front_end():
    """TransformerASR's own engine config (used when no front-end module is wired) follows its input width: 5120 = 20 x 256
    is AISHELL-1's 2-block front-end, 1280 = 20 x 64 the LibriSpeech recipes' 3-block one"""
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    ec = TransformerASR(**dict(TR_KW, num_encoder_layers=1, num_decoder_layers=1)).engine_cfg()
    assert (ec["cnn_channels"], ec["cnn_blocks"], ec["input_size"]) == ((256, 256), 2, 5120)
    ec = TransformerASR(**dict(TR_KW, input_size=1280, d_model=512, num_encoder_layers=1, num_decoder_layers=1)).engine_cfg()
    assert (ec["cnn_channels"], ec["cnn_blocks"]) == ((64, 64), 3)


@pytest.mark.parametrize("kw", [dict(out_channels=(128, 32)), dict(out_channels=(256, 128)), dict(num_layers_per_block=2),
                                dict(kernel_sizes=(5, 5)), dict(residuals=(False, True))])
def test_other_two_block_front_ends_raise(kw):
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    with pytest.raises(NotImplementedError):
        ConvolutionFrontEnd(**dict(CNN_KW, **kw))
