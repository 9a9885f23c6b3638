"""CPU restatement of the AISHELL-1 Transformer recipe's front-end and encoder: ConvolutionFrontEnd(num_blocks=2,
num_layers_per_block=1, out_channels=(256, 256), kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
(oracle/asr_oracle.py's cnn_frontend, which the Conformer recipes' (64, 32) front-end shares) and TransformerASR.encode with
encoder_module="transformer", attention_type="regularMHA" at d_model 256 and 4 heads (tests/transformer_oracle.py).  It
runs in the dtype of its input, float64 for the kernel tests.  Test infrastructure only: tools/make_aishell_golden.py
asserts that it equals the running reference."""
import torch

from oracle import asr_oracle as O
import transformer_oracle as TO

encode = TO.encode


def cnn(feats, sd, prefix="CNN."):
    """feats [B, T0, F0] -> [B, T2, F2, 256], computed in feats' dtype (the weights are cast to it)"""
    w = {k: v.to(feats.dtype) for k, v in sd.items() if k.startswith(prefix)}
    return O.cnn_frontend(feats, w, prefix, num_blocks=2)


def wav_to_cnn(wav, wav_lens, sd, cfg):
    """Fbank -> global InputNormalization -> the 256-channel front-end."""
    f = O.fbank(wav, n_fft=cfg["n_fft"], n_mels=cfg["n_mels"], win_length_ms=cfg["win"] * 1000 // cfg["sample_rate"])
    f = O.input_norm(f, wav_lens, "global", sd["normalize.glob_mean"], sd["normalize.glob_std"])
    return cnn(f, sd)
