"""Deterministic, order-independent synthetic weights keyed by state_dict name.

There is no network in this project (no checkpoints), so parity tests, goldens and
the benchmark all run on seeded random weights.  The reference module and ours
share state_dict keys (SURVEY.md 8b), so the same dict loads into both.
Values depend only on (seed, key, shape) -- not on parameter creation order.
"""
import hashlib
import math

import torch


def _gen(seed: int, key: str) -> torch.Generator:
    h = hashlib.sha256(f"{seed}:{key}".encode()).digest()
    g = torch.Generator(device="cpu")
    g.manual_seed(int.from_bytes(h[:7], "little"))
    return g


def seeded_tensor(seed: int, key: str, shape, kind: str = "auto") -> torch.Tensor:
    shape = tuple(shape)
    g = _gen(seed, key)
    if kind == "auto":
        if key.endswith("glob_std"):
            kind = "std"
        elif key.endswith("glob_mean"):
            kind = "mean"
        elif key.endswith(".weight") and (len(shape) == 1 or key.endswith("norm.weight")):
            kind = "gain"
        elif len(shape) >= 2:
            kind = "matrix"
        else:
            kind = "bias"
    if kind == "gain":  # LayerNorm gains around 1
        return 1.0 + 0.1 * torch.randn(shape, generator=g)
    if kind == "bias":
        return 0.05 * torch.randn(shape, generator=g)
    if kind == "std":
        return 0.5 + torch.rand(shape, generator=g)
    if kind == "mean":
        return torch.randn(shape, generator=g)
    # xavier-normal-like for matrices / conv kernels
    rf = 1
    for s in shape[2:]:
        rf *= s
    fan_in, fan_out = shape[1] * rf, shape[0] * rf
    std = math.sqrt(2.0 / (fan_in + fan_out))
    return std * torch.randn(shape, generator=g)


def seeded_state_dict(module_or_state_dict, seed: int = 0):
    """Return {key: tensor} of seeded values for every float entry of a module's
    state_dict (non-float buffers and sinusoid tables are left untouched)."""
    sd = module_or_state_dict.state_dict() if hasattr(module_or_state_dict, "state_dict") else module_or_state_dict
    out = {}
    for k, v in sd.items():
        if not torch.is_floating_point(v) or k.endswith(".pe") or k.endswith("inv_freq"):
            out[k] = v.clone()
            continue
        out[k] = seeded_tensor(seed, k, v.shape).to(v.dtype)
    return out


def seeded_asr_state(cfg, seed: int = 0):
    """Full flat state for the recipe's modules (CNN., Transformer., seq_lin., ctc_lin.) plus fixed global-CMVN
    statistics (normalize.glob_mean / glob_std), exactly as oracle/make_goldens.py gave the reference."""
    from .shapes import asr_model_shapes

    sd = {k: seeded_tensor(seed, k, shp) for k, shp in asr_model_shapes(cfg).items()}
    sd["normalize.glob_mean"] = seeded_tensor(seed, "normalize.glob_mean", (cfg["n_mels"],)) * 3.0 - 20.0
    sd["normalize.glob_std"] = seeded_tensor(seed, "normalize.glob_std", (cfg["n_mels"],)) * 8.0
    return sd


CONFORMER_LARGE = dict(name="conformer_large", sample_rate=16000, n_fft=512, win=512, hop=160, n_mels=80,
                       cnn_channels=(64, 32), input_size=640, d_model=512, nhead=8, num_encoder_layers=12,
                       num_decoder_layers=6, d_ffn=2048, vocab=5000, kernel_size=31, attention_type="RoPEMHA",
                       decoder_activation="gelu", max_length=2500)
def scale_csgu_conv(sd, tap_gain=1.4, bias_center=1.0):
    """In place: the seeded depthwise taps of every ``csgu.conv.conv.weight`` (C/2, 1, K) rescaled to std tap_gain / sqrt(K)
    and ``bias_center`` added to ``csgu.conv.conv.bias`` (the reference initialises it to ones, convolution.py:88).  With
    the xavier-like seeded taps (std ~0.0065 at C/2 = 1536) the conv hardly changes the gate, so errors in its padding or
    tap order would not show in the outputs."""
    for k in list(sd):
        if k.endswith("csgu.conv.conv.weight"):
            w = sd[k]
            xavier = math.sqrt(2.0 / (w.shape[1] * w.shape[2] + w.shape[0] * w.shape[2]))
            sd[k] = w * (tap_gain / math.sqrt(w.shape[2]) / xavier)
        elif k.endswith("csgu.conv.conv.bias"):
            sd[k] = sd[k] + bias_center
    return sd


# recipes/LibriSpeech/ASR/transformer/hparams/branchformer_large.yaml (seq2seq + CTC, 18 Branchformer layers) and
# recipes/LibriSpeech/ASR/CTC/hparams/branchformer_large.yaml (encoder-only, CTC over 31 characters)
BRANCHFORMER_LARGE = dict(name="branchformer_large", sample_rate=16000, n_fft=512, win=512, hop=160, n_mels=80,
                          cnn_channels=(64, 32), input_size=640, d_model=512, nhead=8, num_encoder_layers=18,
                          num_decoder_layers=6, d_ffn=2048, vocab=5000, kernel_size=31, attention_type="RelPosMHAXL",
                          decoder_activation="gelu", max_length=2500, encoder_module="branchformer",
                          csgu_linear_units=3072, branchformer_activation="gelu")
BRANCHFORMER_CTC = dict(name="branchformer_ctc", sample_rate=16000, n_fft=512, win=400, hop=160, n_mels=80,
                        cnn_channels=(64, 32), input_size=640, d_model=256, nhead=4, num_encoder_layers=18,
                        num_decoder_layers=0, d_ffn=1024, vocab=31, kernel_size=31, attention_type="RelPosMHAXL",
                        decoder_activation="gelu", max_length=2500, encoder_module="branchformer",
                        csgu_linear_units=2400, branchformer_activation="gelu")
def scale_hypernet(sd, gain=1.0):
    """In place: every HyperMixing hypernetwork matrix (``hyper.w{1,2}_gen.fc{1,2}_weights``, (M, out, in)) rescaled to the
    per-head xavier std gain * sqrt(2 / (in + out)).  seeded_tensor treats the (M, out, in) stack as one conv-like kernel and
    gives it std sqrt(2 / (out * in + M * in)), 4-6x smaller: the generated W1 / W2 are then nearly the biases, the same for
    every frame, and errors in the positional input or the per-frame hypernetwork would not show in the outputs."""
    for k in list(sd):
        if k.endswith("_gen.fc1_weights") or k.endswith("_gen.fc2_weights"):
            w = sd[k]
            M, o, i = w.shape
            seeded = math.sqrt(2.0 / (o * i + M * i))
            sd[k] = w * (gain * math.sqrt(2.0 / (i + o)) / seeded)
    return sd


# recipes/LibriSpeech/ASR/transformer/hparams/hyperconformer_22M.yaml: 10 Conformer layers with HyperMixing (8 heads of 32
# channels, hypernetwork width d_ffn / 8 = 128 per head), 4 decoder layers, 5000 tokens
HYPERCONFORMER_22M = dict(name="hyperconformer_22m", sample_rate=16000, n_fft=400, win=400, hop=160, n_mels=80,
                          cnn_channels=(64, 32), input_size=640, d_model=256, nhead=8, num_encoder_layers=10,
                          num_decoder_layers=4, d_ffn=1024, vocab=5000, kernel_size=31, attention_type="hypermixing",
                          decoder_activation="gelu", max_length=2500)
CONFORMER_SMALL = dict(name="conformer_small", sample_rate=16000, n_fft=400, win=400, hop=160, n_mels=80,
                       cnn_channels=(64, 32), input_size=640, d_model=144, nhead=4, num_encoder_layers=12,
                       num_decoder_layers=4, d_ffn=1024, vocab=5000, kernel_size=31, attention_type="RelPosMHAXL",
                       decoder_activation="gelu", max_length=2500)
# recipes/LibriSpeech/ASR/transformer/hparams/transformer.yaml: the 3-block front-end (5x5 / 5x5 / 1x1 + residual, 64
# channels), 12 pre-norm Transformer encoder layers with regularMHA (4 heads of 128), 6 decoder layers, 5000 tokens
TRANSFORMER_LARGE = dict(name="transformer_large", sample_rate=16000, n_fft=400, win=400, hop=160, n_mels=80,
                         cnn_channels=(64, 64), cnn_blocks=3, input_size=1280, d_model=512, nhead=4, num_encoder_layers=12,
                         num_decoder_layers=6, d_ffn=2048, vocab=5000, kernel_size=31, attention_type="regularMHA",
                         decoder_activation="gelu", max_length=2500, encoder_module="transformer")
# recipes/AISHELL-1/ASR/transformer/hparams/train_ASR_transformer.yaml: the 2-block front-end with 256 channels (input
# 20 x 256 = 5120), 12 pre-norm Transformer encoder layers with regularMHA (4 heads of 64), 6 decoder layers, 5000 tokens;
# blank 0, bos 1, eos 2
AISHELL_TRANSFORMER = dict(name="aishell_transformer", sample_rate=16000, n_fft=400, win=400, hop=160, n_mels=80,
                           cnn_channels=(256, 256), input_size=5120, d_model=256, nhead=4, num_encoder_layers=12,
                           num_decoder_layers=6, d_ffn=2048, vocab=5000, kernel_size=31, attention_type="regularMHA",
                           decoder_activation="gelu", max_length=2500, encoder_module="transformer")
# recipes/Libriheavy/ASR/transformer/hparams/conformer_large.yaml: 14 Conformer layers at d_model 640 with RelPosMHAXL (8 heads
# of 80), 6 GELU decoder layers, 5000 tokens; and recipes/PeoplesSpeech/ASR/transformer/hparams/conformer_large.yaml: the same
# encoder, 6 decoder layers with a Swish FFN, 5120 tokens
CONFORMER_640 = dict(name="conformer_640", sample_rate=16000, n_fft=512, win=512, hop=160, n_mels=80,
                     cnn_channels=(64, 32), input_size=640, d_model=640, nhead=8, num_encoder_layers=14,
                     num_decoder_layers=6, d_ffn=2048, vocab=5000, kernel_size=31, attention_type="RelPosMHAXL",
                     decoder_activation="gelu", max_length=2500)
CONFORMER_640_PEOPLES = dict(CONFORMER_640, name="conformer_640_peoples", vocab=5120, decoder_activation="swish")
# recipes/Loquacious/ASR/transformer/hparams/conformer_{small,base,large,xlarge}.yaml: Conformer encoders with
# conformer_activation=torch.nn.GELU and RelPosMHAXL (head width 64), GELU decoders, Fbank with n_fft 400 and the default
# 25 ms window; xlarge is the released 480M model.  Token indices: blank 3, bos 1, eos 2, pad 0.
LOQUACIOUS_SMALL = dict(name="loquacious_small", sample_rate=16000, n_fft=400, win=400, hop=160, n_mels=80,
                        cnn_channels=(64, 32), input_size=640, d_model=256, nhead=4, num_encoder_layers=12,
                        num_decoder_layers=6, d_ffn=1024, vocab=1024, kernel_size=31, attention_type="RelPosMHAXL",
                        decoder_activation="gelu", max_length=2500, conformer_activation="gelu")
LOQUACIOUS_BASE = dict(LOQUACIOUS_SMALL, name="loquacious_base", d_model=512, nhead=8, d_ffn=2048, vocab=5120)
LOQUACIOUS_LARGE = dict(LOQUACIOUS_SMALL, name="loquacious_large", d_model=768, nhead=12, num_encoder_layers=14,
                        d_ffn=3072, vocab=5120)
LOQUACIOUS_XLARGE = dict(LOQUACIOUS_SMALL, name="loquacious_xlarge", d_model=1024, nhead=16, num_encoder_layers=18,
                         d_ffn=3072, vocab=5120)
LOQUACIOUS_BLANK, LOQUACIOUS_BOS, LOQUACIOUS_EOS, LOQUACIOUS_PAD = 3, 1, 2, 0
