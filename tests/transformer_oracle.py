"""CPU fp32 restatement of the Transformer recipes' front-end and encoder on top of oracle/asr_oracle.py's shared pieces:
ConvolutionFrontEnd(num_blocks=3, kernel_sizes=(5, 5, 1), strides=(2, 2, 1), residuals=(False, False, True), 64 channels;
lobes/models/convolution.py:116-320 with nnet/CNN.py Conv2d's reflect "same" padding) and TransformerASR.encode with
encoder_module="transformer", attention_type="regularMHA", normalize_before=True (Transformer.py:311-490).  Test
infrastructure only: tools/make_transformer_golden.py asserts that it equals the running reference, and the Transformer
tests compare the device against it."""
import torch
import torch.nn.functional as F

from oracle import asr_oracle as O


def _conv(x, sd, p, k, stride):
    """nnet/CNN.py Conv2d on channels-last x [B, T, F, C]: the kernel's first axis runs over F, the second over T; "same"
    padding is reflect k // 2 on both axes when stride > 1 and none for the 1x1 convolutions."""
    x = x.permute(0, 3, 2, 1)  # [B, C, F, T]
    if k > 1:
        x = F.pad(x, (k // 2, k // 2, k // 2, k // 2), mode="reflect")
    return F.conv2d(x, sd[p + "weight"], sd[p + "bias"], stride=stride).permute(0, 3, 2, 1)


def _ln2(x, sd, p):
    """nnet/normalization.py LayerNorm over the (F, C) of a frame, eps 1e-5."""
    return F.layer_norm(x, x.shape[-2:], sd[p + "weight"], sd[p + "bias"], 1e-5)


def cnn3(feats, sd, prefix="CNN."):
    """feats [B, T0, F0] -> [B, T2, F2, 64]."""
    x = feats.unsqueeze(-1)
    for i in range(2):
        p = f"{prefix}convblock_{i}.convs."
        x = F.leaky_relu(_ln2(_conv(x, sd, p + "conv_0.conv.", 5, 2), sd, p + "norm_0.norm."), 0.01)
    p = f"{prefix}convblock_2."
    main = F.leaky_relu(_ln2(_conv(x, sd, p + "convs.conv_0.conv.", 1, 1), sd, p + "convs.norm_0.norm."), 0.01)
    return main + _ln2(_conv(x, sd, p + "reduce_conv.conv.conv.", 1, 1), sd, p + "reduce_conv.norm.norm.")


def encode(src, wav_len, sd, cfg, prefix="Transformer."):
    """TransformerASR.py:475-544 with the Transformer encoder: src [B, T, input_size] -> [B, T, d]."""
    if src.dim() == 4:
        src = src.reshape(src.shape[0], src.shape[1], -1)
    B, T, _ = src.shape
    d, nhead = cfg["d_model"], cfg["nhead"]
    kpm = None
    if wav_len is not None:
        kpm = ~O.length_to_mask(torch.round(wav_len * T), T).bool()
    x = O._mm(src, sd[prefix + "custom_src_module.layers.0.w.weight"], sd[prefix + "custom_src_module.layers.0.w.bias"])
    x = x + O.sine_pe(T, d).unsqueeze(0)
    for i in range(cfg["num_encoder_layers"]):
        p = f"{prefix}encoder.layers.{i}."
        a, _ = O._mha_regular(O._ln(x, sd, p + "norm1.norm.", 1e-6), O._ln(x, sd, p + "norm1.norm.", 1e-6), sd,
                              p + "self_att.", nhead, key_padding_mask=kpm)
        x = x + a
        h = O._ln(x, sd, p + "norm2.norm.", 1e-6)
        h = F.gelu(O._mm(h, sd[p + "pos_ffn.ffn.0.weight"], sd[p + "pos_ffn.ffn.0.bias"]))
        x = x + O._mm(h, sd[p + "pos_ffn.ffn.3.weight"], sd[p + "pos_ffn.ffn.3.bias"])
    return O._ln(x, sd, prefix + "encoder.norm.norm.", 1e-6)


def wav_to_cnn(wav, wav_lens, sd, cfg):
    """Fbank -> global InputNormalization -> the 3-block front-end."""
    f = O.fbank(wav, n_fft=cfg["n_fft"], n_mels=cfg["n_mels"], win_length_ms=cfg["win"] * 1000 // cfg["sample_rate"])
    f = O.input_norm(f, wav_lens, "global", sd["normalize.glob_mean"], sd["normalize.glob_std"])
    return cnn3(f, sd)
