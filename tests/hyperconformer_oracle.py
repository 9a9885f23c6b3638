"""CPU fp32 restatement of the HyperConformer encoder: the Conformer layer (Conformer.py:451-499) with self-attention replaced
by multi-head HyperMixing (nnet/hypermixing.py:90-195, 249-372; tied=False, keep_output_size=False), on top of
oracle/asr_oracle.py's shared pieces (FFN and convolution modules, LayerNorm, masks, the ``q=`` operand-rounding hook).
Test infrastructure only: tools/make_hyperconformer_golden.py asserts that it equals the running reference, and the
HyperConformer tests compare the device against it."""
import torch
import torch.nn.functional as F

from oracle import asr_oracle as O

MAX_FRAMES = 3000  # HyperMixing's own PositionalEncoding(d, max_length=3000)


def _id(t):
    return t


def hyper_weights(h, sd, p, q=None):
    """ParallelMLPs.forward (hypermixing.py:339-372): h [B, T, d] -> [B, M, T, k] with M heads of e = d / M channels."""
    q = q or _id
    w1, b1, w2, b2 = (sd[p + n] for n in ("fc1_weights", "fc1_biases", "fc2_weights", "fc2_biases"))
    M, e = w1.shape[0], w1.shape[2]
    x = h.reshape(h.shape[0], h.shape[1], M, e)
    x = torch.einsum("blmf,mhf->bmlh", q(x), q(w1)) + b1.unsqueeze(0).unsqueeze(2)
    x = F.gelu(x)
    return torch.einsum("bmlh,mfh->bmlf", q(x), q(w2)) + b2.unsqueeze(0).unsqueeze(2)


def hypermixing(xn, sd, p, key_padding_mask, q=None):
    """HyperMixing.forward on the norm1 output xn [B, T, d] -> layer_norm(mixing) [B, T, d].  ``q`` rounds the operands of
    every product (hin, the hypernetworks' hidden layers, xm, W1, W2, GELU(H)), as the device keeps them in fp16."""
    qq = q or _id
    B, T, d = xn.shape
    if T > MAX_FRAMES:
        raise RuntimeError(f"HyperMixing: {T} frames exceed its {MAX_FRAMES}-row positional table")
    valid = torch.ones(B, T) if key_padding_mask is None else (~key_padding_mask).float()
    xm = xn * valid.unsqueeze(-1)
    hin = xm + O.sine_pe(T, d)  # the module's positional_encoding.pe buffer, rows [0, T)
    W1 = hyper_weights(hin, sd, p + "hyper.w1_gen.", q) * valid[:, None, :, None]
    W2 = hyper_weights(hin, sd, p + "hyper.w2_gen.", q) * valid[:, None, :, None]
    M = W1.shape[1]
    xh = xm.transpose(1, 2).reshape(B, M, d // M, T)            # [B, M, e, T]: channels m*e .. m*e + e - 1
    H = torch.matmul(qq(xh), qq(W1))                            # [B, M, e, k]
    y = torch.matmul(qq(F.gelu(H)), qq(W2).transpose(-1, -2))   # [B, M, e, T]
    y = y.reshape(B, d, T).transpose(1, 2)
    return O._ln(y, sd, p + "layer_norm.", 1e-5)


def max_abs_h(xn, sd, p, key_padding_mask):
    """max |H| of one HyperMixing layer (the fp16 range the device's G store has to cover)."""
    B, T, d = xn.shape
    valid = torch.ones(B, T) if key_padding_mask is None else (~key_padding_mask).float()
    xm = xn * valid.unsqueeze(-1)
    W1 = hyper_weights(xm + O.sine_pe(T, d), sd, p + "hyper.w1_gen.") * valid[:, None, :, None]
    M = W1.shape[1]
    return float(torch.matmul(xm.transpose(1, 2).reshape(B, M, d // M, T), W1).abs().max())


def hyperconformer_layer(x, sd, p, key_padding_mask, q=None):
    """Conformer.py:451-499 ConformerEncoderLayer.forward with mha_layer = HyperMixing (attn_mask and pos_embs unused)."""
    conv_mask = key_padding_mask.unsqueeze(-1) if key_padding_mask is not None else None
    x = x + 0.5 * O.conformer_ffn(x, sd, p + "ffn_module1.", q)
    x = x + hypermixing(O._ln(x, sd, p + "norm1.norm.", 1e-5), sd, p + "mha_layer.", key_padding_mask, q)
    x = x + O.conv_module(x, sd, p + "convolution_module.", conv_mask, q)
    return O._ln(x + 0.5 * O.conformer_ffn(x, sd, p + "ffn_module2.", q), sd, p + "norm2.norm.", 1e-5)


def encode(src, wav_len, sd, cfg, prefix="", q=None, return_layers=False):
    """TransformerASR.py:475-544 TransformerASR.encode with attention_type="hypermixing" (no positional encoding on the
    source, ConformerEncoder.forward with its final LayerNorm eps 1e-6)."""
    if src.dim() == 4:
        src = src.reshape(src.shape[0], src.shape[1], -1)
    B, T, _ = src.shape
    kpm = None
    if wav_len is not None:
        kpm = ~O.length_to_mask(torch.round(wav_len * T))
    x = O._mm(src, sd[prefix + "custom_src_module.layers.0.w.weight"], sd[prefix + "custom_src_module.layers.0.w.bias"], q)
    layers = []
    for i in range(cfg["num_encoder_layers"]):
        x = hyperconformer_layer(x, sd, f"{prefix}encoder.layers.{i}.", kpm, q)
        layers.append(x)
    x = O._ln(x, sd, prefix + "encoder.norm.norm.", 1e-6)
    return (x, layers) if return_layers else x


def wav_to_states(wav, wav_len, sd, cfg, q=None):
    """wav -> Fbank -> global CMVN -> CNN -> HyperConformer encoder (``cfg``: a seeded_init config dict)."""
    ocfg = dict(cfg, win_length=cfg["win"] * 1000 // cfg["sample_rate"])
    return encode(O.full_pipeline_features(wav, wav_len, sd, ocfg), wav_len, sd, ocfg, "Transformer.", q=q)
