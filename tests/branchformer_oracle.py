"""CPU fp32 restatement of the Branchformer encoder (lobes/models/transformer/Branchformer.py:92-410 and the CSGU,
lobes/models/convolution.py:22-113) on top of oracle/asr_oracle.py's shared pieces (RelPosMHAXL, LayerNorm, masks, the
``q=`` operand-rounding hook).  Test infrastructure only: tools/make_branchformer_golden.py asserts that it equals the
running reference, and the Branchformer tests compare the device against it."""
import torch
import torch.nn.functional as F

from mirrors import seeded
from oracle import asr_oracle as O


def state(cfg, fx):
    """the fixture's weights: seeded with its weight_seed, the CSGU convolutions rescaled by its tap_gain and bias_center"""
    from speechbrain_b200.utils.seeded_init import scale_csgu_conv
    return seeded(cfg, fx["weight_seed"], lambda sd: scale_csgu_conv(sd, fx["tap_gain"], fx["bias_center"]))


def csgu(u, sd, p, q=None):
    """ConvolutionalSpatialGatingUnit.forward (gate Identity, no linear after the conv): a, b = u.chunk(2);
    a * Conv1d(LN(b)) with speechbrain's Conv1d(padding="same") default padding_mode "reflect" over the batch-padded length
    (CNN.py:376,495; F.pad fails for T <= (K-1)/2).  ``q`` rounds u (the device keeps it in fp16)."""
    if q is not None:
        u = q(u)
    a, b = u.chunk(2, dim=-1)
    b = O._ln(b, sd, p + "norm.norm.", 1e-5)
    w = sd[p + "conv.conv.weight"]
    pad = (w.shape[-1] - 1) // 2
    h = F.pad(b.transpose(1, 2), (pad, pad), mode="reflect")
    h = F.conv1d(h, w, sd[p + "conv.conv.bias"], groups=w.shape[0]).transpose(1, 2)
    return h * a


def branchformer_layer(x, sd, p, nhead, key_padding_mask, pos_embs, act, q=None):
    """Branchformer.py:180-234 BranchformerEncoderLayer.forward (RelPosMHAXL; the convolution branch is never masked)."""
    x1 = O.relpos_mha(O._ln(x, sd, p + "norm_mhsa.norm.", 1e-5), pos_embs, sd, p + "mha_layer.", nhead, key_padding_mask, q)
    cb = p + "convolution_branch."
    x2 = act(O._mm(O._ln(x, sd, p + "norm_conv.norm.", 1e-5), sd[cb + "pre_channel_proj.weight"],
                   sd[cb + "pre_channel_proj.bias"], q))
    x2 = O._mm(csgu(x2, sd, cb + "csgu.", q), sd[cb + "post_channel_proj.weight"], sd[cb + "post_channel_proj.bias"], q)
    return x + O._mm(torch.cat([x1, x2], dim=-1), sd[p + "merge_proj.weight"], sd[p + "merge_proj.bias"], q)


def encode(src, wav_len, sd, cfg, prefix="", q=None, return_layers=False):
    """TransformerASR.py:475-544 TransformerASR.encode with encoder_module="branchformer" (BranchformerEncoder.forward,
    Branchformer.py:330-410, final LayerNorm eps 1e-6)."""
    if src.dim() == 4:
        src = src.reshape(src.shape[0], src.shape[1], -1)
    B, T, _ = src.shape
    kpm = None
    if wav_len is not None:
        kpm = ~O.length_to_mask(torch.round(wav_len * T))
    x = O._mm(src, sd[prefix + "custom_src_module.layers.0.w.weight"], sd[prefix + "custom_src_module.layers.0.w.bias"], q)
    pos = O.relpos_table(T, x.shape[-1])
    act = F.relu if cfg.get("branchformer_activation", "gelu") == "relu" else F.gelu
    layers = []
    for i in range(cfg["num_encoder_layers"]):
        x = branchformer_layer(x, sd, f"{prefix}encoder.layers.{i}.", cfg["nhead"], kpm, pos, act, q)
        layers.append(x)
    x = O._ln(x, sd, prefix + "encoder.norm.norm.", 1e-6)
    return (x, layers) if return_layers else x


def wav_to_states(wav, wav_len, sd, cfg, q=None):
    """wav -> Fbank -> global CMVN -> CNN -> Branchformer encoder (``cfg``: a seeded_init config dict)."""
    ocfg = dict(cfg, win_length=cfg["win"] * 1000 // cfg["sample_rate"])
    return encode(O.full_pipeline_features(wav, wav_len, sd, ocfg), wav_len, sd, ocfg, "Transformer.", q=q)
