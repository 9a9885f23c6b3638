"""Plain-PyTorch fp32 restatement of the reference ASR inference path.

TEST INFRASTRUCTURE (see oracle/__init__.py). Every function cites the reference
file:line it follows (paths relative to /root/reference/speechbrain/).

All model functions take ``sd``: a flat ``{key: tensor}`` dict using the
reference's own ``state_dict`` key names (SURVEY.md 8b), and a small config dict.
"""
import math

import torch
import torch.nn.functional as F

# --------------------------------------------------------------------------
# Frontend: STFT -> power -> mel filterbank -> dB (+ top_db clip)
# --------------------------------------------------------------------------


def stft_power(wav, n_fft=400, win_length_ms=25, hop_length_ms=10, sample_rate=16000):
    """processing/features.py:109-188 (STFT) + :341-378 (spectral_magnitude, power=1).

    torch.stft(center=True, pad_mode="constant", periodic hamming window,
    onesided) followed by re^2 + im^2.  Returns (B, T_f, n_fft//2+1).
    """
    win = int(round(sample_rate / 1000.0 * win_length_ms))
    hop = int(round(sample_rate / 1000.0 * hop_length_ms))
    window = torch.hamming_window(win)
    if win < n_fft:  # torch.stft centres a short window inside n_fft
        left = (n_fft - win) // 2
        window = F.pad(window, (left, n_fft - win - left))
    x = F.pad(wav.float(), (n_fft // 2, n_fft // 2))  # zeros ("constant")
    frames = x.unfold(1, n_fft, hop) * window
    spec = torch.fft.rfft(frames, dim=-1)
    return spec.real.pow(2) + spec.imag.pow(2)


def mel_matrix(n_mels=40, n_fft=400, sample_rate=16000, f_min=0, f_max=None):
    """processing/features.py:487-507 (band edges) + :620-650 (triangular filters).

    Returns the (n_fft//2+1, n_mels) matrix the reference rebuilds every call.
    """
    if f_max is None:
        f_max = sample_rate // 2
    n_stft = n_fft // 2 + 1
    to_mel = lambda hz: 2595 * math.log10(1 + hz / 700)
    mel = torch.linspace(to_mel(f_min), to_mel(f_max), n_mels + 2)
    hz = 700 * (10 ** (mel / 2595) - 1)
    band = (hz[1:] - hz[:-1])[:-1]
    f_central = hz[1:-1]
    all_freqs = torch.linspace(0, sample_rate // 2, n_stft)
    all_freqs_mat = all_freqs.repeat(f_central.shape[0], 1)
    f_central_mat = f_central.repeat(all_freqs_mat.shape[1], 1).transpose(0, 1)
    band_mat = band.repeat(all_freqs_mat.shape[1], 1).transpose(0, 1)
    slope = (all_freqs_mat - f_central_mat) / band_mat
    left_side = slope + 1.0
    right_side = -slope + 1.0
    zero = torch.zeros(1)
    return torch.max(zero, torch.min(left_side, right_side)).transpose(0, 1)


def fbank(wav, n_fft=400, n_mels=40, win_length_ms=25, hop_length_ms=10,
          sample_rate=16000, f_min=0, f_max=None, amin=1e-10, top_db=80.0):
    """lobes/features.py:147-169 (Fbank.forward, deltas=False, context=False) with
    processing/features.py:512-586 (Filterbank.forward) and :736-759 (_amplitude_to_DB).
    """
    power = stft_power(wav, n_fft, win_length_ms, hop_length_ms, sample_rate)
    fb = torch.matmul(power, mel_matrix(n_mels, n_fft, sample_rate, f_min, f_max))
    x_db = 10.0 * torch.log10(torch.clamp(fb, min=amin))
    # db_multiplier = log10(max(amin, ref_value=1)) = 0
    new_max = x_db.amax(dim=(-2, -1)) - top_db  # per sequence, incl. padding
    return torch.max(x_db, new_max.view(-1, 1, 1))


def padding_mask(T, lengths, eps=1e-6):
    """processing/features.py:1554-1615 make_padding_mask -> (B, T) bool, True = valid."""
    abs_lengths = (lengths * T - eps).unsqueeze(1)
    return torch.arange(T).unsqueeze(0) < abs_lengths


def input_norm(x, lengths=None, norm_type="global", glob_mean=None, glob_std=None,
               std_norm=True, avoid_padding_norm=False, epsilon=1e-10):
    """processing/features.py:1404-1455 InputNormalization.forward in eval mode
    ("global": fixed stats; "sentence": masked per-utterance stats :1478-1486)."""
    B, T, _ = x.shape
    if lengths is None:
        lengths = torch.ones(B)
    mask = padding_mask(T, lengths).unsqueeze(-1)
    if norm_type == "global":
        mean, std = glob_mean.unsqueeze(0), glob_std.unsqueeze(0)
    elif norm_type == "sentence":
        n = mask.sum(1, keepdim=True)
        mean = (x * mask).sum(1, keepdim=True) / n
        var = ((x - mean) * mask).square().sum(1, keepdim=True) / n
        mean, std = mean.squeeze(1), var.squeeze(1).sqrt()
    else:
        raise ValueError(norm_type)
    if not std_norm:
        std = torch.ones_like(mean)
    mean, std = mean.unsqueeze(1), std.unsqueeze(1)
    if avoid_padding_norm:
        mean = mean.masked_fill(~mask, 0.0)
        std = std.masked_fill(~mask, 1.0)
    return (x - mean) / std.clamp(min=epsilon)


def cnn_frontend(x, sd, prefix="", num_blocks=2):
    """lobes/models/convolution.py:116-320 (ConvolutionFrontEnd/ConvBlock, one conv
    per block, stride 2, no residual) + nnet/CNN.py:654-751 (Conv2d: channels-last
    API, reflect "same" padding k//2 when stride>1) + nnet/normalization.py:185-242
    (LayerNorm over the last two dims) + LeakyReLU(0.01).

    x: (B, T, F) -> (B, T', F', C).
    """
    x = x.transpose(1, -1).unsqueeze(1)  # (B, 1, F, T)
    for i in range(num_blocks):
        p = f"{prefix}convblock_{i}.convs."
        w, b = sd[p + "conv_0.conv.weight"], sd[p + "conv_0.conv.bias"]
        x = F.pad(x, (1, 1, 1, 1), mode="reflect")
        x = F.conv2d(x, w, b, stride=2)  # (B, C, F', T')
        x = x.transpose(1, -1)  # (B, T', F', C)
        g, be = sd[p + "norm_0.norm.weight"], sd[p + "norm_0.norm.bias"]
        x = F.layer_norm(x, g.shape, g, be, 1e-5)
        x = F.leaky_relu(x, 0.01)
        if i + 1 < num_blocks:
            x = x.transpose(1, -1)  # back to (B, C, F', T')
    return x


# --------------------------------------------------------------------------
# Conformer encoder
# --------------------------------------------------------------------------


def length_to_mask(length, max_len=None):
    """dataio/dataio.py:803-848."""
    if max_len is None:
        max_len = int(length.max().long().item())
    return torch.arange(max_len, dtype=length.dtype).expand(len(length), max_len) < length.unsqueeze(1)


def rope_tables(T, head_dim):
    """nnet/attention.py:1012-1055 PrecomputedRoPESinusoids: (cos, signed sin), (T, head_dim)."""
    angles = torch.exp(torch.arange(0, head_dim, 2, dtype=torch.float32) * -(math.log(10000.0) / head_dim))
    times = torch.arange(0, T, dtype=torch.float32)
    ta = torch.outer(times, angles)
    cos = torch.stack([torch.cos(ta)] * 2, dim=-1).reshape(T, head_dim)
    uns = torch.stack([torch.sin(ta)] * 2, dim=-1).reshape(T, head_dim)
    sin = ((-1) ** torch.arange(head_dim, dtype=torch.float32)) * -uns
    return cos, sin


def rope_rotate(x):
    """nnet/attention.py:1161-1188 _rope_rotate; x: (B, L, H, d_h).

    The reference memoises tables of length 2**ceil(log2(L)) and slices [:L]; the
    values for t < L are identical, so we build exactly L rows."""
    _, L, _, dh = x.shape
    cos, sin = rope_tables(L, dh)
    idx = torch.arange(dh).view(-1, 2).flip(1).reshape(-1)
    return x * cos.unsqueeze(1) + x[..., idx] * sin.unsqueeze(1)


def relpos_table(T, d):
    """nnet/attention.py:360-408 RelPosEncXL.make_pe -> (1, 2T-1, d)."""
    inv_freq = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    tot = torch.empty((2, T, d))
    pos = torch.arange(0, T, dtype=torch.float32).unsqueeze(-1)
    sinus = torch.sin(pos * inv_freq)
    tot[0][:, 0::2] = sinus
    tot[0][:, 1::2] = torch.cos(pos * inv_freq)
    tot[1][:, 0::2] = sinus
    tot[1][:, 1::2] = torch.cos(-pos * inv_freq)
    past = torch.flip(tot[0], (0,)).unsqueeze(0)
    future = tot[1][1:].unsqueeze(0)
    return torch.cat([past, future], dim=1)


def _mm(x, w, b=None, q=None):
    """x @ w.T (+b). ``q`` optionally rounds both operands (used only to *predict*
    the error of reduced-precision tensor-core operands; q=None is the oracle)."""
    if q is not None:
        x, w = q(x), q(w)
    return F.linear(x, w, b)


def chunk_mask(T, chunk_size, left_context_chunks=None):
    """TransformerASR.py:46-105 make_transformer_src_mask with a DynChunkTrainConfig: (T, T) bool, True = masked.
    Frame i (chunk c = i // chunk_size) sees keys j < (c + 1) * chunk_size and, with a finite left context of n chunks,
    j >= (c - n) * chunk_size."""
    i = torch.arange(T)
    hi = (i // chunk_size + 1) * chunk_size
    m = i[None, :] >= hi[:, None]
    if left_context_chunks is not None:
        lo = hi - chunk_size * (left_context_chunks + 1)
        m = m | (i[None, :] < lo[:, None])
    return m


def rope_mha(x, sd, p, nhead, key_padding_mask, q=None, attn_mask=None):
    """nnet/attention.py:1284-1399 RoPEMHA.forward (self-attention branch) with
    masks_union :1402-1440 and SDPA(scale=1/sqrt(embed_dim) :1272)."""
    B, T, d = x.shape
    dh = d // nhead
    qkv = _mm(x, sd[p + "in_proj_weight"], None, q).view(B, T, nhead, 3 * dh)
    qh, kh, vh = qkv.chunk(3, dim=-1)
    qh, kh = rope_rotate(qh), rope_rotate(kh)
    scale = 1.0 / math.sqrt(d)
    s = torch.einsum("bihd,bjhd->bhij", qh, kh) * scale
    if key_padding_mask is not None:
        s = s.masked_fill(key_padding_mask.view(B, 1, 1, T), float("-inf"))
    if attn_mask is not None:  # masks_union :1402-1440 (chunked attention, True = masked)
        s = s.masked_fill(attn_mask.view(1, 1, T, T), float("-inf"))
    a = torch.softmax(s, dim=-1)
    o = torch.einsum("bhij,bjhd->bihd", a, vh).reshape(B, T, d)
    return _mm(o, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"], q)


def relpos_mha(x, pos_embs, sd, p, nhead, key_padding_mask, q=None, attn_mask=None):
    """nnet/attention.py:555-742 RelPosMHAXL.forward + rel_shift :537-553.

    Quirks kept: scale 1/sqrt(embed_dim); pos_bias_{u,v} stored (d_h, H) but
    *viewed* (H, d_h); interleaved per-head QKV rows."""
    B, T, d = x.shape
    dh = d // nhead
    qkv = _mm(x, sd[p + "in_proj_weight"], None, q).view(B, T, nhead, 3 * dh)
    qh, kh, vh = qkv.chunk(3, dim=-1)
    p_k = _mm(pos_embs, sd[p + "linear_pos.weight"], None, q).view(1, -1, nhead, dh)
    u = sd[p + "pos_bias_u"].reshape(1, 1, nhead, dh)
    v = sd[p + "pos_bias_v"].reshape(1, 1, nhead, dh)
    scale = 1.0 / math.sqrt(d)
    q_u = (qh + u).transpose(1, 2) * scale
    q_v = (qh + v).transpose(1, 2) * scale
    ac = torch.matmul(q_u, kh.permute(0, 2, 3, 1))
    bd = torch.matmul(q_v, p_k.permute(0, 2, 3, 1))  # (B,H,T,2T-1)
    b_, h_, ql, pl = bd.shape
    bd = F.pad(bd, (1, 0)).view(b_, h_, -1, ql)[:, :, 1:].reshape(b_, h_, ql, pl)[..., : pl // 2 + 1]
    s = ac + bd
    if attn_mask is not None:  # attention.py:694-702 (bool mask: masked_fill -inf before the softmax, 0 after)
        s = s.masked_fill(attn_mask.view(1, 1, T, T), float("-inf"))
    if key_padding_mask is not None:
        s = s.masked_fill(key_padding_mask.view(B, 1, 1, T), float("-inf"))
    a = torch.softmax(s, dim=-1)
    if attn_mask is not None:
        a = a.masked_fill(attn_mask.view(1, 1, T, T), 0.0)
    if key_padding_mask is not None:
        a = a.masked_fill(key_padding_mask.view(B, 1, 1, T), 0.0)
    o = torch.matmul(a, vh.transpose(1, 2)).transpose(1, 2).reshape(B, T, d)
    return _mm(o, sd[p + "out_proj.weight"], sd[p + "out_proj.bias"], q)


def _ln(x, sd, p, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[p + "weight"], sd[p + "bias"], eps)


def conformer_ffn(x, sd, p, q=None):
    """Conformer.py:425-445 ffn_module{1,2}: LN(1e-5) -> Linear -> Swish -> Linear
    (nnet/attention.py:889-947 PositionalwiseFeedForward)."""
    h = _ln(x, sd, p + "0.", 1e-5)
    h = F.silu(_mm(h, sd[p + "1.ffn.0.weight"], sd[p + "1.ffn.0.bias"], q))
    return _mm(h, sd[p + "1.ffn.3.weight"], sd[p + "1.ffn.3.bias"], q)


def conv_module(x, sd, p, conv_mask, q=None, chunk_size=None):
    """Conformer.py:314-330 ConvolutionModule.forward (non-chunked branch) and :190-313 (Dynamic Chunk Convolution: a normal
    'same' convolution in which, for every output frame, the inputs beyond the end of its own chunk are zero)."""
    d = x.shape[-1]
    h = _ln(x, sd, p + "layer_norm.", 1e-5)
    w = sd[p + "bottleneck.0.weight"]
    h = _mm(h, w[:, :, 0], sd[p + "bottleneck.0.bias"], q)  # Conv1d k=1
    h = F.glu(h, dim=-1)
    wdw = sd[p + "conv.weight"]
    K = wdw.shape[-1]
    if chunk_size is None:
        h = F.conv1d(h.transpose(1, 2), wdw, sd[p + "conv.bias"], padding=(K - 1) // 2, groups=d).transpose(1, 2)
    else:  # explicit sum over taps with the future-of-the-chunk mask (restates the unfold / pad construction of the reference)
        B_, T_, _ = h.shape
        pad = (K - 1) // 2
        hp = F.pad(h, (0, 0, pad, pad))
        t = torch.arange(T_)
        chunk_end = (t // chunk_size + 1) * chunk_size
        out = sd[p + "conv.bias"].view(1, 1, d).expand(B_, T_, d).clone()
        for k in range(K):
            src_t = t + k - pad
            ok = (src_t < chunk_end).view(1, T_, 1)
            out = out + torch.where(ok, hp[:, k:k + T_, :], torch.zeros(())) * wdw[:, 0, k].view(1, 1, d)
        h = out
    h = F.silu(_ln(h, sd, p + "after_conv.0.", 1e-5))
    h = _mm(h, sd[p + "after_conv.2.weight"], sd[p + "after_conv.2.bias"], q)
    if conv_mask is not None:
        h = h.masked_fill(conv_mask, 0.0)
    return h


def conformer_layer(x, sd, p, nhead, attention_type, key_padding_mask, pos_embs, q=None, attn_mask=None, chunk_size=None):
    """Conformer.py:451-499 ConformerEncoderLayer.forward."""
    conv_mask = key_padding_mask.unsqueeze(-1) if key_padding_mask is not None else None
    x = x + 0.5 * conformer_ffn(x, sd, p + "ffn_module1.", q)
    skip = x
    h = _ln(x, sd, p + "norm1.norm.", 1e-5)
    if attention_type == "RoPEMHA":
        h = rope_mha(h, sd, p + "mha_layer.", nhead, key_padding_mask, q, attn_mask)
    elif attention_type == "RelPosMHAXL":
        h = relpos_mha(h, pos_embs, sd, p + "mha_layer.", nhead, key_padding_mask, q, attn_mask)
    else:
        raise ValueError(attention_type)
    x = h + skip
    x = x + conv_module(x, sd, p + "convolution_module.", conv_mask, q, chunk_size)
    return _ln(x + 0.5 * conformer_ffn(x, sd, p + "ffn_module2.", q), sd, p + "norm2.norm.", 1e-5)


def encode(src, wav_len, sd, cfg, prefix="", q=None, return_layers=False, dynchunk=None):
    """TransformerASR.py:475-544 TransformerASR.encode (+ :106-164 masks,
    Conformer.py:705-778 ConformerEncoder.forward incl. final LayerNorm(eps=1e-6))."""
    if src.dim() == 4:
        bz, t, c1, c2 = src.shape
        src = src.reshape(bz, t, c1 * c2)
    B, T, _ = src.shape
    kpm = None
    if wav_len is not None:
        abs_len = torch.round(wav_len * T)
        kpm = ~length_to_mask(abs_len)
        if kpm.shape[1] != T:
            raise ValueError("longest relative length must be 1.0")
    x = _mm(src, sd[prefix + "custom_src_module.layers.0.w.weight"],
            sd[prefix + "custom_src_module.layers.0.w.bias"], q)
    pos = relpos_table(T, x.shape[-1]) if cfg["attention_type"] == "RelPosMHAXL" else None
    amask = csz = None
    if dynchunk is not None:  # (chunk_size, left_context_chunks or None): encode(..., dynchunktrain_config=...) masked mode
        csz = dynchunk[0]
        amask = chunk_mask(T, csz, dynchunk[1])
    layers = []
    for i in range(cfg["num_encoder_layers"]):
        x = conformer_layer(x, sd, f"{prefix}encoder.layers.{i}.", cfg["nhead"],
                            cfg["attention_type"], kpm, pos, q, amask, csz)
        layers.append(x)
    x = _ln(x, sd, prefix + "encoder.norm.norm.", 1e-6)
    return (x, layers) if return_layers else x


# --------------------------------------------------------------------------
# Transformer decoder (no KV cache -- exactly like the reference) and searchers
# --------------------------------------------------------------------------


def sine_pe(n, d):
    """Transformer.py:252-303 PositionalEncoding table rows [0, n)."""
    pe = torch.zeros(n, d)
    pos = torch.arange(0, n).unsqueeze(1).float()
    den = torch.exp(torch.arange(0, d, 2).float() * -(math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(pos * den)
    pe[:, 1::2] = torch.cos(pos * den)
    return pe


def _mha_regular(qx, kx, sd, p, nhead, attn_mask=None, key_padding_mask=None):
    """nnet/attention.py:802-886 -> torch.nn.MultiheadAttention (in_proj [Wq;Wk;Wv]
    with bias, scale 1/sqrt(d_h))."""
    n, s, d = qx.shape
    dh = d // nhead
    W, b = sd[p + "att.in_proj_weight"], sd[p + "att.in_proj_bias"]
    qh = F.linear(qx, W[:d], b[:d]).view(n, s, nhead, dh).transpose(1, 2)
    kh = F.linear(kx, W[d:2 * d], b[d:2 * d]).view(n, -1, nhead, dh).transpose(1, 2)
    vh = F.linear(kx, W[2 * d:], b[2 * d:]).view(n, -1, nhead, dh).transpose(1, 2)
    sc = torch.matmul(qh, kh.transpose(-1, -2)) / math.sqrt(dh)
    if attn_mask is not None:
        sc = sc + attn_mask
    if key_padding_mask is not None:
        sc = sc.masked_fill(key_padding_mask.view(n, 1, 1, -1), float("-inf"))
    a = torch.softmax(sc, dim=-1)
    o = torch.matmul(a, vh).transpose(1, 2).reshape(n, s, d)
    return F.linear(o, sd[p + "att.out_proj.weight"], sd[p + "att.out_proj.bias"]), a.mean(1)


def decode(tgt, enc_out, enc_len, sd, cfg, prefix=""):
    """TransformerASR.py:426-473 TransformerASR.decode + Transformer.py:751-834,
    :915-963 (pre-norm decoder layers, eps 1e-6, GELU FFN) -- whole prefix each call."""
    n, s = tgt.shape
    d = cfg["d_model"]
    tgt_mask = torch.triu(torch.full((s, s), float("-inf")), diagonal=1)  # Transformer.py:1037-1068
    mem_kpm = None
    if enc_len is not None:
        mem_kpm = ~length_to_mask(enc_len.float())
    x = F.embedding(tgt.long(), sd[prefix + "custom_tgt_module.layers.0.emb.Embedding.weight"]) * math.sqrt(d)
    x = x + sine_pe(s, d).unsqueeze(0)
    attn = None
    act = F.gelu if cfg.get("decoder_activation", "gelu") == "gelu" else F.relu
    for j in range(cfg["num_decoder_layers"]):
        p = f"{prefix}decoder.layers.{j}."
        h = _ln(x, sd, p + "norm1.norm.", 1e-6)
        h, _ = _mha_regular(h, h, sd, p + "self_attn.", cfg["nhead"], attn_mask=tgt_mask)
        x = x + h
        h = _ln(x, sd, p + "norm2.norm.", 1e-6)
        h, attn = _mha_regular(h, enc_out, sd, p + "multihead_attn.", cfg["nhead"], key_padding_mask=mem_kpm)
        x = x + h
        h = _ln(x, sd, p + "norm3.norm.", 1e-6)
        h = F.linear(act(F.linear(h, sd[p + "pos_ffn.ffn.0.weight"], sd[p + "pos_ffn.ffn.0.bias"])),
                     sd[p + "pos_ffn.ffn.3.weight"], sd[p + "pos_ffn.ffn.3.bias"])
        x = x + h
    return _ln(x, sd, prefix + "decoder.norm.norm.", 1e-6), attn


def greedy_search(enc_states, wav_len, sd, cfg, seq_lin_w, seq_lin_b, bos_index=1, eos_index=2,
                  min_decode_ratio=0.0, max_decode_ratio=1.0, prefix="", return_logits=False):
    """decoders/seq2seq.py:181-276 S2SGreedySearcher.forward (temperature 0) with
    S2STransformerGreedySearcher.forward_step :360-367.

    Returns (hyps list[list[int]], top_lengths (B,1), top_scores (B,1,L), top_log_probs (B,1,L,V))."""
    B, T, _ = enc_states.shape
    enc_lens = torch.round(T * wav_len).int()
    memory = None
    inp = torch.full((B,), bos_index, dtype=torch.long)
    lp_list, logit_list = [], []
    has_ended = torch.zeros(B, dtype=torch.bool)
    for _ in range(int(T * min_decode_ratio), int(T * max_decode_ratio)):
        memory = inp.unsqueeze(1) if memory is None else torch.cat([memory, inp.unsqueeze(1)], dim=-1)
        pred, _ = decode(memory, enc_states, enc_lens, sd, cfg, prefix)
        logits = F.linear(pred, seq_lin_w, seq_lin_b)[:, -1, :]
        logit_list.append(logits)
        inp = logits.argmax(dim=-1)
        lp = F.log_softmax(logits.float(), dim=-1)
        lp_list.append(lp)
        has_ended = has_ended | (inp == eos_index)
        lp[has_ended] = -torch.inf
        inp[has_ended] = eos_index
        if has_ended.all():
            break
    log_probs = torch.stack(lp_list, dim=1)
    scores, preds = log_probs.max(dim=-1)
    m = scores == -torch.inf
    scores[m] = 0
    preds[m] = eos_index
    L = preds.shape[1]
    lens = []
    for b in range(B):
        nz = (preds[b] == eos_index).nonzero()
        lens.append(int(nz[0]) if len(nz) > 0 else L)
    hyps = [preds[b, : lens[b]].tolist() for b in range(B)]
    top_lengths = torch.tensor(lens, dtype=torch.float) / L
    out = (hyps, top_lengths.unsqueeze(1), scores.unsqueeze(1), log_probs.unsqueeze(1))
    if return_logits:
        return out + (torch.stack(logit_list, dim=1),)
    return out


def full_pipeline_features(wav, wav_lens, sd, cfg):
    """inference/ASR.py:100-128 encode_batch up to the encoder input: Fbank ->
    InputNormalization(global) -> ConvolutionFrontEnd."""
    f = fbank(wav, n_fft=cfg["n_fft"], n_mels=cfg["n_mels"], win_length_ms=cfg["win_length"])
    f = input_norm(f, wav_lens, "global", sd["normalize.glob_mean"], sd["normalize.glob_std"])
    return cnn_frontend(f, sd, "CNN.")


# --------------------------------------------------------------------------
# Beam search (no scorers): decoders/seq2seq.py:752-1749 S2SBeamSearcher + :1853-1934
# --------------------------------------------------------------------------


def beam_search(enc_states, wav_len, sd, cfg, seq_lin_w, seq_lin_b, bos_index=1, eos_index=2, beam_size=4,
                min_decode_ratio=0.0, max_decode_ratio=1.0, temperature=1.0, using_eos_threshold=True,
                eos_threshold=1.5, length_normalization=True, minus_inf=-1e20, topk=1, prefix="", return_history=False,
                lm=None, ctc=None, return_topk=False, length_weight=0.0, forced=None, coverage=None):
    """S2STransformerBeamSearcher.forward, using_max_attn_shift=False; scorer=None, or a ScorerBuilder with full scorers
    TransformerLMScorer (``lm`` = dict(sd, cfg, weight, temperature, prefix)) and/or CTCScorer (``ctc`` = dict(w, b, weight,
    blank_index)), in the recipe's order [transformerlm, ctc] (scorer.py:1221-1268; conformer_large.yaml:209-223).

    Follows init_beam_search_data (:1267-1369), search_step (:1478-1598), _compute_scores_and_next_inp_tokens
    (:1204-1265), _update_sequences_and_log_probs (:1152-1202), _update_hyps_and_scores_if_eos_token (:1371-1416),
    _fill_alived_hyps_with_eos_token (:1600-1630), _get_topk_prediction (:1418-1476) -- whole-prefix decode, no cache.
    Returns (hyps, best_lens, best_scores, best_log_probs) like return_topk=False.

    ``forced`` (test helper, needs beam_size=1): a list of B token lists.  The search is walked along exactly these tokens
    (candidate = forced token instead of the top-1) and the function returns a (B,) tensor with the search score the
    reference assigns to each path at its last token -- used to judge a hypothesis the CUDA search found when fp16 rounding
    made it pick another near-tied hypothesis than the fp32 reference."""
    if forced is not None:
        assert beam_size == 1 and len(forced) == enc_states.shape[0]
        max_decode_ratio = (max(len(f) for f in forced) + 0.5) / enc_states.shape[1]
        forced_scores = torch.zeros(len(forced))
    B, T, _ = enc_states.shape
    V = seq_lin_w.shape[0]
    n_bh = B * beam_size
    enc_lens = torch.round(T * wav_len).int()
    enc = enc_states.repeat_interleave(beam_size, dim=0)
    enc_l = enc_lens.repeat_interleave(beam_size, dim=0)
    inp = torch.full((n_bh,), bos_index, dtype=torch.long)
    beam_offset = torch.arange(B) * beam_size
    seq_scores = torch.full((n_bh,), float("-inf"))
    seq_scores[beam_offset] = 0.0
    alived_seq = torch.empty(n_bh, 0, dtype=torch.long)
    alived_lp = torch.empty(n_bh, 0)
    finished = [[] for _ in range(B)]
    min_steps, max_steps = int(T * min_decode_ratio), int(T * max_decode_ratio)
    memory = None
    scores = None
    history = []
    attn_weight = 1.0
    ctc_state = ctc_mem = None
    if ctc is not None:  # seq2seq.py:791-804 (attn_weight = 1 - ctc_weight), scorer.py:243-249 (CTCScorer.reset_mem)
        assert len({bos_index, eos_index, ctc["blank_index"]}) == 3
        attn_weight = 1.0 - ctc["weight"]
        ctc_state = ctc_prefix_reset(F.log_softmax(F.linear(enc_states, ctc["w"], ctc["b"]), dim=-1), enc_lens,
                                     ctc["blank_index"], eos_index)

    def add_eos_hyps(tokens, scores_):
        is_eos = tokens.eq(eos_index)
        for index in torch.nonzero(is_eos, as_tuple=True)[0].tolist():
            b = index // beam_size
            if len(finished[b]) == beam_size:
                continue
            finished[b].append((alived_seq[index, :], alived_lp[index, :], scores_[index].clone()))
        return is_eos

    for step in range(max_steps):
        if forced is None and [len(f) for f in finished] == [beam_size] * B:
            break
        memory = inp.unsqueeze(1) if memory is None else torch.cat([memory, inp.unsqueeze(1)], dim=-1)
        pred, attn = decode(memory, enc, enc_l, sd, cfg, prefix)
        log_probs = F.log_softmax(F.linear(pred, seq_lin_w, seq_lin_b) / temperature, dim=-1)[:, -1, :]
        if ctc is not None:
            log_probs = attn_weight * log_probs  # _attn_weight_step (:916-921)
        lp_clone = log_probs.clone().reshape(B, -1)
        if step < min_steps:
            log_probs[:, eos_index] = minus_inf
        if using_eos_threshold:
            max_probs, _ = torch.max(log_probs, dim=-1)
            cond = log_probs[:, eos_index] > (eos_threshold * max_probs)
            log_probs[:, eos_index] = torch.where(cond, log_probs[:, eos_index], torch.tensor(minus_inf))
        if lm is not None:  # _scorer_step: the LM sees the same token prefix as the decoder (memory incl. inp)
            log_probs = log_probs + lm["weight"] * lm_scorer_log_probs(memory, lm["sd"], lm["cfg"], lm["temperature"],
                                                                      lm.get("prefix", ""))
        if ctc is not None:  # ScorerBuilder.score: block blank, add weight * (psi - psi_prev) over the full vocabulary
            log_probs[:, ctc["blank_index"]] = ctc_state["minus_inf"]
            ctc_score, ctc_mem = ctc_prefix_step(ctc_state, inp, ctc_mem, beam_size)
            log_probs = log_probs + ctc["weight"] * ctc_score
        if coverage is not None:  # CoverageScorer.score (scorer.py:880-922): attn (n_bh, s, T) of the last decoder layer
            cov = attn.sum(dim=1)
            penalty = torch.max(cov, cov.clone().fill_(coverage["threshold"])).sum(-1) - cov.size(-1) * coverage["threshold"]
            log_probs = log_probs + coverage["weight"] * (-penalty / (step + 1)).unsqueeze(1)
        if length_weight != 0.0:  # LengthScorer.score (scorer.py:1043-1071): ones * weight on every token
            log_probs = log_probs + length_weight
        sc = seq_scores.unsqueeze(1) + log_probs
        if length_normalization:
            sc = sc / (step + 1)
        scores, cand = sc.view(B, -1).topk(beam_size, dim=-1)
        if forced is not None:
            cand = torch.tensor([[f[step] if step < len(f) else eos_index] for f in forced])
            scores = sc.view(B, -1).gather(1, cand)
            for b_, f in enumerate(forced):
                if step == len(f) - 1:
                    forced_scores[b_] = scores[b_, 0]
        if ctc is not None:  # permute_scorer_mem: the CTC memory follows ``candidates`` (scorer.py:1286-1290)
            ctc_mem = ctc_prefix_permute(ctc_state, ctc_mem, cand)
        inp = (cand % V).view(n_bh)
        scores = scores.view(n_bh)
        seq_scores = scores * (step + 1) if length_normalization else scores.clone()
        predecessors = (torch.div(cand, V, rounding_mode="floor") + beam_offset.unsqueeze(1)).view(n_bh)
        memory = torch.index_select(memory, 0, predecessors)
        beam_lp = lp_clone[torch.arange(B).unsqueeze(1), cand].reshape(n_bh)
        alived_seq = torch.cat([torch.index_select(alived_seq, 0, predecessors), inp.unsqueeze(1)], dim=-1)
        alived_lp = torch.cat([torch.index_select(alived_lp, 0, predecessors), beam_lp.unsqueeze(1)], dim=-1)
        history.append((inp.clone(), predecessors.clone(), scores.clone(), beam_lp.clone()))
        if forced is not None:
            continue
        is_eos = add_eos_hyps(inp, scores)
        seq_scores = seq_scores.masked_fill(is_eos, float("-inf"))
    if forced is not None:
        return forced_scores
    if [len(f) for f in finished] != [beam_size] * B:
        add_eos_hyps(torch.full((n_bh,), eos_index, dtype=torch.long), scores)
    out = finalize_beams(finished, beam_size, topk, return_topk)
    return out + (history,) if return_history else out


def finalize_beams(finished, beam_size, topk=1, return_topk=False):
    """_get_topk_prediction (:1418-1476) + the tail of forward (:1709-1723): return_topk=True gives the padded
    (topk_hyps, topk_lengths, topk_scores, topk_log_probs), else (hyps, best_lens, best_scores, best_log_probs)."""
    B = len(finished)
    top_hyps, top_lp, top_scores, top_len = [], [], [], []
    for i in range(B):
        hyps, lps, scs = zip(*finished[i])
        top_hyps += hyps
        top_scores += scs
        top_lp += lps
        top_len += [len(h) for h in hyps]
    top_hyps = torch.nn.utils.rnn.pad_sequence(top_hyps, batch_first=True, padding_value=0)
    top_lp = torch.nn.utils.rnn.pad_sequence(top_lp, batch_first=True, padding_value=0)
    top_len = (torch.tensor(top_len, dtype=torch.float) - 1) / top_hyps.size(1)
    top_scores = torch.stack(top_scores, dim=0).view(B, -1)
    tk_scores, idx = top_scores.topk(topk, dim=-1)
    idx = (idx + (torch.arange(B) * beam_size).unsqueeze(1)).view(B * topk)
    tk_hyps = torch.index_select(top_hyps, 0, idx).view(B, topk, -1)
    tk_len = torch.index_select(top_len, 0, idx).view(B, topk)
    tk_lp = torch.index_select(top_lp, 0, idx).view(B, topk, -1)
    if return_topk:
        return tk_hyps, tk_len, tk_scores, tk_lp
    best_hyps, best_lens = tk_hyps[:, 0, :], tk_len[:, 0]
    hyps = [best_hyps[b, : int(torch.round(best_lens[b] * best_hyps.shape[1]))].tolist() for b in range(B)]
    return hyps, best_lens, tk_scores[:, 0], tk_lp[:, 0, :]


# --------------------------------------------------------------------------
# TransformerLM + TransformerLMScorer (shallow fusion): TransformerLM.py:22-187, Transformer.py:331-481,597-660,
# decoders/scorer.py:455-560 (score / permute_mem), :1221-1268 (ScorerBuilder.score, full scorers only)
# --------------------------------------------------------------------------


def transformer_lm_forward(tokens, sd, cfg, prefix=""):
    """TransformerLM.forward(src) for the recipe's LM: 12 post-norm TransformerEncoder layers (normalize_before=False),
    causal mask + key-padding mask on token id 0 (make_masks, pad_idx=0), final LayerNorm(1e-6), output_proj =
    Linear(d,d) -> LayerNorm(1e-6) -> Linear(d,vocab).  tokens (n, s) -> logits (n, s, vocab)."""
    n, s = tokens.shape
    d, H = cfg["d_model"], cfg["nhead"]
    x = F.embedding(tokens.long(), sd[prefix + "custom_src_module.emb.Embedding.weight"]) * math.sqrt(d)
    x = x + sine_pe(s, d).unsqueeze(0)
    causal = torch.triu(torch.full((s, s), float("-inf")), diagonal=1)
    kpm = tokens.long() == 0
    act = F.gelu if cfg.get("activation", "gelu") == "gelu" else F.relu
    for i in range(cfg["num_encoder_layers"]):
        p = f"{prefix}encoder.layers.{i}."
        h, _ = _mha_regular(x, x, {k.replace("self_att.", "A."): v for k, v in sd.items() if k.startswith(p + "self_att.")},
                            p + "A.", H, attn_mask=causal, key_padding_mask=kpm)
        x = _ln(x + h, sd, p + "norm1.norm.", 1e-6)
        h = F.linear(act(F.linear(x, sd[p + "pos_ffn.ffn.0.weight"], sd[p + "pos_ffn.ffn.0.bias"])),
                     sd[p + "pos_ffn.ffn.3.weight"], sd[p + "pos_ffn.ffn.3.bias"])
        x = _ln(x + h, sd, p + "norm2.norm.", 1e-6)
    x = _ln(x, sd, prefix + "encoder.norm.norm.", 1e-6)
    x = F.linear(x, sd[prefix + "output_proj.layers.0.w.weight"], sd[prefix + "output_proj.layers.0.w.bias"])
    x = _ln(x, sd, prefix + "output_proj.layers.1.norm.", 1e-6)
    return F.linear(x, sd[prefix + "output_proj.layers.2.w.weight"], sd[prefix + "output_proj.layers.2.w.bias"])


def lm_scorer_log_probs(memory_tokens, sd_lm, cfg_lm, temperature, prefix=""):
    """TransformerLMScorer.score (scorer.py:510-543): log_softmax(lm(memory) / temperature)[:, -1, :]."""
    logits = transformer_lm_forward(memory_tokens, sd_lm, cfg_lm, prefix)
    return F.log_softmax(logits / temperature, dim=-1)[:, -1, :]


# --------------------------------------------------------------------------
# CTC prefix scorer (joint CTC/attention decoding, full-vocabulary scoring): decoders/ctc.py:46-295 (CTCPrefixScore),
# decoders/scorer.py:183-249 (CTCScorer); ctc_window_size = 0 and candidates = None (the recipe's full scorer).
# --------------------------------------------------------------------------


def ctc_prefix_reset(x, enc_lens, blank_index, eos_index, minus_inf=-1e20):
    """CTCPrefixScore.__init__ (ctc.py:46-78): x = log_softmax(ctc_lin(enc)) (B, T, V); frames >= enc_len get minus_inf for
    every non-blank token and 0 for the blank (x[:, :, 0] is hard-coded there, i.e. the blank must be index 0)."""
    B, T, V = x.shape
    x = x.clone()
    pad = ~(torch.arange(T).unsqueeze(0) < enc_lens.unsqueeze(1))  # (B, T)
    x.masked_fill_(pad.unsqueeze(-1), minus_inf)
    x[:, :, 0] = x[:, :, 0].masked_fill(pad, 0.0)
    return dict(x_nb=x.transpose(0, 1).contiguous(),  # (T, B, V)
                x_b=x[:, :, blank_index].transpose(0, 1).contiguous(),  # (T, B)
                last=(enc_lens - 1).long(), blank=blank_index, eos=eos_index, minus_inf=minus_inf, prefix_length=-1,
                B=B, T=T, V=V)


def ctc_prefix_step(st, last_char, states, beam_size):
    """CTCPrefixScore.forward_step (ctc.py:80-249), candidates=None.  states = (r_prev (T, 2, n_bh), psi_prev (n_bh, V)) or
    None.  Returns (psi - psi_prev, (r (T, 2, n_bh, V), psi (n_bh, V)))."""
    T, B, V, NEG = st["T"], st["B"], st["V"], st["minus_inf"]
    n_bh = last_char.shape[0]
    st["prefix_length"] += 1
    pl = st["prefix_length"]
    if states is None:
        r_prev = torch.full((T, 2, B, beam_size), NEG)
        r_prev[:, 1] = torch.cumsum(st["x_nb"][:, :, st["blank"]], 0).unsqueeze(2)
        r_prev = r_prev.view(T, 2, n_bh)
        psi_prev = torch.zeros(n_bh, V)
    else:
        r_prev, psi_prev = states
    x_nb = st["x_nb"].repeat_interleave(beam_size, dim=1)  # (T, n_bh, V)
    x_b = st["x_b"].repeat_interleave(beam_size, dim=1).unsqueeze(-1)  # (T, n_bh, 1)
    r = torch.full((T, 2, n_bh, V), NEG)
    if pl == 0:
        r[0, 0] = x_nb[0]
    r_sum = torch.logsumexp(r_prev, 1)  # (T, n_bh)
    phi = r_sum.unsqueeze(2).repeat(1, 1, V)
    rows = torch.arange(n_bh)
    phi[:, rows, last_char] = r_prev[:, 1, :]
    start, end = max(1, pl), T
    for t in range(start, end):
        rnb, rb = r[t - 1, 0], r[t - 1, 1]
        r[t, 0] = torch.logsumexp(torch.stack([rnb, phi[t - 1]]), 0) + x_nb[t]
        r[t, 1] = torch.logsumexp(torch.stack([rnb, rb]), 0) + x_b[t]
    psi_init = r[start - 1, 0].unsqueeze(0)
    phix = torch.cat((phi[0].unsqueeze(0), phi[:-1]), dim=0) + x_nb
    psi = torch.logsumexp(torch.cat((phix[start:end], psi_init), dim=0), dim=0)
    psi[rows, st["eos"]] = r_sum[st["last"].repeat_interleave(beam_size), rows]
    if st["eos"] != st["blank"]:
        psi[:, st["blank"]] = NEG
    return psi - psi_prev, (r, psi)


def ctc_prefix_permute(st, memory, cand):
    """CTCPrefixScore.permute_mem (ctc.py:251-295) for scoring_table=None: ``cand`` (B, beam) indexes beam*V per batch."""
    r, psi = memory
    V, T = st["V"], st["T"]
    B, beam = cand.shape
    n_bh = B * beam
    off = (torch.arange(B) * beam).unsqueeze(1)
    cand_index = (cand + off * V).view(n_bh)
    psi_sel = psi.reshape(-1)[cand_index].view(-1, 1).repeat(1, V)
    r_sel = r.reshape(T, 2, n_bh * V)[:, :, cand_index]
    return r_sel, psi_sel


def ctc_prefix_scores(logits, enc_len, beam, blank, bos, eos, hist_tok, hist_pred, n_steps, minus_inf=-1e20, chunk=256,
                      pick=None):
    """The CTC prefix scorer along a forced search history, in float64: CTCPrefixScore.__init__ + n_steps x (forward_step,
    permute_mem) (ctc.py:46-295), candidates = None.  Same inputs as the sbk_ctc_prefix_test hook: ``logits`` (B, T, V)
    ctc_lin output before log_softmax, ``enc_len`` (B,) in [0, T], ``hist_tok`` / ``hist_pred`` (>= n_steps - 1, B * beam)
    int tensors: token and global parent row of every hypothesis after each step.  With ``pick`` the history is chosen on
    the way: ``pick(s, score_s, last_tokens)`` returns row s of (hist_tok, hist_pred), which are filled in place.

    Unlike ctc_prefix_step it never materialises the (T, 2, n_bh, V) forward variables: psi(h, c) = logsumexp over frames
    of phi_h[t - 1] + x[t, c] (Alg.2-13, plus the seed x[0, c] at step 0) is evaluated directly, token chunk by token chunk,
    and the recurrence (Alg.2-11/12) runs only for the (parent, token) pairs the history keeps.  So it scales to T = 10240
    and V = 5000.  It follows the reference's start = max(1, prefix_length), its padded frames (minus_inf everywhere but 0
    in channel 0, ctc.py:59-62), its eos column r_sum[enc_len - 1] (a Python index: enc_len = 0 reads frame T - 1) and its
    blank column.

    Returns a dict of float64 tensors: ``score`` (n_steps, n_bh, V) = psi - psi_prev, ``psi`` (same shape), ``psi_prev``
    (n_steps, n_bh), and ``low`` (n_steps, n_bh, V) bool: entries whose largest term lies more than 69 + log(T) nats below
    the maximum of the phi variant it uses -- where a linear-domain sum of exp(phi - max) * exp(x) underflows fp32."""
    x = torch.log_softmax(logits.double(), dim=-1)
    B, T, V = x.shape
    n_bh = B * beam
    enc_len = enc_len.long()
    pad = ~(torch.arange(T).unsqueeze(0) < enc_len.unsqueeze(1))
    x = x.masked_fill(pad.unsqueeze(-1), minus_inf)
    x[:, :, 0] = x[:, :, 0].masked_fill(pad, 0.0)
    xb = x[:, :, blank]                                   # (B, T)
    last_frame = torch.where(enc_len > 0, enc_len - 1, T - 1)
    utt = torch.arange(n_bh) // beam
    neg = torch.tensor(minus_inf, dtype=torch.float64)
    # states = None (ctc.py:108-123)
    r_nb = torch.full((n_bh, T), minus_inf, dtype=torch.float64)
    r_b = torch.cumsum(xb, dim=1)[utt]
    psi_prev = torch.zeros(n_bh, dtype=torch.float64)
    score = torch.empty(n_steps, n_bh, V, dtype=torch.float64)
    psi_all = torch.empty(n_steps, n_bh, V, dtype=torch.float64)
    prev_all = torch.empty(n_steps, n_bh, dtype=torch.float64)
    low = torch.zeros(n_steps, n_bh, V, dtype=torch.bool)
    thr = -69.0 - math.log(T)
    for s in range(n_steps):
        last = torch.full((n_bh,), bos, dtype=torch.long) if s == 0 else hist_tok[s - 1].long()
        r_sum = torch.logaddexp(r_nb, r_b)                # (n_bh, T)
        start = max(1, s)
        psi = torch.empty(n_bh, V, dtype=torch.float64)
        for b in range(B):
            rows = slice(b * beam, (b + 1) * beam)
            for var, phi_all in ((0, r_sum), (1, r_b)):   # variant 1: phi = r_b for the row's last token (Alg.2-10)
                phi = phi_all[rows, start - 1:T - 1]      # phi[t - 1] for t in [start, T)
                m = phi.max(dim=1).values if phi.shape[1] else torch.full((beam,), -math.inf, dtype=torch.float64)
                if s == 0:
                    m = torch.maximum(m, torch.zeros_like(m))  # the seed term: phi = 0 before frame 0
                for c0 in range(0, V, chunk):
                    xc = x[b, start:, c0:c0 + chunk]      # (T - start, C)
                    terms = phi.unsqueeze(2) + xc.unsqueeze(0)
                    seed = x[b, 0, c0:c0 + chunk].expand(beam, -1) if s == 0 else neg.expand(beam, xc.shape[1])
                    allt = torch.cat([terms, seed.unsqueeze(1)], dim=1)
                    val = torch.logsumexp(allt, dim=1)
                    if s == 0 or terms.shape[1]:          # largest term of the sum, relative to the variant's maximum
                        top = allt.max(dim=1).values if s == 0 else terms.max(dim=1).values
                        top = top - m.unsqueeze(1)
                    else:                                  # no frame left: an empty sum
                        top = torch.zeros_like(val)
                    cols = torch.arange(c0, c0 + xc.shape[1])
                    sel = (last[rows].unsqueeze(1) == cols.unsqueeze(0))
                    if var == 0:
                        psi[rows, c0:c0 + chunk] = val
                        low[s, rows, c0:c0 + chunk] = top < thr
                    else:
                        psi[rows, c0:c0 + chunk] = torch.where(sel, val, psi[rows, c0:c0 + chunk])
                        low[s, rows, c0:c0 + chunk] = torch.where(sel, top < thr, low[s, rows, c0:c0 + chunk])
        psi[:, eos] = r_sum[torch.arange(n_bh), last_frame[utt]]   # Alg.2-3
        if eos != blank:
            psi[:, blank] = minus_inf
        low[s, :, eos] = False
        low[s, :, blank] = False
        score[s] = psi - psi_prev.unsqueeze(1)
        psi_all[s] = psi
        prev_all[s] = psi_prev
        if s + 1 == n_steps:
            break
        if pick is not None:
            tok_s, par_s = pick(s, score[s], last)
            hist_tok[s], hist_pred[s] = tok_s, par_s
        # permute_mem: forward variables of the kept (parent, token) pairs only (Alg.2-11/12)
        par, tok = hist_pred[s].long(), hist_tok[s].long()
        bu = utt[par]
        xn = x[bu, :, tok]                                # (n_bh, T)
        phi = torch.where((tok == last[par]).unsqueeze(1), r_b[par], r_sum[par])
        nb = torch.full((n_bh, T), minus_inf, dtype=torch.float64)
        bl = torch.full((n_bh, T), minus_inf, dtype=torch.float64)
        if s == 0:
            nb[:, 0] = xn[:, 0]
        xbu = xb[bu]
        for t in range(start, T):
            nb[:, t] = torch.logaddexp(nb[:, t - 1], phi[:, t - 1]) + xn[:, t]
            bl[:, t] = torch.logaddexp(nb[:, t - 1], bl[:, t - 1]) + xbu[:, t]
        r_nb, r_b = nb, bl
        psi_prev = psi[par, tok]
    return dict(score=score, psi=psi_all, psi_prev=prev_all, low=low, hist_tok=hist_tok, hist_pred=hist_pred)


def ctc_history_picker(B, beam, V, blank, eos, seed):
    """A ``pick`` for ctc_prefix_scores that makes search-like histories: parents drawn within each utterance with
    replacement (some parents get several children, some none; slots 0 and 1 always share one), and tokens that cycle
    through the parent's best-scoring token, the parent's own last token (phi = r_b, Alg.2-10) and a random token.
    Never blank or eos (those end or void a prefix)."""
    gen = torch.Generator().manual_seed(seed)
    banned = torch.zeros(V, dtype=torch.bool)
    banned[[blank, eos]] = True
    allowed = (~banned).nonzero().squeeze(1)

    def pick(s, score, last):
        tok = torch.empty(B * beam, dtype=torch.int32)
        par = torch.empty(B * beam, dtype=torch.int32)
        for b in range(B):
            loc = torch.randint(0, beam, (beam,), generator=gen)
            if beam >= 2:
                loc[1] = loc[0]
            for k in range(beam):
                p = b * beam + int(loc[k])
                kind = (k + s) % 3
                if kind == 1 and not banned[int(last[p])]:
                    t = int(last[p])
                elif kind == 0:
                    t = int(score[p].masked_fill(banned, -math.inf).argmax())
                else:
                    t = int(allowed[torch.randint(0, allowed.numel(), (1,), generator=gen)])
                tok[b * beam + k], par[b * beam + k] = t, p
        return tok, par
    return pick


# --------------------------------------------------------------------------
# TransformerLMRescorer.rescore_hyps (decoders/scorer.py:1793-1882) + RescorerBuilder.rescore (:2113-2162)
# --------------------------------------------------------------------------


class StubTokenizer:
    """Stands in for the sentencepiece processor the recipes pass (only ``encode_as_ids`` is called, scorer.py:1817):
    one id per character, ids in [3, 4993), deterministic."""

    def encode_as_ids(self, text):
        return [3 + (ord(ch) * 131) % 4990 for ch in text]


def lm_rescore_hyps(topk_hyps, tokenizer, sd_lm, cfg_lm, temperature=1.0, bos_index=0, eos_index=0, pad_index=0, prefix=""):
    """preprocess_func (:1793-1833: upper-case, bos + ids + eos, pad) then rescore_hyps (:1835-1882): one LM forward over the
    padded batch, log-softmax(logits / T) with the pad column at -inf and renormalised, sum of the target log-probs over the
    valid positions (nansum)."""
    enc = [torch.tensor([bos_index] + tokenizer.encode_as_ids(seq.upper()) + [eos_index]) for batch in topk_hyps for seq in batch]
    lengths = torch.tensor([e.shape[0] for e in enc])
    padded = torch.nn.utils.rnn.pad_sequence(enc, batch_first=True, padding_value=pad_index)
    logits = transformer_lm_forward(padded, sd_lm, cfg_lm, prefix)
    log_probs = F.log_softmax(logits / temperature, dim=-1)
    log_probs[:, :, pad_index] = float("-inf")
    tgt = log_probs[:, :-1].gather(2, padded[:, 1:].unsqueeze(2)).squeeze(2)
    tgt = tgt - log_probs[:, :-1].logsumexp(dim=-1)
    mask = torch.arange(padded.shape[1]).unsqueeze(0) < lengths.unsqueeze(1)
    return torch.nansum(tgt * mask[:, 1:], dim=-1)


def rescorer_builder_rescore(topk_candidates, topk_scores, lm_scores, weight):
    """RescorerBuilder.rescore (:2113-2162) with one rescorer: add weight * score, sort each utterance's candidates."""
    new_scores = [list(r) for r in topk_scores]
    it = iter(lm_scores.tolist())
    for i in range(len(new_scores)):
        for j in range(len(new_scores[i])):
            new_scores[i][j] += weight * next(it)
    out_c, out_s = [], []
    for cands, scs in zip(topk_candidates, new_scores):
        order = sorted(zip(cands, scs), key=lambda x: x[1], reverse=True)
        out_c.append([c for c, _ in order])
        out_s.append([s_ for _, s_ in order])
    return out_c, out_s


# --------------------------------------------------------------------------
# EncoderASR CTC greedy decoding: inference/ASR.py:325-373, decoders/ctc.py:298-378
# --------------------------------------------------------------------------


def ctc_log_probs(enc, w, b):
    """The tail of the recipe's encoder Sequential: log_softmax(ctc_lin(enc)) (B, T, V)."""
    return F.log_softmax(F.linear(enc, w, b), dim=-1)


def ctc_greedy_decode(log_probs, seq_lens, blank_id):
    """decoders/ctc.py:335-378 + filter_ctc_output (:298-332): per-frame arg-max over the first round(len * T) frames, merge
    repetitions, drop blanks."""
    T = log_probs.shape[1]
    out = []
    for seq, rel in zip(log_probs, seq_lens):
        n = int(torch.round(rel * T))
        pred = seq[:n].argmax(-1).tolist()
        merged = [t for i, t in enumerate(pred) if i == 0 or t != pred[i - 1]]
        out.append([t for t in merged if t != blank_id])
    return out
