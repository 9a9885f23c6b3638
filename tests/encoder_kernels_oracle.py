"""float64 references of the two per-layer encoder kernels that the device hooks expose alone:

- attention_ref: encoder_attention_kernel (sbk_encoder_attention_test), RoPE / regularMHA and RelPosMHAXL, with the key
  padding mask and Dynamic Chunk windows;
- dwconv_ref: dwconv_ln_swish_kernel (sbk_dwconv_test), the Conformer convolution module's depthwise conv, LayerNorm and
  SiLU, with the Dynamic Chunk Convolution limit.

They take the inputs the kernels receive (fp16 q/k/v/P, fp32 pos_u/pos_v, fp32 GLU output and weights) in float64 and work
on whatever device those tensors are on.  test_encoder_kernels_oracle.py pins them to oracle.asr_oracle.relpos_mha,
rope_mha and conv_module (which make_goldens.py pins to the running reference) to 1e-10."""
import torch
import torch.nn.functional as F

from oracle.asr_oracle import chunk_mask


def visible_keys(T, lens, B, chunk=0, left_chunks=-1, device=None):
    """[B, T, T] bool, True = query i of utterance b sees key j: j < len_b and, with chunk > 0, the chunk window of
    oracle.asr_oracle.chunk_mask (left_chunks < 0 = the whole past)."""
    lens = torch.full((B,), T) if lens is None else lens.cpu().clamp(max=T)
    vis = (torch.arange(T).view(1, 1, T) < lens.view(B, 1, 1)).expand(B, T, T)
    if chunk > 0:
        vis = vis & ~chunk_mask(T, chunk, None if left_chunks < 0 else left_chunks).view(1, T, T)
    return vis.to(device)


def attention_ref(q, k, v, lens=None, P=None, pos_u=None, pos_v=None, scale=1.0, chunk=0, left_chunks=-1):
    """q, k, v [B, T, H, dh] -> out [B, T, H, dh] float64.

    P is None: scores = q.k^T (q already scaled, scale unused).
    Else RelPosMHAXL: scores = ((q + u).k^T + (q + v).P[|i - j|]^T) * scale, P [T, H * dh] (row r = distance r),
    pos_u / pos_v [H * dh].  Keys j >= len and keys outside the chunk window are masked; a row that sees no key is 0
    (RelPosMHAXL's post-softmax masked_fill).  Computed per (utterance, head): no [B, H, T, 2T] tensor."""
    B, T, H, dh = q.shape
    q, k, v = q.double(), k.double(), v.double()
    vis = visible_keys(T, lens, B, chunk, left_chunks, q.device)
    out = torch.zeros(B, T, H, dh, dtype=torch.float64, device=q.device)
    if P is not None:
        Ph = P.double().view(T, H, dh)
        u, w = pos_u.double().view(H, dh), pos_v.double().view(H, dh)
        i = torch.arange(T, device=q.device)
        dist = (i.view(T, 1) - i.view(1, T)).abs()
    for b in range(B):
        for h in range(H):
            qh, kh, vh = q[b, :, h], k[b, :, h], v[b, :, h]
            if P is None:
                s = qh @ kh.T
            else:
                bd = (qh + w[h]) @ Ph[:, h].T           # [T, T]: column r = distance r
                s = ((qh + u[h]) @ kh.T + bd.gather(1, dist)) * scale
            s = s.masked_fill(~vis[b], float("-inf"))
            a = torch.softmax(s, dim=-1).nan_to_num(0.0)  # rows without a visible key: 0
            out[b, :, h] = a @ vh
    return out


def dwconv_ref(x, taps, bias, ln_g, ln_b, chunk=0, eps=1e-5):
    """x [B, T, D] (GLU output) -> SiLU(LayerNorm(Conv1d_K(x) + bias)) float64, taps [D, 1, K].  The conv is 'same' with
    zero padding outside [0, T) only: padded frames inside T are inputs.  chunk > 0: for output frame t the inputs at or
    past the end of its chunk, (t // chunk + 1) * chunk, count as zero (oracle.asr_oracle.conv_module)."""
    B, T, D = x.shape
    K = taps.shape[-1]
    pad = (K - 1) // 2
    x, taps, bias = x.double(), taps.double(), bias.double()
    if chunk <= 0:
        h = F.conv1d(x.transpose(1, 2), taps, bias, padding=pad, groups=D).transpose(1, 2)
    else:
        t = torch.arange(T, device=x.device)
        end = (t // chunk + 1) * chunk
        xp = F.pad(x, (0, 0, pad, pad))
        h = bias.view(1, 1, D).expand(B, T, D).clone()
        for kk in range(K):
            ok = (t + kk - pad < end).view(1, T, 1)
            h = h + torch.where(ok, xp[:, kk:kk + T], torch.zeros((), dtype=x.dtype, device=x.device)) * taps[:, 0, kk]
    h = F.layer_norm(h, (D,), ln_g.double(), ln_b.double(), eps)
    return F.silu(h)
