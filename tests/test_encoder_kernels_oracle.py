"""The float64 kernel references of encoder_kernels_oracle.py against the CPU oracle (oracle.asr_oracle), which
make_goldens.py pins to the running reference: relpos_mha, rope_mha and conv_module on small random float64 weights, with
out_proj / after_conv.2 set to the identity so that the oracle returns the attention output / the conv-LN-SiLU output.
The references get the oracle's own projected q/k/v/P (or GLU output), so the rel-shift, the roles of pos_bias_u and
pos_bias_v, the masks and the chunk windows are checked to be the reference's, not a restatement of the kernel."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import encoder_kernels_oracle as EK  # noqa: E402
from oracle import asr_oracle as O  # noqa: E402

TOL = 1e-10
# (chunk, left_chunks) windows; None = full context
WINDOWS = [None, (1, 0), (4, None), (5, 1), (16, 0), (7, 2)]


def _attn_state(d, H, g):
    dh = d // H
    return {"in_proj_weight": torch.randn(3 * d, d, generator=g, dtype=torch.float64) / math.sqrt(d),
            "linear_pos.weight": torch.randn(d, d, generator=g, dtype=torch.float64) / math.sqrt(d),
            "pos_bias_u": torch.randn(dh, H, generator=g, dtype=torch.float64),
            "pos_bias_v": torch.randn(dh, H, generator=g, dtype=torch.float64),
            "out_proj.weight": torch.eye(d, dtype=torch.float64), "out_proj.bias": torch.zeros(d, dtype=torch.float64)}


def _masks(T, lens, window):
    kpm = ~O.length_to_mask(lens, T)
    amask = None if window is None else O.chunk_mask(T, window[0], window[1])
    return kpm, amask


def _kernel_window(window):
    return (0, -1) if window is None else (window[0], -1 if window[1] is None else window[1])


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("T", [1, 37, 70])
def test_relpos_reference_vs_oracle(T, window):
    B, H, d = 3, 2, 16
    dh = d // H
    g = torch.Generator().manual_seed(T * 31 + (0 if window is None else window[0] * 7 + (window[1] or 9)))
    sd = _attn_state(d, H, g)
    x = torch.randn(B, T, d, generator=g, dtype=torch.float64)
    lens = torch.tensor([T, max(1, (2 * T) // 3), max(1, T // 6)])
    kpm, amask = _masks(T, lens, window)
    pos = O.relpos_table(T, d).double()
    ref = O.relpos_mha(x, pos, sd, "", H, kpm, attn_mask=amask)
    qkv = (x @ sd["in_proj_weight"].T).view(B, T, H, 3 * dh)
    q, k, v = qkv.chunk(3, dim=-1)
    p_k = (pos @ sd["linear_pos.weight"].T)[0]            # rows = relative positions T-1, ..., 0, ..., -(T-1)
    P = p_k[T - 1 - torch.arange(T)]                       # row r = distance r
    chunk, left = _kernel_window(window)
    out = EK.attention_ref(q, k, v, lens, P, sd["pos_bias_u"].reshape(-1), sd["pos_bias_v"].reshape(-1), 1.0 / math.sqrt(d),
                           chunk, left).reshape(B, T, d)
    assert torch.isfinite(ref).all()
    assert float((out - ref).abs().max()) <= TOL
    if window == (1, 0):  # padded query rows of a short utterance see no key: 0 in both
        assert T == 1 or (ref[2, int(lens[2]):] == 0).all()


@pytest.mark.parametrize("window", WINDOWS)
@pytest.mark.parametrize("T", [1, 37, 70])
def test_rope_reference_vs_oracle(T, window):
    B, H, d = 3, 2, 16
    dh = d // H
    g = torch.Generator().manual_seed(T * 17 + (0 if window is None else window[0] * 5 + (window[1] or 3)))
    sd = _attn_state(d, H, g)
    x = torch.randn(B, T, d, generator=g, dtype=torch.float64)
    lens = torch.tensor([T, max(1, (2 * T) // 3), max(1, T // 6)])
    kpm, amask = _masks(T, lens, window)
    ref = O.rope_mha(x, sd, "", H, kpm, attn_mask=amask)
    qkv = (x @ sd["in_proj_weight"].T).view(B, T, H, 3 * dh)
    q, k, v = qkv.chunk(3, dim=-1)
    q, k = O.rope_rotate(q) / math.sqrt(d), O.rope_rotate(k)   # the kernel receives rotated, pre-scaled q
    chunk, left = _kernel_window(window)
    out = EK.attention_ref(q, k, v, lens, chunk=chunk, left_chunks=left).reshape(B, T, d)
    seen = EK.visible_keys(T, lens, B, chunk, left).any(-1)   # SDPA gives NaN for a row without a visible key
    assert torch.isfinite(ref[seen]).all() and not torch.isfinite(ref[~seen]).any()
    assert float((out[seen] - ref[seen]).abs().max()) <= TOL
    assert (out[~seen] == 0).all()


@pytest.mark.parametrize("chunk", [None, 1, 4, 5, 16])
@pytest.mark.parametrize("T,K", [(1, 31), (7, 15), (37, 31), (40, 3), (70, 15)])
def test_dwconv_reference_vs_oracle(T, K, chunk):
    B, d = 2, 12
    g = torch.Generator().manual_seed(T * 13 + K + (chunk or 0))
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    sd = {"layer_norm.weight": 1 + 0.1 * r(d), "layer_norm.bias": 0.1 * r(d),
          "bottleneck.0.weight": r(2 * d, d, 1) / math.sqrt(d), "bottleneck.0.bias": 0.1 * r(2 * d),
          "conv.weight": r(d, 1, K) / math.sqrt(K), "conv.bias": 0.1 * r(d),
          "after_conv.0.weight": 1 + 0.1 * r(d), "after_conv.0.bias": 0.1 * r(d),
          "after_conv.2.weight": torch.eye(d, dtype=torch.float64), "after_conv.2.bias": torch.zeros(d, dtype=torch.float64)}
    x = r(B, T, d)
    ref = O.conv_module(x, sd, "", None, chunk_size=chunk)
    h = F.layer_norm(x, (d,), sd["layer_norm.weight"], sd["layer_norm.bias"], 1e-5)
    glu = F.glu(F.linear(h, sd["bottleneck.0.weight"][:, :, 0], sd["bottleneck.0.bias"]), dim=-1)
    out = EK.dwconv_ref(glu, sd["conv.weight"], sd["conv.bias"], sd["after_conv.0.weight"], sd["after_conv.0.bias"], chunk or 0)
    assert float((out - ref).abs().max()) <= TOL
