"""-m gpu tests of the persistent wide-tile GEMM (gemm_tc2.cu, N % 256 == 0): every fused epilogue at the encoder's row
count (M = 8032 = 32 x 251 frames: 62 full 128-row tiles and a 96-row tail, several tiles per CTA), the M tail and M < 128,
K not a multiple of 64, and the all-layer cross-attention K/V launch against one launch per layer."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401

pytestmark = pytest.mark.gpu

EPI_F16, EPI_F32, EPI_RESID, EPI_GLU, EPI_ROPE = 0, 1, 2, 3, 4
ACT_NONE, ACT_SILU, ACT_GELU = 0, 1, 2


def _operands(dev, M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).half()
    W = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    bias = torch.randn(N, generator=g)
    A, W, bias = A.to(dev), W.to(dev), bias.to(dev)
    acc = A.double() @ W.double().T + bias.double()  # fp16 operands are exact in double
    return A, W, bias, acc


def _gemm(A, W, bias, out, ldo, mode, M, N, K, act=ACT_NONE, alpha=1.0, resid=None, row_lens=None, T=1, cos=None, sin=None,
          head_dim=64, kv_heads=0, kv_part_stride=0, kv_layer_stride=0):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    check(lib().sbk_gemm_epilogue_test(ptr(A), ptr(W), ptr(bias), ptr(out), ldo, mode, act, ctypes.c_float(alpha), ptr(resid),
                                       ptr(row_lens), T, ptr(cos), ptr(sin), head_dim, kv_heads,
                                       ctypes.c_longlong(kv_part_stride), ctypes.c_longlong(kv_layer_stride), M, N, K,
                                       stream_ptr(A.device)), "gemm epilogue")
    torch.cuda.synchronize()


def _assert_close(got, ref, atol, rtol, what):
    err = (got.double() - ref).abs()
    bad = err > atol + rtol * ref.abs()
    print(f"{what}: max abs err {err.max().item():.3e}")
    assert not bad.any(), f"{what}: {int(bad.sum())} elements out of tolerance, max abs err {err.max().item():.3e}"


# M = 8032 with N = 2048 is 63 x 16 = 1008 tiles of 128 x 128: far more than one per CTA of the persistent grid
@pytest.mark.parametrize("M,N,K", [(8032, 2048, 512), (8032, 512, 2048), (8032, 1024, 144), (37, 512, 640), (200, 256, 144),
                                   (128, 256, 64)])
@pytest.mark.parametrize("mode,act", [(EPI_F16, ACT_NONE), (EPI_F16, ACT_SILU), (EPI_F16, ACT_GELU), (EPI_F32, ACT_NONE)])
def test_wide_gemm_plain(dev, M, N, K, mode, act):
    A, W, bias, acc = _operands(dev, M, N, K, M + 3 * N + 7 * K + mode + 11 * act)
    out = torch.full((M, N), float("nan"), device=dev, dtype=torch.float32 if mode == EPI_F32 else torch.float16)
    _gemm(A, W, bias, out, N, mode, M, N, K, act=act)
    ref = acc
    if act == ACT_SILU:
        ref = torch.nn.functional.silu(acc)
    elif act == ACT_GELU:
        ref = torch.nn.functional.gelu(acc)
    if mode == EPI_F32:
        _assert_close(out, ref, 2e-3, 0.0, f"f32 M={M} N={N} K={K}")
    else:  # fp16 rounding; SiLU through tanh.approx (abs. error ~5e-4 of the tanh)
        _assert_close(out, ref, 5e-3, 2e-3, f"f16 act={act} M={M} N={N} K={K}")


@pytest.mark.parametrize("M,N,K", [(8032, 512, 512), (8032, 512, 2048), (37, 512, 144)])
def test_wide_gemm_residual_row_lens(dev, M, N, K):
    """x = x + alpha * (A W^T + b) in place; rows t >= row_lens[utt] keep x (conv pw2's masked_fill of padded frames)."""
    T = 251 if M % 251 == 0 else M
    B = M // T
    A, W, bias, acc = _operands(dev, M, N, K, 5 * M + N + K)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(M, N, generator=g).to(dev)
    lens = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    lens[0] = T
    lens = lens.to(dev)
    keep = (torch.arange(T, device=dev)[None, :] < lens[:, None]).reshape(M, 1).double()
    ref = x.double() + 0.5 * keep * acc
    _gemm(A, W, bias, x, N, EPI_RESID, M, N, K, alpha=0.5, resid=x, row_lens=lens, T=T)
    _assert_close(x, ref, 2e-3, 0.0, f"resid M={M} N={N} K={K}")


@pytest.mark.parametrize("M", [8032, 37])
def test_wide_gemm_glu(dev, M):
    N, K = 2048, 512
    A, W, bias, acc = _operands(dev, M, N, K, 17 + M)
    out = torch.full((M, N // 2), float("nan"), device=dev)
    _gemm(A, W, bias, out, N // 2, EPI_GLU, M, N, K)
    v = acc.view(M, N // 32, 2, 16)
    ref = (v[:, :, 0] * torch.sigmoid(v[:, :, 1])).reshape(M, N // 2)
    _assert_close(out, ref, 5e-3, 2e-3, f"glu M={M}")


@pytest.mark.parametrize("M", [8032, 37])
def test_wide_gemm_rope(dev, M):
    """QKV projection: per head [q | k | v] columns; q and k rotated pairwise by the frame's angle, q scaled by alpha."""
    N, K, dh = 1536, 512, 64
    T = 251 if M % 251 == 0 else M
    A, W, bias, acc = _operands(dev, M, N, K, 29 + M)
    ang = torch.arange(T, dtype=torch.float64)[:, None] * (10000.0 ** (-torch.arange(dh // 2, dtype=torch.float64) * 2 / dh))
    cos, sin = torch.cos(ang).float().to(dev), torch.sin(ang).float().to(dev)
    out = torch.full((M, N), float("nan"), device=dev, dtype=torch.float16)
    alpha = 0.125
    _gemm(A, W, bias, out, N, EPI_ROPE, M, N, K, alpha=alpha, T=T, cos=cos, sin=sin, head_dim=dh)
    t = torch.arange(M, device=dev) % T
    c, s = cos.double()[t][:, None, :], sin.double()[t][:, None, :]
    x = acc.view(M, N // (3 * dh), 3, dh // 2, 2)
    ref = x.clone()
    for sect, sc in ((0, alpha), (1, 1.0)):
        x0, x1 = x[:, :, sect, :, 0], x[:, :, sect, :, 1]
        ref[:, :, sect, :, 0] = (x0 * c - x1 * s) * sc
        ref[:, :, sect, :, 1] = (x1 * c + x0 * s) * sc
    _assert_close(out, ref.reshape(M, N), 4e-3, 2e-3, f"rope M={M}")


@pytest.mark.parametrize("M,T", [(8032, 251), (200, 100)])
def test_cross_kv_all_layers_one_launch(dev, M, T):
    """The decoder's cross-attention K/V of all layers in one N = layers * 2d GEMM equals one N = 2d GEMM per layer, element
    for element, in the head-major [layer][K|V][utt][head][t][64] layout."""
    L, H = 6, 8
    d = H * 64
    A, W, bias, acc = _operands(dev, M, L * 2 * d, d, 41 + M)
    merged = torch.full((L, 2, M * d), float("nan"), device=dev, dtype=torch.float16)
    _gemm(A, W, bias, merged, L * 2 * d, EPI_F16, M, L * 2 * d, d, T=T, kv_heads=H, kv_part_stride=M * d,
          kv_layer_stride=M * 2 * d)
    per_layer = torch.full_like(merged, float("nan"))
    for l in range(L):
        _gemm(A, W[l * 2 * d:(l + 1) * 2 * d], bias[l * 2 * d:(l + 1) * 2 * d], per_layer[l], 2 * d, EPI_F16, M, 2 * d, d,
              T=T, kv_heads=H, kv_part_stride=M * d)
    assert torch.equal(merged, per_layer)
    ref = acc.view(M // T, T, L, 2, H, 64).permute(2, 3, 0, 4, 1, 5).reshape(L, 2, M * d)
    _assert_close(merged, ref, 4e-3, 2e-3, f"cross K/V M={M}")
