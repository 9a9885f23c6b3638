"""-m gpu parity tests of the two per-layer encoder kernels alone, against the float64 references of
encoder_kernels_oracle.py (pinned to the CPU oracle by test_encoder_kernels_oracle.py):

- encoder_attention_kernel through sbk_encoder_attention_test: head widths 64, 36 (zero-padded to 48), 32 and 128; RoPE /
  regularMHA and RelPosMHAXL; the last-key-block padding mask; Dynamic Chunk windows with and without left context;
  RelPosMHAXL up to T = 2500 (max_len);
- dwconv_ln_swish_kernel through sbk_dwconv_test: the register-tap path (K = 31, 1, 2 or 4 channels per thread) and the
  runtime-K path, with and without the Dynamic Chunk Convolution limit.

The inputs are built to expose a subtly wrong kernel: logits with a standard deviation of about 3 (peaked rows); a RelPos
position term about as large as the content term, with distinct random P rows per distance; pos_bias_u != pos_bias_v;
K / V of padded frames at about +-3e4, so that one key that should be masked and is not dominates its row; asymmetric random
conv taps; every row < T compared, padded query rows included.

Bars, about twice the worst value measured over every case of this file on an H100 80GB HBM3 (400 W power limit):
- attention, per (utterance, head): max |d| / (|ref| + rms(ref)) over the rows that see a key, and rel-L2 over the valid
  rows.  Budget: fp16 probabilities for P.V, ex2.approx and the fp16 output; RelPos adds (q+u)*scale and (q+v)*scale
  rounded to fp16, which moves every logit.  Rows that see no key are exactly 0.
- depthwise conv: max |d| / (|ref| + rms(ref)).  Budget: the fp16 output (2^-11 relative).
Reruns are bit-identical, and an utterance alone is bit-identical to the same utterance inside a batch."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401
import encoder_kernels_oracle as EK  # noqa: E402

#                 (max |d| / (|ref| + rms), rel-L2)   measured worst
ATT_BARS = {False: (1.5e-3, 5e-4),                  # RoPE / regularMHA: 7.1e-4, 2.4e-4
            True: (1.2e-2, 1.2e-3)}                 # RelPosMHAXL: 6.0e-3 (dh 32, T = 2500), 5.8e-4
DW_BAR = 9e-4                                       # 4.3e-4

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ attention
def _ragged_len(T):
    """a length in [1, T) that is not a multiple of the 64-key block (T for T == 1)"""
    n = max(1, (2 * T) // 3)
    return n - 1 if n % 64 == 0 else n


def _att_inputs(B, T, H, dh, lens, relpos, seed, dev):
    """fp16 qkv [B*T, 3*H*dh] in per-head [q | k | v] blocks (+ RelPos: pos_u, pos_v fp32 [H*dh], P fp16 [T, H*dh]).
    Keys and values of frames >= lens[b] are about +-3e4."""
    g = torch.Generator().manual_seed(seed)
    d = H * dh
    scale = 1.0 / math.sqrt(d)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    if relpos:  # content and position terms each with a std of 3 / sqrt(2): |q + u| ~ 1.12 sq, k and P rows ~ N(0, 1)
        sq = 3.0 / math.sqrt(2) / (1.118 * math.sqrt(dh) * scale)
    else:       # scores = q.k with q pre-scaled: std 3
        sq = 3.0 / math.sqrt(dh)
    q, k, v = sq * r(B, T, H, dh), r(B, T, H, dh), r(B, T, H, dh)
    if lens is not None:
        for b in range(B):
            n = int(lens[b])
            if n < T:
                big = lambda: 3e4 * torch.sign(r(T - n, H, dh)) * (0.5 + 0.5 * torch.rand(T - n, H, dh, generator=g))  # noqa: E731
                k[b, n:], v[b, n:] = big(), big()
    qkv = torch.cat([q, k, v], dim=-1).reshape(B * T, 3 * d).half().to(dev)
    extra = (None, None, None)
    if relpos:
        extra = ((0.5 * sq * r(d)).to(dev), (0.5 * sq * r(d)).to(dev), r(T, d).half().to(dev))
    return qkv, extra, scale


def _att_dev(qkv, B, T, H, dh, lens, relpos, u, w, P, scale, chunk=0, left=-1):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    out = torch.full((B * T, H * dh), float("nan"), dtype=torch.float16, device=qkv.device)
    check(lib().sbk_encoder_attention_test(ptr(qkv), B, T, H, dh, ptr(lens), int(relpos), ptr(u), ptr(w), ptr(P),
                                           ctypes.c_float(scale), chunk, left, ptr(out), stream_ptr(qkv.device)),
          "sbk_encoder_attention_test")
    return out


def _att_ref(qkv, B, T, H, dh, lens, relpos, u, w, P, scale, chunk=0, left=-1):
    q, k, v = qkv.double().view(B, T, H, 3 * dh).split(dh, dim=-1)
    if relpos:
        return EK.attention_ref(q, k, v, lens, P, u, w, scale, chunk, left)
    return EK.attention_ref(q, k, v, lens, chunk=chunk, left_chunks=left)


def _att_check(name, out, ref, lens, relpos, chunk=0, left=-1):
    """asserts the bars over every (utterance, head); returns the [B, T] mask of rows that see a key"""
    B, T, H, dh = ref.shape
    out = out.double().view(B, T, H, dh)
    seen = EK.visible_keys(T, lens, B, chunk, left, ref.device).any(-1)   # [B, T]
    lens_ = torch.full((B,), T) if lens is None else lens.cpu()
    zero_err = float(out[~seen].abs().max()) if (~seen).any() else 0.0
    emax = el2 = 0.0
    for b in range(B):
        rows = seen[b]
        valid = rows & (torch.arange(T, device=ref.device) < int(lens_[b]))
        for h in range(H):
            o, r = out[b, rows, h], ref[b, rows, h]
            if o.numel() == 0:
                continue
            emax = max(emax, float(((o - r).abs() / (r.abs() + r.pow(2).mean().sqrt())).max()))
            ov, rv = out[b, valid, h], ref[b, valid, h]
            el2 = max(el2, float((ov - rv).norm() / rv.norm().clamp_min(1e-30)))
    bmax, bl2 = ATT_BARS[bool(relpos)]
    finite = bool(torch.isfinite(out).all())   # NaN also marks a row the kernel did not write
    msg = (f"{name}: max |d|/(|ref|+rms) {emax:.3e} (bar {bmax}), rel-L2 {el2:.3e} (bar {bl2}), "
           f"max |out| on {int((~seen).sum())} rows without a key {zero_err:.3e} (must be 0), finite {finite}")
    print("MEASURE attention " + msg)
    assert finite and emax <= bmax and el2 <= bl2 and zero_err == 0, msg
    return seen


def _run_att_case(dev, name, B, T, H, dh, relpos, lens, seed, chunk=0, left=-1):
    lens_dev = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    lens_t = None if lens is None else torch.tensor(lens)
    qkv, (u, w, P), scale = _att_inputs(B, T, H, dh, lens_t, relpos, seed, dev)
    out = _att_dev(qkv, B, T, H, dh, lens_dev, relpos, u, w, P, scale, chunk, left)
    ref = _att_ref(qkv, B, T, H, dh, lens_t, relpos, u, w, P, scale, chunk, left)
    seen = _att_check(name, out, ref, lens_t, relpos, chunk, left)
    assert torch.equal(out, _att_dev(qkv, B, T, H, dh, lens_dev, relpos, u, w, P, scale, chunk, left)), f"{name}: rerun differs"
    return qkv, (u, w, P), scale, out, seen


FULL_CASES = [(64, False), (64, True), (36, False), (36, True), (32, False), (32, True), (128, False)]


@pytest.mark.parametrize("T", [1, 17, 63, 64, 65, 251, 1000])
@pytest.mark.parametrize("dh,relpos", FULL_CASES)
def test_attention_full_context(dev, dh, relpos, T):
    """B = 3 with lengths {T, not a multiple of 64, 1}; H = 8 at T = 251.  The middle utterance alone (B = 1) is
    bit-identical to its rows in the batch.  T = 65 and 251 also run without lengths: the zero-filled keys past T in the
    last key block are masked."""
    H = 8 if T == 251 else 2
    lens = [T, _ragged_len(T), 1]
    name = f"dh={dh} {'relpos' if relpos else 'plain'} T={T}"
    qkv, (u, w, P), scale, out, _ = _run_att_case(dev, name, 3, T, H, dh, relpos, lens, T * 131 + dh * 7 + relpos)
    d = H * dh
    alone = _att_dev(qkv[T:2 * T].contiguous(), 1, T, H, dh, torch.tensor(lens[1:2], dtype=torch.int32, device=dev), relpos,
                     u, w, P, scale)
    assert torch.equal(alone, out[T:2 * T]), f"{name}: B = 1 differs from the batch"
    if T in (65, 251):
        _run_att_case(dev, name + " no lens", 2, T, H, dh, relpos, None, T * 17 + dh + relpos)
    assert out.shape == (3 * T, d)


WINDOWS = [(1, 0), (4, -1), (5, 3), (16, 1), (64, 0), (65, 2), (100, -1)]


@pytest.mark.parametrize("T", [251, 300])
@pytest.mark.parametrize("chunk,left", WINDOWS)
@pytest.mark.parametrize("relpos", [False, True])
@pytest.mark.parametrize("dh", [64, 36])
def test_attention_dynamic_chunk(dev, dh, relpos, chunk, left, T):
    """Dynamic Chunk windows (left < 0 = the whole past), B = 3 with lengths {T, not a multiple of 64, 20}: with a finite
    left context, padded query rows of the 20-frame utterance see no valid key and must be exactly 0."""
    lens = [T, _ragged_len(T), 20]
    name = f"dh={dh} {'relpos' if relpos else 'plain'} T={T} chunk={chunk} left={left}"
    _, _, _, _, seen = _run_att_case(dev, name, 3, T, 2, dh, relpos, lens, T * 7 + chunk * 101 + left + dh + relpos,
                                     chunk, left)
    if left >= 0:
        assert not seen[2].all(), "the case should hold rows without a visible key"


@pytest.mark.parametrize("dh,T", [(64, 1036), (64, 1037), (64, 1500), (64, 2500), (36, 1442), (36, 1443), (36, 2500),
                                  (32, 2172), (32, 2173), (32, 2500)])
def test_attention_relpos_long(dev, dh, T):
    """RelPosMHAXL up to max_len = 2500 frames: shared memory does not depend on T (a T-row P table stopped fitting at
    1037 / 1443 / 2173 frames for head widths 64 / 36 / 32)."""
    _run_att_case(dev, f"dh={dh} relpos long T={T}", 2, T, 2, dh, True, [T, _ragged_len(T)], T + dh)


def test_attention_rejects_unbuilt_head_widths(dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    T, H = 16, 2
    qkv = torch.zeros(T, 3 * H * 128, dtype=torch.float16, device=dev)
    out = torch.zeros(T, H * 128, dtype=torch.float16, device=dev)
    uv = torch.zeros(H * 128, device=dev)
    P = torch.zeros(T, H * 128, dtype=torch.float16, device=dev)
    st = stream_ptr(dev)
    call = lambda dh, rp: lib().sbk_encoder_attention_test(ptr(qkv), 1, T, H, dh, None, rp, ptr(uv), ptr(uv), ptr(P),  # noqa: E731
                                                           ctypes.c_float(0.1), 0, -1, ptr(out), st)
    assert call(48, 0) != 0 and call(96, 0) != 0 and call(48, 1) != 0
    assert call(128, 1) != 0      # RelPos is built for head widths up to 64
    assert call(128, 0) == 0 and call(64, 1) == 0


# ------------------------------------------------------------------------------------------------ depthwise conv
def _dw_inputs(B, T, D, K, seed, dev):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    x = r(B, T, D)
    for b, frac in enumerate((1.0, 0.7, 0.4)[:B]):  # ragged batch: the padded frames hold other values (they are inputs)
        n = max(1, int(frac * T))
        x[b, n:] = 0.25 * r(T - n, D) - 0.1
    taps = r(D, 1, K) * (1.4 / K ** 0.5)            # asymmetric: tap k and tap K-1-k differ
    bias = 0.1 * r(D)
    ln_g, ln_b = 1.0 + 0.1 * r(D), 0.05 * r(D)
    return [t.to(dev).contiguous() for t in (x, taps, bias, ln_g, ln_b)]


def _dw_dev(x, taps, bias, ln_g, ln_b, chunk):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    B, T, D = x.shape
    out = torch.full((B, T, D), float("nan"), dtype=torch.float16, device=x.device)
    check(lib().sbk_dwconv_test(ptr(x), B, T, D, taps.shape[-1], ptr(taps), ptr(bias), ptr(ln_g), ptr(ln_b), chunk, ptr(out),
                                stream_ptr(x.device)), "sbk_dwconv_test")
    return out


def _dw_check(name, x, taps, bias, ln_g, ln_b, chunk):
    out = _dw_dev(x, taps, bias, ln_g, ln_b, chunk)
    ref = EK.dwconv_ref(x, taps, bias, ln_g, ln_b, chunk)
    o = out.double()
    err = float(((o - ref).abs() / (ref.abs() + ref.pow(2).mean().sqrt())).max())
    msg = f"{name}: max |d|/(|ref|+rms) {err:.3e} (bar {DW_BAR})"
    print("MEASURE dwconv " + msg)
    assert torch.isfinite(o).all() and err <= DW_BAR, msg
    assert torch.equal(out, _dw_dev(x, taps, bias, ln_g, ln_b, chunk)), f"{name}: rerun differs"


@pytest.mark.parametrize("T", [1, 15, 16, 17, 251, 3000])
@pytest.mark.parametrize("K", [31, 15, 3])
@pytest.mark.parametrize("D", [144, 256, 512, 1024])
def test_dwconv_kernel(dev, D, K, T):
    """K = 31: taps in registers, 1 / 1 / 2 / 4 channels per thread for D = 144 / 256 / 512 / 1024; K = 15, 3: runtime K.
    chunk 0 (full context) and Dynamic Chunk Convolution chunks {1, 4, 5, 16, 64}; ragged B = 3.  At T = 16 and 251 also
    conv outputs with row means of about 50 and a spread of about 1 (LayerNorm cancellation)."""
    x, taps, bias, ln_g, ln_b = _dw_inputs(3, T, D, K, D * 7 + K * 1009 + T, dev)
    for chunk in (0, 1, 4, 5, 16, 64):
        _dw_check(f"D={D} K={K} T={T} chunk={chunk}", x, taps, bias, ln_g, ln_b, chunk)
    if T in (16, 251):
        for chunk in (0, 5):
            _dw_check(f"D={D} K={K} T={T} chunk={chunk} mean 50", x, taps, bias + 50.0, ln_g, ln_b, chunk)


def test_dwconv_rejects_bad_shapes(dev):
    """even K, D % 4 != 0, D > 1024, and a K whose input slab does not fit shared memory at D = 1024 (the largest K that
    fits, 35, runs and matches)."""
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    st = stream_ptr(dev)
    T = 20

    def call(D, K):
        x = torch.zeros(T, D, device=dev)
        taps = torch.zeros(D, 1, K, device=dev)
        v = torch.ones(D, device=dev)
        out = torch.zeros(T, D, dtype=torch.float16, device=dev)
        return lib().sbk_dwconv_test(ptr(x), 1, T, D, K, ptr(taps), ptr(v), ptr(v), ptr(v), 0, ptr(out), st)

    assert call(256, 30) != 0 and call(146, 31) != 0 and call(1028, 31) != 0 and call(1024, 37) != 0
    x, taps, bias, ln_g, ln_b = _dw_inputs(2, T, 1024, 35, 35, dev)
    _dw_check("D=1024 K=35 T=20", x, taps, bias, ln_g, ln_b, 0)
