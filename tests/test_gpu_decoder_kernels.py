"""-m gpu parity tests of the decode-step kernels alone, against the float64 references of decoder_kernels_oracle.py (pinned
to the CPU oracle by test_decoder_kernels_oracle.py):

- the step projections through sbk_step_proj_test on both back ends: weight streaming (skinny_gemm_kernel: UNR 4 / 8,
  NT 1 / 2, the LayerNorm-fused variants at K = 256 / 512 / 768 / 1024) and wgmma (gemm_f16_small), every epilogue
  (fp16, fp16 GELU, fp16 ReLU, fp32, residual, QKV -> cache), row counts around the 32-row and 64-row tiles, N tails
  of the 8- and 16-column tiles, K tails past the last full UNR chunk;
- the decode attention through sbk_dec_attention_test: dec_attention_kernel<64 / 128> and dec_attention_generic_kernel
  (head widths 36 and 32), self-attention over the KV cache with and without a beam lineage table and the
  TransformerLM's pad-token mask, cross-attention over up to 2500 frames (2560 for the generic kernel) in the head-major
  and the row-major K/V layouts;
- an utterance with no encoder frame through the greedy search and the teacher-forced decoder.

The inputs are built to expose a subtly wrong kernel: LayerNorm inputs whose row means are about 300x their spread (a
one-pass fp32 variance fails); one fp16 case past 65504 (saturating stores); output columns past N, rows past the row
count and cache positions other than the step hold sentinels that must survive; attention logits with a standard
deviation of about 3; keys and values that must not be seen (masked frames, pad tokens, cache positions past the step) at
about +-3e4, so that one leaked key dominates its row; lineage tables that never point a row at itself, with the other
parity's table filled with a different valid one.

Bars, about twice the worst value measured over every case of this file on an H100 80GB HBM3 (700 W power limit), as
max |d| / (|ref| + rms(ref)) and rel-L2 over the case's outputs:
- fp16 outputs of fp16 operands: the fp16 store (2^-11 relative);
- fp32 and residual outputs: fp32 accumulation only;
- LayerNorm-fused or LayerNorm-fed projections: the LayerNorm output is rounded to fp16 before the GEMM;
- attention: ex2.approx, fp32 accumulation and the fp16 output.
Reruns are bit-identical, a row (or an utterance) computed alone is bit-identical to the same row inside a batch, and the
two projection back ends agree within the bars."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401
import decoder_kernels_oracle as DK  # noqa: E402

#                (max |d| / (|ref| + rms), rel-L2)   measured worst
PROJ_BARS = {"f16": (1e-3, 5e-4),    # 4.1e-4, 2.3e-4; back ends apart 7.3e-4 (one fp16 ulp, at most 2^-10, sets the bar)
             "f32": (2e-5, 6e-6),    # 9.9e-6 (K = 3072), 2.6e-6; back ends apart 9.5e-6
             "ln": (2.8e-3, 7e-4)}   # 1.4e-3, 3.2e-4; back ends apart 7.7e-4
ATT_BAR = (8e-4, 5e-4)               # 3.6e-4, 2.4e-4

pytestmark = pytest.mark.gpu
SENT = -777.0   # sentinel of output entries a call must not write (exact in fp16)
BIG = 3e4       # keys / values that must not be seen


def _vp(t, off=0):
    """address of element `off` of a contiguous tensor"""
    assert t.is_contiguous()
    return ctypes.c_void_p(t.data_ptr() + off * t.element_size())


def _metrics(out, ref):
    o, r = out.double(), ref.double()
    rms = r.pow(2).mean().sqrt()
    emax = float(((o - r).abs() / (r.abs() + rms)).max())
    el2 = float((o - r).norm() / r.norm().clamp_min(1e-30))
    return emax, el2


def _bits(t):
    """bit pattern (NaN-safe equality)"""
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _big(g, *shape):
    return BIG * torch.sign(torch.randn(*shape, generator=g)) * (0.5 + 0.5 * torch.rand(*shape, generator=g))


# ------------------------------------------------------------------------------------------------ projections
EPI = {name: i for i, name in enumerate(DK.EPILOGUES)}
ROWS = [1, 31, 32, 33, 63, 64, 100, 320, 512]
DIMS = [144, 256, 512, 768, 1024]
S_MAX = 7
# (N, K, epilogue, LayerNorm-fed variants)
PROJ_CASES = (
    [(d, d, e, (False, True)) for d in DIMS for e in ("f16", "f32", "resid")]      # out_proj, cross query, the head at d
    + [(3 * d, d, "qkv_cache", (False, True)) for d in DIMS]                       # self-attention in_proj -> caches
    + [(1000, 512, e, (False, True)) for e in ("f16_gelu", "f16_relu", "f32")]    # NT = 1 (N < 1024)
    + [(5000, 512, "f32", (False, True)),                                          # NT = 2, 8-column tail: the vocabulary
       (2048, 512, "f16_gelu", (False, True)), (2048, 512, "f16_relu", (False, True)),   # ffn1
       (512, 2048, "resid", (False,)), (512, 3072, "resid", (False,)),             # UNR = 8: ffn2
       (512, 1040, "resid", (False,)), (1024, 1040, "f16", (False,)),              # UNR = 8 with K tails
       (512, 1536, "resid", (False,)), (1024, 1536, "f16", (False,))])


def _proj_inputs(rows, N, K, ln, seed, dev):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    inp = {"W": (r(N, K) / math.sqrt(K)).half().to(dev), "bias": (0.1 * r(N)).to(dev), "x0": r(rows, N).to(dev),
           "A": None, "X": None, "ln": None}
    if ln:   # row means about 300x the spread: a one-pass fp32 variance cancels catastrophically
        spread = 0.5 + torch.rand(rows, 1, generator=g)
        mean = 300.0 * spread * torch.sign(r(rows, 1))
        inp["X"] = (mean + spread * r(rows, K)).to(dev)
        inp["ln"] = ((1.0 + 0.1 * r(K)).to(dev), (0.1 * r(K)).to(dev))
    else:
        inp["A"] = r(rows, K).half().to(dev)
    return inp


def _proj_dev(backend, epi, inp, rows, step, dev):
    """-> (rc, out [rows + 2, ldo] with sentinels, kcache, vcache [rows + 1, S_MAX, N / 3] prefilled with NaN)"""
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    W = inp["W"]
    N, K = W.shape
    qkv = epi == "qkv_cache"
    w = N // 3 if qkv else N
    ldo = w + 8
    f32 = epi in ("f32", "resid")
    out = torch.full((rows + 2, ldo), SENT, dtype=torch.float32 if f32 else torch.float16, device=dev)
    if epi == "resid":
        out[:rows, :N] = inp["x0"][:rows]
    kc = vc = None
    if qkv:
        kc = torch.full((rows + 1, S_MAX, w), float("nan"), dtype=torch.float16, device=dev)
        vc = kc.clone()
    A, X = inp["A"], inp["X"]
    g, b = inp["ln"] if inp["ln"] is not None else (None, None)
    rc = lib().sbk_step_proj_test(backend, EPI[epi], ptr(A), K if A is not None else 0, ptr(X), ptr(g), ptr(b), ptr(W),
                                  ptr(inp["bias"]), rows, N, K, ptr(out), ldo, ptr(kc), ptr(vc), S_MAX, step, stream_ptr(dev))
    return rc, out, kc, vc


def _row(inp, i):
    """the inputs of row i alone"""
    one = dict(inp)
    one["x0"] = inp["x0"][i:i + 1]
    one["A"] = None if inp["A"] is None else inp["A"][i:i + 1].contiguous()
    one["X"] = None if inp["X"] is None else inp["X"][i:i + 1].contiguous()
    return one


def _proj_check(name, epi, ln, inp, rows, step, out, kc, vc):
    """asserts the bars and the sentinels; returns the case's valid outputs (for the back-end comparison)"""
    W = inp["W"]
    N = W.shape[0]
    w = N // 3 if epi == "qkv_cache" else N
    lnp = inp["ln"] if ln else (None, None)
    if epi == "qkv_cache":
        q, kr, vr = DK.proj_ref(inp["A"], W, inp["bias"], epi, X=inp["X"], ln_g=lnp[0], ln_b=lnp[1], kcache=kc[:rows],
                                vcache=vc[:rows], step=step)
        got = torch.cat([out[:rows, :w], kc[:rows, step], vc[:rows, step]], dim=1)
        ref = torch.cat([q, kr[:, step], vr[:, step]], dim=1)
        others = [p for p in range(S_MAX) if p != step]
        untouched = bool(torch.isnan(kc[:, others]).all() and torch.isnan(vc[:, others]).all()
                         and torch.isnan(kc[rows]).all() and torch.isnan(vc[rows]).all())
    else:
        ref = DK.proj_ref(inp["A"], W, inp["bias"], epi, out=inp["x0"], X=inp["X"], ln_g=lnp[0], ln_b=lnp[1])
        got = out[:rows, :w]
        untouched = True
    sent = bool((out[:rows, w:] == SENT).all() and (out[rows:] == SENT).all())
    emax, el2 = _metrics(got, ref)
    kind = "ln" if ln else ("f32" if epi in ("f32", "resid") else "f16")
    bmax, bl2 = PROJ_BARS[kind]
    finite = bool(torch.isfinite(got).all())
    msg = (f"{name}: max |d|/(|ref|+rms) {emax:.3e} (bar {bmax}), rel-L2 {el2:.3e} (bar {bl2}), finite {finite}, "
           f"sentinels kept {sent and untouched}")
    print(f"MEASURE proj-{kind} " + msg)
    assert finite and sent and untouched and emax <= bmax and el2 <= bl2, msg
    return got, ref, kind


@pytest.mark.parametrize("N,K,epi,lns", PROJ_CASES, ids=[f"N{c[0]}-K{c[1]}-{c[2]}" for c in PROJ_CASES])
def test_step_projection(dev, N, K, epi, lns):
    """every row count of ROWS on both back ends (wgmma where the QKV width is a multiple of 32), with fp16 A and, where
    listed, A = LayerNorm(X) (fused into the weight-streaming kernel at K = 256 / 512 / 768 / 1024).  Reruns are
    bit-identical; the last row alone equals its row in the batch; the back ends agree within the bars."""
    backends = (0, 1) if not (epi == "qkv_cache" and (N // 3) % 32) else (0,)
    for ln in lns:
        for rows in ROWS:
            inp = _proj_inputs(rows, N, K, ln, N * 7 + K * 13 + rows * 31 + ln + len(epi), dev)
            step = rows % S_MAX
            got = {}
            for be in backends:
                name = f"N={N} K={K} {epi}{' ln' if ln else ''} rows={rows} {('stream', 'wgmma')[be]}"
                rc, out, kc, vc = _proj_dev(be, epi, inp, rows, step, dev)
                assert rc == 0, name
                got[be], ref, kind = _proj_check(name, epi, ln, inp, rows, step, out, kc, vc)
                rc, out2, kc2, vc2 = _proj_dev(be, epi, inp, rows, step, dev)
                assert rc == 0 and torch.equal(_bits(out), _bits(out2)), f"{name}: rerun differs"
                if kc is not None:
                    assert torch.equal(_bits(kc), _bits(kc2)) and torch.equal(_bits(vc), _bits(vc2)), f"{name}: rerun differs"
                if rows > 32:
                    i = rows - 1
                    rc, one, kc1, vc1 = _proj_dev(be, epi, _row(inp, i), 1, step, dev)
                    assert rc == 0 and torch.equal(_bits(one[0]), _bits(out[i])), f"{name}: row {i} alone differs"
                    if kc is not None:
                        assert torch.equal(_bits(kc1[0]), _bits(kc[i])) and torch.equal(_bits(vc1[0]), _bits(vc[i]))
            if len(got) == 2:
                r = ref.double()
                emax = float(((got[0].double() - got[1].double()).abs() / (r.abs() + r.pow(2).mean().sqrt())).max())
                print(f"MEASURE proj-backends N={N} K={K} {epi}{' ln' if ln else ''} rows={rows}: stream vs wgmma {emax:.3e}")
                assert emax <= PROJ_BARS[kind][0], f"back ends differ: {emax:.3e}"


def test_step_projection_saturates(dev):
    """fp16 outputs past +-65504 are stored as +-65504 (satfinite), never inf, on both back ends"""
    rows, N, K = 40, 256, 256
    inp = _proj_inputs(rows, N, K, False, 5, dev)
    inp["bias"][::3] = 7e4
    inp["bias"][1::3] = -7e4
    for be in (0, 1):
        rc, out, _, _ = _proj_dev(be, "f16", inp, rows, 0, dev)
        assert rc == 0
        _proj_check(f"saturation {('stream', 'wgmma')[be]}", "f16", False, inp, rows, 0, out, None, None)
        assert (out[:rows, 0:N:3] == 65504).all() and (out[:rows, 1:N:3] == -65504).all()


def test_step_projection_rejects_bad_arguments(dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    rows, N, K = 4, 96, 64
    W = torch.zeros(N, K, dtype=torch.float16, device=dev)
    A = torch.zeros(rows, K, dtype=torch.float16, device=dev)
    X = torch.zeros(rows, K, device=dev)
    v = torch.ones(K, device=dev)
    out = torch.zeros(rows, N + 8, dtype=torch.float16, device=dev)
    kc = torch.zeros(rows, S_MAX, N // 3, dtype=torch.float16, device=dev)
    st = stream_ptr(dev)

    def call(be=0, epi=0, a=A, x=None, n=N, k=K, ldo=N, step=0, cache=None):
        return lib().sbk_step_proj_test(be, epi, ptr(a), K, ptr(x), ptr(v), ptr(v), ptr(W), None, rows, n, k, ptr(out), ldo,
                                        ptr(cache), ptr(cache), S_MAX, step, st)

    assert call() == 0 and call(be=1) == 0 and call(a=None, x=X) == 0 and call(ldo=N + 4) == 0
    assert call(be=2) != 0 and call(epi=6) != 0 and call(a=None) != 0 and call(x=X) != 0
    assert call(k=40) != 0 and call(ldo=N - 1) != 0 and call(be=1, ldo=N + 4) != 0   # wgmma: 16-byte row stores
    assert call(epi=5, ldo=N // 3) != 0                          # QKV without caches
    assert call(epi=5, ldo=N // 3, cache=kc, step=S_MAX) != 0 and call(epi=5, ldo=N // 3, cache=kc, step=-1) != 0
    assert call(epi=5, ldo=N // 3, cache=kc, step=S_MAX - 1) == 0


# ------------------------------------------------------------------------------------------------ attention
def _att_dev(q, k, v, row_stride, key_stride, head_stride, rpb, H, dh, max_keys, step, enc_len=None, lin=None, tok=None,
             lin_stride=0):
    """k, v = (buffer, element offset); -> (rc, out [rows, H * dh] fp16)"""
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    rows = q.shape[0]
    out = torch.full((rows, H * dh), float("nan"), dtype=torch.float16, device=q.device)
    rc = lib().sbk_dec_attention_test(ptr(q), H * dh, _vp(*k), _vp(*v), ctypes.c_longlong(row_stride), key_stride,
                                      head_stride, rpb, rows, H, dh, max_keys, step, ptr(enc_len), ptr(lin), ptr(tok),
                                      lin_stride, 0, ptr(out), H * dh, stream_ptr(q.device))
    return rc, out


def _att_check(name, out, ref):
    rows, H, dh = ref.shape
    o = out.double().view(rows, H, dh)
    nan_ref = torch.isnan(ref)
    same_nan = bool(torch.equal(torch.isnan(o), nan_ref))
    ok = ~nan_ref.view(rows, -1).any(-1)
    emax, el2 = _metrics(o[ok], ref[ok]) if ok.any() else (0.0, 0.0)
    finite = bool(torch.isfinite(o[ok]).all())
    bmax, bl2 = ATT_BAR
    msg = (f"{name}: max |d|/(|ref|+rms) {emax:.3e} (bar {bmax}), rel-L2 {el2:.3e} (bar {bl2}), finite {finite}, "
           f"NaN rows as the reference {same_nan} ({int((~ok).sum())})")
    print("MEASURE attention " + msg)
    assert finite and same_nan and emax <= bmax and el2 <= bl2, msg


SELF_STEPS = [0, 1, 30, 31, 32, 127, 128, 129, 499]
SELF_MODES = ["plain", "lineage", "tokens", "lineage+tokens"]
HEAD_DIMS = [64, 128, 36, 32]


def _self_inputs(R, H, dh, S, step, mode, seed, dev):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    q = (3.0 / math.sqrt(dh)) * r(R, H, dh)
    kc, vc = r(R, S, H, dh), r(R, S, H, dh)
    kc[:, step + 1:], vc[:, step + 1:] = _big(g, R, S - step - 1, H, dh), _big(g, R, S - step - 1, H, dh)
    lin = tok = None
    if "lineage" in mode:   # ancestors never the row itself; the other parity's table differs from it everywhere
        rr = torch.arange(R).view(R, 1)
        cur = (rr + 1 + torch.randint(0, R - 1, (R, S), generator=g)) % R
        other = (cur + 1 + torch.randint(0, R - 1, (R, S), generator=g)) % R
        lin = torch.empty(2, R, S, dtype=torch.int32)
        lin[step & 1], lin[(step + 1) & 1] = cur, other
    if "tokens" in mode:    # pad id 0 at the start (row 0), inside (row 1), at the end (row 2), start and end (row 3)
        tok = torch.randint(1, 50, (R, S), generator=g, dtype=torch.int32)
        tok[0, 0] = 0
        tok[1, step // 3] = tok[1, (2 * step) // 3] = 0
        tok[2, step] = 0
        tok[3, 0] = tok[3, step] = 0
        pad = tok == 0
        kc[pad], vc[pad] = _big(g, int(pad.sum()), H, dh), _big(g, int(pad.sum()), H, dh)
    t = lambda x: None if x is None else x.contiguous().to(dev)  # noqa: E731
    return q.half().to(dev), kc.half().to(dev), vc.half().to(dev), t(lin), t(tok)


def _self_run(q, kc, vc, H, dh, step, lin, tok):
    R, S = kc.shape[:2]
    d = H * dh
    return _att_dev(q.view(R, d), (kc, 0), (vc, 0), S * d, d, 0, 1, H, dh, S, step, lin=lin, tok=tok,
                    lin_stride=S if (lin is not None or tok is not None) else 0)


@pytest.mark.parametrize("mode", SELF_MODES)
@pytest.mark.parametrize("dh", HEAD_DIMS)
def test_self_attention(dev, dh, mode):
    """R = 5 rows, 2 heads, a 512-position cache, step in SELF_STEPS (both lineage parities); without a lineage a row
    alone is bit-identical to its row in the batch."""
    R, H, S = 5, 2, 512
    for step in SELF_STEPS:
        name = f"self dh={dh} {mode} step={step}"
        q, kc, vc, lin, tok = _self_inputs(R, H, dh, S, step, mode, step * 97 + dh * 5 + len(mode), dev)
        rc, out = _self_run(q, kc, vc, H, dh, step, lin, tok)
        assert rc == 0, name
        ref = DK.dec_attention_ref(q, kc, vc, step + 1, lineage=None if lin is None else lin[step & 1], tok=tok)
        _att_check(name, out, ref)
        assert torch.equal(_bits(out), _bits(_self_run(q, kc, vc, H, dh, step, lin, tok)[1])), f"{name}: rerun differs"
        if lin is None:
            i = 2
            rc, one = _self_run(q[i:i + 1].contiguous(), kc[i:i + 1].contiguous(), vc[i:i + 1].contiguous(), H, dh, step, None,
                                None if tok is None else tok[i:i + 1].contiguous())
            assert rc == 0 and torch.equal(_bits(one[0]), _bits(out[i])), f"{name}: row {i} alone differs"


def _cross_buffers(K, V, layout):
    """K, V [U, T, H, dh] fp16 -> (buffer, k offset, v offset, row_stride, key_stride, head_stride) in the engine's layouts:
    head-major [K | V][utt][head][T][dh], or row-major [utt][T][K (H * dh) | V (H * dh)]"""
    U, T, H, dh = K.shape
    d = H * dh
    if layout == "head":
        buf = torch.stack([K.permute(0, 2, 1, 3), V.permute(0, 2, 1, 3)]).contiguous()
        return buf, 0, U * T * d, T * d, dh, T * dh
    buf = torch.cat([K.reshape(U, T, d), V.reshape(U, T, d)], dim=-1).contiguous()
    return buf, 0, d, T * 2 * d, 2 * d, 0


def _cross_run(q, K, V, layout, rpu, enc_len, max_keys):
    U, T, H, dh = K.shape
    buf, ko, vo, rs, ks, hs = _cross_buffers(K, V, layout)
    return _att_dev(q.view(q.shape[0], H * dh), (buf, ko), (buf, vo), rs, ks, hs, rpu, H, dh, max_keys, -1, enc_len=enc_len)


def _ragged(T):
    n = max(1, (2 * T) // 3)
    return n - 1 if n % 32 == 0 and n > 1 else n


CROSS_T = [1, 3, 127, 128, 129, 251, 1001, 2500]


@pytest.mark.parametrize("dh,layout", [(64, "head"), (64, "row"), (128, "row"), (36, "row"), (32, "row")])
def test_cross_attention(dev, dh, layout):
    """3 utterances with enc_len {T, ragged, 1}, rows_per_utt in {1, 4, 10}, T in CROSS_T (and 2560, the generic
    kernel's limit, at head widths 36 / 32); frames past enc_len at +-3e4.  Without lengths every frame is a key.  The
    middle utterance alone is bit-identical to its rows in the batch."""
    U, H = 3, 2
    Ts = CROSS_T + ([2560] if dh not in (64, 128) else [])
    for T in Ts:
        for rpu in (1, 4, 10):
            name = f"cross dh={dh} {layout} T={T} rows_per_utt={rpu}"
            g = torch.Generator().manual_seed(T * 11 + rpu * 3 + dh)
            r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
            lens = torch.tensor([T, _ragged(T), 1], dtype=torch.int32)
            K, V = r(U, T, H, dh), r(U, T, H, dh)
            for b in range(U):
                n = int(lens[b])
                if n < T:
                    K[b, n:], V[b, n:] = _big(g, T - n, H, dh), _big(g, T - n, H, dh)
            q = ((3.0 / math.sqrt(dh)) * r(U * rpu, H, dh)).half().to(dev)
            K, V, lens_d = K.half().to(dev), V.half().to(dev), lens.to(dev)
            rc, out = _cross_run(q, K, V, layout, rpu, lens_d, T)
            assert rc == 0, name
            _att_check(name, out, DK.dec_attention_ref(q, K, V, lens, rows_per_block=rpu))
            assert torch.equal(_bits(out), _bits(_cross_run(q, K, V, layout, rpu, lens_d, T)[1])), f"{name}: rerun differs"
            rc, one = _cross_run(q[rpu:2 * rpu].contiguous(), K[1:2].contiguous(), V[1:2].contiguous(), layout, rpu,
                                 lens_d[1:2].contiguous(), T)
            assert rc == 0 and torch.equal(_bits(one), _bits(out[rpu:2 * rpu])), f"{name}: utterance 1 alone differs"
            if rpu == 4 and T in (3, 129):
                Kf, Vf = r(U, T, H, dh).half().to(dev), r(U, T, H, dh).half().to(dev)
                rc, out = _cross_run(q, Kf, Vf, layout, rpu, None, T)
                assert rc == 0
                _att_check(name + " no lengths", out, DK.dec_attention_ref(q, Kf, Vf, T, rows_per_block=rpu))


def test_attention_rejects_bad_arguments(dev):
    """2561 keys at a generic head width, lineage entries outside [0, rows), enc_len outside [0, max_keys], step past the
    table or the cache, a lineage on cross-attention: errors, nothing launched"""
    R, H, S = 5, 2, 16
    q, kc, vc, lin, tok = _self_inputs(R, H, 36, S, 5, "lineage+tokens", 1, dev)
    assert _self_run(q, kc, vc, H, 36, 5, lin, tok)[0] == 0
    bad = lin.clone()
    bad[1, 2, 3] = R
    assert _self_run(q, kc, vc, H, 36, 5, bad, tok)[0] != 0
    bad[1, 2, 3] = -1
    assert _self_run(q, kc, vc, H, 36, 5, bad, tok)[0] != 0
    assert _self_run(q, kc, vc, H, 36, S, None, None)[0] != 0          # step + 1 keys > the cache
    d = H * 36
    assert _att_dev(q.view(R, d), (kc, 0), (vc, 0), S * d, d, 0, 1, H, 36, S, -1, lin=lin, lin_stride=S)[0] != 0
    T = 2561
    K = torch.zeros(1, T, H, 36, dtype=torch.float16, device=dev)
    q1 = torch.zeros(1, H, 36, dtype=torch.float16, device=dev)
    assert _cross_run(q1, K, K, "row", 1, None, T)[0] != 0
    assert _cross_run(q1, K[:, :2560].contiguous(), K[:, :2560].contiguous(), "row", 1, None, 2560)[0] == 0
    K = torch.zeros(1, 8, H, 64, dtype=torch.float16, device=dev)
    q1 = torch.zeros(1, H, 64, dtype=torch.float16, device=dev)
    assert _cross_run(q1, K, K, "head", 1, torch.tensor([9], dtype=torch.int32, device=dev), 8)[0] != 0
    assert _cross_run(q1, K, K, "head", 1, torch.tensor([-1], dtype=torch.int32, device=dev), 8)[0] != 0
    assert _cross_run(q1, K, K, "head", 1, torch.tensor([8], dtype=torch.int32, device=dev), 8)[0] == 0


# ------------------------------------------------------------------------------------------------ zero-length utterance
@pytest.fixture(scope="module")
def small_asr(dev):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    cfg = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=2)
    sd = seeded_asr_state(cfg, 0)
    return cfg, sd, AsrEngine(cfg, sd, device=dev)


def test_greedy_zero_length_utterance(dev, small_asr):
    """wav_lens [1.0, 0.0, 0.6]: the middle utterance has no encoder frame.  Its logits are NaN; like the reference (torch's
    arg-max of a NaN row is its first index) it emits token 0 at every step with NaN scores, and the other utterances are
    bit-identical to a run without it."""
    from oracle import asr_oracle as O
    cfg, sd, eng = small_asr
    T, steps = 40, 8
    g = torch.Generator().manual_seed(6)
    enc = torch.randn(3, T, cfg["d_model"], generator=g)
    wl = torch.tensor([1.0, 0.0, 0.6])
    pred, score, _, done = eng.greedy_from_enc(enc.to(dev), wl.to(dev), steps, 1, 2)
    torch.cuda.synchronize()
    assert done == steps and (pred[1] == 0).all() and torch.isnan(score[1]).all(), (pred[1].tolist(), score[1].tolist())
    pred2, score2, _, _ = eng.greedy_from_enc(enc[[0, 2]].contiguous().to(dev), wl[[0, 2]].to(dev), steps, 1, 2)
    assert torch.equal(pred[[0, 2]], pred2) and torch.equal(score[[0, 2]], score2)
    with torch.no_grad():
        hyps, _, oscores, _ = O.greedy_search(enc, wl, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], 1, 2, 0.0,
                                              (steps + 0.5) / T, "Transformer.")
    assert hyps[1] == pred[1].tolist() and torch.isnan(oscores[1, 0]).all()


def test_teacher_forced_zero_length_utterance(dev, small_asr):
    """enc_len {T, 0, 25}: NaN decoder outputs exactly where the reference has them (every position of the middle
    utterance), finite elsewhere."""
    from oracle import asr_oracle as O
    cfg, sd, eng = small_asr
    T, S = 40, 5
    g = torch.Generator().manual_seed(7)
    enc = torch.randn(3, T, cfg["d_model"], generator=g)
    tgt = torch.randint(3, cfg["vocab"], (3, S), generator=g)
    tgt[:, 0] = 1
    enc_len = torch.tensor([T, 0, 25])
    out = eng.decode_teacher_forced(tgt.to(dev), enc.to(dev), enc_len.to(dev)).cpu()
    with torch.no_grad():
        ref, _ = O.decode(tgt, enc, enc_len, sd, cfg, "Transformer.")
    assert torch.equal(torch.isnan(out), torch.isnan(ref)) and torch.isnan(ref[1]).all()
    assert torch.isfinite(out[[0, 2]]).all()
    rel = float((out[[0, 2]] - ref[[0, 2]]).norm() / ref[[0, 2]].norm())
    assert rel < 1e-2, rel
