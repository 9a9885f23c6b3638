"""-m gpu tests of the folded cross-attention (csrc/decoder.cu dec_xatt_fold_kernel, csrc/engine.cu xatt_fold), which greedy
and teacher-forced decoding select on the wgmma step back end once n_utt T >= 11 (H - 1) d: each layer attends over the fp16
encoder states with W_k folded into the query projection and W_v into the output projection.

- The layer's cross-attention block alone through sbk_xatt_fold_test (folded query projection, kernel, folded output
  projection added to the residual) against the UNFOLDED float64 reference of decoder_kernels_oracle.py: q = W_q h + b_q,
  K = W_k e + b_k, V = W_v e + b_v, dec_attention_ref, out_proj.  Frame counts around the kernel's 32-frame blocks up to
  2500, full, ragged and empty (NaN) utterances, 64 / 224 / 257 rows, d_model 512 with 8 heads and 256 with 4, attention
  logits with a standard deviation of about 3 and a case scaled x9 (the folded queries W_k^T q stay in fp16 range).
  Masked frames hold +-3e4, output columns past d a sentinel.  Bars: max |d| / (|ref| + rms(ref)) <= 1e-3 and rel-L2 <=
  5e-4 on the layer output, or 1.25 x what the unfolded path (the step's K / V GEMMs, dec_attention_kernel, out_proj on
  the same inputs) reaches against the same reference where that is more.  From fp16 h and fp32 weights the unfolded path
  itself measures 1.0e-3 - 1.6e-3 rel-L2 (4.8e-3 at x9) on an H100 80GB HBM3 (700 W power limit): it rounds q, K, V and
  the attention output to fp16.  The fold measured 6.5e-4 - 1.0e-3 (2.9e-3 at x9), a max error within 1.15 x the unfolded
  path's.  Reruns are bit-identical, an utterance alone is bit-identical to the same utterance in a batch.
- The bench shape end to end: the 10 s goldens' 4 utterances repeated to 224 rows, one group call of 7 batches of 32
  (greedy tokens against the reference with the margin rule), teacher-forced decoding on 224 rows (which must take the
  fold: its GEMMs are the folded step's, with no cross-attention K/V GEMM), and a zero-length utterance among 224."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import case_wav, check_greedy, dev, rel  # noqa: E402,F401
import decoder_kernels_oracle as DK  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BAR = (1e-3, 5e-4)   # max |d| / (|ref| + rms), rel-L2
SENT = -777.0
BIG = 3e4
PAD = 8              # sentinel columns past d


def _metrics(out, ref):
    o, r = out.double(), ref.double()
    rms = r.pow(2).mean().sqrt()
    return float(((o - r).abs() / (r.abs() + rms)).max()), float((o - r).norm() / r.norm().clamp_min(1e-30))


def _layer(d, H, logit_scale, seed):
    """a cross-attention layer's fp32 weights with attention logits of std ~ 3 * logit_scale for unit-variance inputs"""
    g = torch.Generator().manual_seed(seed)
    s = (3.0 * logit_scale) ** 0.5
    wq = torch.randn(d, d, generator=g) * (s * (d // H) ** 0.5 / d ** 0.5)   # q . k / sqrt(dh) ~ 3 * logit_scale
    wk = torch.randn(d, d, generator=g) * (s / d ** 0.5)
    wv = torch.randn(d, d, generator=g) / d ** 0.5
    w = torch.cat([wq, wk, wv]).contiguous()
    b = (0.1 * torch.randn(3 * d, generator=g)).contiguous()
    wo = (torch.randn(d, d, generator=g) / d ** 0.5).contiguous()
    bo = (0.1 * torch.randn(d, generator=g)).contiguous()
    return w, b, wo, bo


def _inputs(rows, T, d, seed, dev):
    g = torch.Generator().manual_seed(seed)
    h = torch.randn(rows, d, generator=g).half()
    e = torch.randn(rows, T, d, generator=g)
    lens = torch.randint(1, T + 1, (rows,), generator=g, dtype=torch.int32)
    lens[0] = T
    lens[min(1, rows - 1)] = 0 if rows > 1 else T
    for r in range(rows):  # frames past enc_len must not be seen
        e[r, lens[r]:] = BIG * torch.sign(torch.randn(T - int(lens[r]), d, generator=g))
    x = torch.full((rows, d + PAD), SENT)
    x[:, :d] = torch.randn(rows, d, generator=g)
    return h.to(dev), e.half().to(dev), lens.to(dev), x.to(dev)


def _bits(t):
    """the bit pattern of a float32 tensor: NaN rows compare equal to themselves"""
    return t.contiguous().view(torch.int32)


def _run(h, e, lens, x, layer, H):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    w, b, wo, bo = layer
    rows, T, d = e.shape
    out = x.clone()
    check(lib().sbk_xatt_fold_test(ptr(h), ptr(w), ptr(b), ptr(wo), ptr(bo), ptr(e), ptr(lens), rows, T, H, d, ptr(out),
                                   d + PAD, stream_ptr(h.device)), "sbk_xatt_fold_test")
    return out


def _ref(h, e, lens, x, layer, H):
    w, b, wo, bo = (t.to(h.device) for t in layer)
    rows, T, d = e.shape
    dh = d // H
    wq, bq = DK.fold_query_scale(w, b, d, dh)
    q = DK.proj_ref(h, wq[:d], bq[:d], "f16").view(rows, H, dh)
    ed = e.double()
    k = (ed @ w[d:2 * d].double().T + b[d:2 * d].double()).view(rows, T, H, dh)
    v = (ed @ w[2 * d:].double().T + b[2 * d:].double()).view(rows, T, H, dh)
    att = DK.dec_attention_ref(q, k, v, lens.long())
    return DK.proj_ref(att.reshape(rows, d), wo, bo, "resid", out=x[:, :d])


CASES = [(1, 257), (31, 64), (32, 224), (33, 257), (251, 224), (1001, 64), (2500, 64)]


@pytest.mark.parametrize("d,H", [(512, 8), (256, 4)])
@pytest.mark.parametrize("T,rows", CASES)
def test_folded_cross_attention(dev, T, rows, d, H):
    _check_case(dev, T, rows, d, H, 1.0, seed=T * 1000 + rows + d)


def test_folded_cross_attention_scaled_logits(dev):
    """attention logits x9: the folded queries W_k^T q grow with them and are stored in fp16"""
    _check_case(dev, 251, 224, 512, 8, 9.0, seed=99)


def _unfolded(h, e, lens, x, layer, H):
    """the same layer through the path the fold replaces: wgmma query projection, K / V GEMMs into fp16, dec_attention_kernel
    over row-major K / V, wgmma out_proj + residual"""
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    w, b, wo, bo = (t.to(h.device) for t in layer)
    rows, T, d = e.shape
    wq, bq = DK.fold_query_scale(w, b, d, d // H)
    st = stream_ptr(h.device)
    q = torch.empty(rows, d, dtype=torch.half, device=h.device)
    check(lib().sbk_step_proj_test(1, 0, ptr(h), d, None, None, None, ptr(wq[:d].half().contiguous()),
                                   ptr(bq[:d].contiguous()), rows, d, d, ptr(q), d, None, None, 0, 0, st), "query")
    ef = e.reshape(rows * T, d)
    kv = []
    for i in (1, 2):
        t = torch.empty(rows * T, d, dtype=torch.half, device=h.device)
        check(lib().sbk_gemm_f16_test(ptr(ef), ptr(w[i * d:(i + 1) * d].half().contiguous()),
                                      ptr(b[i * d:(i + 1) * d].contiguous()), ptr(t), 0, 0, rows * T, d, d, st), "K / V")
        kv.append(t)
    att = torch.empty(rows, d, dtype=torch.half, device=h.device)
    check(lib().sbk_dec_attention_test(ptr(q), d, ptr(kv[0]), ptr(kv[1]), ctypes.c_longlong(T * d), d, 0, 1, rows, H, d // H,
                                       T, -1, ptr(lens), None, None, 0, 0, ptr(att), d, st), "attention")
    out = x[:, :d].contiguous()
    check(lib().sbk_step_proj_test(1, 4, ptr(att), d, None, None, None, ptr(wo.half().contiguous()), ptr(bo), rows, d, d,
                                   ptr(out), d, None, None, 0, 0, st), "out_proj")
    return out


def _check_case(dev, T, rows, d, H, logit_scale, seed):
    layer = _layer(d, H, logit_scale, seed)
    h, e, lens, x = _inputs(rows, T, d, seed + 1, dev)
    out = _run(h, e, lens, x, layer, H)
    ref = _ref(h, e, lens, x, layer, H)
    assert torch.equal(out[:, d:], x[:, d:]), "columns past d were written"
    o = out[:, :d].double()
    nan_ref = torch.isnan(ref).any(-1)
    assert torch.equal(torch.isnan(o).any(-1), nan_ref) and torch.isnan(o[nan_ref]).all(), "NaN rows differ"
    assert torch.isfinite(o[~nan_ref]).all()
    emax, el2 = _metrics(o[~nan_ref], ref[~nan_ref])
    umax, ul2 = _metrics(_unfolded(h, e, lens, x, layer, H)[~nan_ref], ref[~nan_ref])
    print(f"fold T={T} rows={rows} d={d} H={H} x{logit_scale:g}: max {emax:.3e}, rel-L2 {el2:.3e}; "
          f"unfolded path {umax:.3e}, {ul2:.3e}")
    assert emax <= max(BAR[0], 1.25 * umax) and el2 <= max(BAR[1], 1.25 * ul2), (emax, el2, umax, ul2)
    assert torch.equal(_bits(_run(h, e, lens, x, layer, H)), _bits(out)), "rerun not bit-identical"
    r = rows - 1  # an utterance alone
    alone = _run(h[r:r + 1].contiguous(), e[r:r + 1].contiguous(), lens[r:r + 1].contiguous(), x[r:r + 1].contiguous(), layer, H)
    assert torch.equal(_bits(alone), _bits(out[r:r + 1])), "an utterance alone differs from the same utterance in the batch"


# ------------------------------------------------------------------------------------------------ bench shape
@pytest.fixture(scope="module")
def large(dev):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    g = torch.load(os.path.join(GOLDEN, "bench_conformer_large_rope_10s.pt"))
    cfg = dict(CONFORMER_LARGE, attention_type=g["cfg"]["attention_type"])
    return g, cfg, AsrEngine(cfg, seeded_asr_state(cfg, 0), device=dev)


def test_group_call_greedy_224_rows(dev, large):
    """7 batches of 32 (the golden's 4 utterances 8 times each) in one group call: 224 rows over T = 251 frames fold"""
    g, cfg, eng = large
    wav, lens = case_wav(g)
    B, G, S = 32, 7, g["greedy_tokens"].shape[1]
    w32, l32 = wav.repeat(B // 4, 1).to(dev), lens.repeat(B // 4).to(dev)
    preds = [torch.full((B, S), -7, dtype=torch.int32, device=dev) for _ in range(G)]
    assert eng.transcribe_greedy_group_dev([w32] * G, [l32] * G, S, 1, 2, preds) == S
    torch.cuda.synchronize()
    pred = torch.cat(preds).cpu()
    rep = G * B // 4
    check_greedy("group 7 x 32, folded", pred, torch.zeros(pred.shape), g["greedy_tokens"].repeat(rep, 1),
                 g["greedy_margin"].repeat(rep, 1), min_compared=0.6)


def test_teacher_forced_224_rows_folds(dev, large):
    """decode_teacher_forced on the decode golden repeated to 224 rows: rel-L2 <= 2e-3 against the reference, and the GEMMs
    launched are exactly the folded step's (query projection N = H d, output projection K = H d), with no K/V GEMM"""
    from speechbrain_b200 import _lib
    g, cfg, eng = large
    gd = torch.load(os.path.join(GOLDEN, "bench_decode_conformer_large_rope_10s.pt"))["decode"]
    n = 224
    rep = n // gd["tgt"].shape[0]
    tgt, enc, el = gd["tgt"].repeat(rep, 1), g["enc_out"].repeat(rep, 1, 1), gd["enc_len"].repeat(rep)
    L = _lib.lib()
    L.sbk_gemm_profile_enable(1)
    try:
        out = eng.decode_teacher_forced(tgt.to(dev), enc.to(dev), el.to(dev))
        torch.cuda.synchronize()
        cnt, fl = ctypes.c_int(), ctypes.c_double()
        _lib.check(L.sbk_gemm_profile_read(ctypes.byref(cnt), None, ctypes.byref(fl)), "sbk_gemm_profile_read")
    finally:
        L.sbk_gemm_profile_enable(0)
    S, Ld, d, F, H = tgt.shape[1], cfg["num_decoder_layers"], cfg["d_model"], cfg["d_ffn"], cfg["nhead"]
    assert cnt.value == S * Ld * 6
    assert fl.value == S * Ld * 2 * n * (3 * d * d + d * d + 2 * H * d * d + 2 * F * d)
    r = rel(out.cpu(), gd["pred"].repeat(rep, 1, 1))
    print(f"teacher-forced 224 rows, folded: rel-L2 {r:.3e}")
    assert r < 2e-3


def test_zero_length_utterance_among_224(dev, large):
    """one utterance of 224 with no encoder frame: token 0 and NaN scores on its row, every other row bit-identical to the
    same call with that utterance at full length"""
    g, cfg, eng = large
    n, steps = 224, 12
    rep = n // 4
    enc = g["enc_out"].repeat(rep, 1, 1).to(dev)
    wl = g["wav_lens"].repeat(rep).to(dev)
    wl0 = wl.clone()
    wl0[5] = 0.0
    pred, score, _, done = eng.greedy_from_enc(enc, wl0, steps, 1, 2)
    pred1, score1, _, _ = eng.greedy_from_enc(enc, wl, steps, 1, 2)
    torch.cuda.synchronize()
    assert done == steps and (pred[5] == 0).all() and torch.isnan(score[5]).all()
    keep = torch.arange(n, device=dev) != 5
    assert torch.equal(pred[keep], pred1[keep]) and torch.equal(score[keep], score1[keep])
