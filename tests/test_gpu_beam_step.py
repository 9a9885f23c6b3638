"""-m gpu parity tests of the beam-search step kernels alone, against the float64 references of decoder_kernels_oracle.py
(pinned to oracle.asr_oracle.beam_search by test_decoder_kernels_oracle.py):

- beam_step through sbk_beam_step_test on both selection paths: rows + merge (beam_rows_kernel + beam_merge_kernel) at
  beam {1, 2, 3, 10, 15, 16}, and the radix select (beam_step_large_kernel) at those widths and at {17, 32, 66, 80, 127,
  128}; vocabularies {beam, 31, 255, 256, 257, 1024, 5000, 5120}; batches {1, 3, 32};
- coverage_score through sbk_coverage_score_test: T {1, 251, 2500, 12288}, enc_len {T, ragged, 1, 0}, rows_per_utt {1,
  10, 66}, 8 heads of 64, both K layouts, steps 0 and 5;
- an utterance with no encoder frame inside AsrEngine.beam_from_enc on both paths.

The inputs are built to expose a subtly wrong kernel: diffuse (randn) and peaked (20 * randn) logits; exact ties inside a
row and across two rows of an utterance with identical logits and sequence scores; a row of V equal logits at step 0 (more
ties at the threshold than the radix select's tie buffer holds); states at step 0 and with finished rows at -inf; steps 0,
1, 37 and 499 under length normalisation; min_steps above and below the step; eos-threshold rows whose eos log-prob is
clearly above or below 1.5 * max; eos at 2 and V - 1; the CTC blank at 0 and V - 1 with the decoder weight 0.7; add_scores
with entries at -1e20 and -inf, negative add_row, nonzero length weight; the LM outputs on and off, with embeddings past
the fp16 range; eos winning in several rows so that `finished` crosses its cap; NaN rows and a whole utterance of NaN;
fewer than `beam` finite candidates.  Buffer entries a step must not write hold sentinels that must survive.

Selection: the (token, predecessor) at every rank equals the reference's, except that two candidates whose float64 scores
lie within the score bar may swap (exact ties never); NaN ranks first and ties go to the lowest candidate index.  Scores,
log-probs and the next sequence scores are within the score bar, relative to |seq| + |logit / T| + |lse| + |add| at the
candidate (divided by step + 1 under length normalisation).  Lineage, finished, n_full, the step counters and the token
cache are exact; the next decoder and LM inputs are within fp32 rounding, the LM's fp16 copy within the saturating store.
Reruns are bit-identical, an utterance alone is bit-identical to the same utterance in the batch, and the two paths agree.

Bars, about twice the worst value measured over every case of this file on an H100 80GB HBM3 (700 W power limit):
- SCORE_BAR, scores / log-probs / next sequence scores: fp32 expf / logf over V <= 5120 and the fp32 sums;
- COV_BAR, coverage and its score: __expf, fp32 sums over T <= 12288 and the fp16 keys.
The worst values are beside the bars."""
import ctypes
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401
import decoder_kernels_oracle as DK  # noqa: E402

SCORE_BAR = 2e-7     # worst 9.7e-8; the two paths apart 1.9e-7 relative to |score| + 1 (bar 2 * SCORE_BAR)
COV_BAR = 1.2e-5     # worst 6.0e-6 (score relative to its penalty terms, coverage relative to |c| + 1 / T)

pytestmark = pytest.mark.gpu
SENT = -777.0
ISENT = -7
NEG = float("-inf")
WORST = {"score": 0.0, "cov": 0.0}


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


# ------------------------------------------------------------------------------------------------ inputs
def _state(B, beam, V, step, seed, kind="diffuse", T=1.0, ties=False, cross_ties=False, flat_row=False, dead=False,
           nan_rows=(), nan_utt=None, eos=2, lm=False, add=False, add_row=False, few=False, eos_win=False):
    """host tensors of one beam step: logits, seq (the parity read at `step`), finished counters, lineage table, add
    scores / add_row, embedding tables"""
    g = torch.Generator().manual_seed(seed)
    n = B * beam
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    lg = r(n, V) * (20.0 if kind == "peaked" else 1.0)
    if step == 0:
        seq = torch.full((n,), NEG)
        seq[::beam] = 0.0
    else:
        seq = -(step + 1) * (1.0 + torch.rand(n, generator=g))
        if dead:   # finished rows at -inf
            seq[1::3] = NEG
    if ties:       # repeated values inside every row, at the top of the row
        top = lg.argmax(-1)
        for k in range(4):
            j = (top + 1 + 7 * k) % V
            lg[torch.arange(n), j] = lg[torch.arange(n), top]
    if cross_ties and beam >= 2:   # rows 0 and 1 of every utterance identical
        lg.view(B, beam, V)[:, 1] = lg.view(B, beam, V)[:, 0]
        seq.view(B, beam)[:, 1] = seq.view(B, beam)[:, 0]
    if flat_row:
        lg[0] = 0.25
    if eos_win:   # eos the clear winner in several rows
        lg[::2, eos] = lg[::2].max(-1).values + 30.0
    if few:       # one finite logit per row: fewer than `beam` finite candidates at step 0
        keep = lg.argmax(-1)
        lg[:] = NEG
        lg[torch.arange(n), keep] = 1.0
        lg[:, eos] = NEG
    for i in nan_rows:
        if i < n:
            lg[i] = float("nan")
    if nan_utt is not None:
        lg[nan_utt * beam:(nan_utt + 1) * beam] = float("nan")
    out = {"B": B, "logits": lg, "seq": seq, "finished": torch.randint(0, max(beam - 1, 1), (B,), generator=g, dtype=torch.int32)}
    if eos_win:
        out["finished"][0] = beam - 1
        if B > 1:
            out["finished"][1] = beam
    S = step + 3
    out["S_max"] = S
    rr = torch.arange(n).view(n, 1)
    out["lin"] = ((rr + 1 + torch.randint(0, max(n - 1, 1), (2, n, S), generator=g)) % n).to(torch.int32)
    out["add"] = None
    if add:
        a = -3.0 * torch.rand(n, V, generator=g)
        a[:, 1::17] = -1e20
        a[:, 5::29] = NEG
        out["add"] = a
    out["add_row"] = -2.0 * torch.rand(n, generator=g) if add_row else None
    d = 16
    out["emb"], out["pe"] = r(V, d), r(S, d)
    out["lm"] = (3000.0 * r(V, 64), r(S, 64)) if lm else None
    return out


def _params(beam, eos=2, min_steps=0, T=1.0, thr=False, ln=True, minus_inf=-1e20, ctc=0.0, blank=-1, lw=0.0):
    from speechbrain_b200._lib import sbk_beam_params
    return sbk_beam_params(beam, 0, min_steps, 1, eos, T, int(thr), 1.5, int(ln), minus_inf, 0.0, 1.0, ctc, blank, lw, 0.0, 0.5)


def _run(st, p, path, step, dev, n_hist=None):
    """-> (rc, dict of device outputs incl. sentinel regions)"""
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    lg = st["logits"]
    n, V = lg.shape
    B = st["B"]
    S = st["S_max"]
    H = n_hist if n_hist is not None else step + 2
    t = lambda x, **k: x.contiguous().to(dev, **k)  # noqa: E731
    o = {"seq": torch.full((2, n + 1), SENT), "lin": st["lin"].clone(), "step": torch.full((n + 1,), ISENT, dtype=torch.int32),
         "fin": torch.full((B + 1,), ISENT, dtype=torch.int32), "n_full": torch.tensor([3], dtype=torch.int32),
         "tok": torch.full((H, n + 1), ISENT, dtype=torch.int32), "pred": torch.full((H, n + 1), ISENT, dtype=torch.int32),
         "score": torch.full((H, n + 1), SENT), "lp": torch.full((H, n + 1), SENT), "x": torch.full((n + 1, 16), SENT)}
    o["seq"][step & 1, :n] = st["seq"]
    o["step"][:n] = step
    o["fin"][:B] = st["finished"]
    lm = st["lm"]
    if lm is not None:
        o["lm_x"] = torch.full((n + 1, 64), SENT)
        o["lm_x16"] = torch.full((n + 1, 64), SENT, dtype=torch.float16)
        o["tok_cache"] = torch.full((n + 1, S), ISENT, dtype=torch.int32)
    o = {k: t(v) for k, v in o.items()}
    # the hook takes [2][n_bh] / [n_hist][n_bh] buffers: pass views without the sentinel column
    seq = o["seq"][:, :n].contiguous()
    hist = {k: o[k][:, :n].contiguous() for k in ("tok", "pred", "score", "lp")}
    dl = {k: t(v) for k, v in (("lg", lg), ("emb", st["emb"]), ("pe", st["pe"]))}
    add = t(st["add"]) if st["add"] is not None else None
    arow = t(st["add_row"]) if st["add_row"] is not None else None
    lme = lmp = None
    if lm is not None:
        lme, lmp = t(lm[0]), t(lm[1])
    rc = lib().sbk_beam_step_test(ctypes.byref(p), path, B, V, S, H, ptr(dl["lg"]), ptr(seq), ptr(o["lin"]), ptr(o["step"]),
                                  ptr(o["fin"]), ptr(o["n_full"]), ptr(hist["tok"]), ptr(hist["pred"]), ptr(hist["score"]),
                                  ptr(hist["lp"]), ptr(add), ptr(arow), ptr(dl["emb"]), ptr(dl["pe"]), 16, ptr(o["x"]),
                                  ptr(lme), ptr(lmp), 64 if lm is not None else 0, ptr(o.get("lm_x")), ptr(o.get("lm_x16")),
                                  ptr(o.get("tok_cache")), stream_ptr(dev))
    torch.cuda.synchronize(dev)
    o["seq"][:, :n] = seq
    for k in hist:
        o[k][:, :n] = hist[k]
    return rc, {k: v.cpu() for k, v in o.items()}


def _ref(st, p, step):
    kw = dict(min_steps=p.min_steps, temperature=p.temperature, using_eos_threshold=bool(p.using_eos_threshold),
              eos_threshold=p.eos_threshold, length_normalization=bool(p.length_normalization), minus_inf=p.minus_inf,
              length_weight=p.length_weight)
    if p.ctc_weight != 0.0:
        kw.update(ctc_weight=p.ctc_weight, blank=p.blank_index)
    lm = st["lm"]
    return DK.beam_step_ref(st["logits"], st["seq"], step, p.beam_size, p.eos, add_scores=st["add"], add_row=st["add_row"],
                            finished=st["finished"], lineage=st["lin"][step & 1], emb=st["emb"], pe=st["pe"],
                            lm_emb=None if lm is None else lm[0], lm_pe=None if lm is None else lm[1], **kw)


def _scale(st, p, step):
    """|seq| + |logit / T| + |lse| + |add| per candidate (non-finite parts 0), / (step + 1) under length normalisation"""
    lg = st["logits"].double() / p.temperature
    fin = lambda x: torch.where(torch.isfinite(x), x.abs(), torch.zeros_like(x))  # noqa: E731
    lse = torch.logsumexp(lg, -1, keepdim=True)
    s = fin(st["seq"].double()).view(-1, 1) + fin(lg) + fin(lse) + abs(p.length_weight)
    if st["add"] is not None:
        s = s + fin(st["add"].double())
    if st["add_row"] is not None:
        s = s + fin(st["add_row"].double()).view(-1, 1)
    return s / (step + 1) if p.length_normalization else s, fin(lg) + fin(lse)


def _close(got, ref, scale, what, name):
    """NaN / inf where the reference has them, |d| <= SCORE_BAR * (scale + |ref|) elsewhere"""
    got, ref = got.double(), ref.double()
    same = torch.equal(torch.isnan(got), torch.isnan(ref)) and torch.equal(torch.isinf(got), torch.isinf(ref))
    same = same and torch.equal(got[torch.isinf(ref)], ref[torch.isinf(ref)])
    f = torch.isfinite(ref)
    err = float(((got[f] - ref[f]).abs() / (scale[f] + ref[f].abs())).max()) if f.any() else 0.0
    WORST["score"] = max(WORST["score"], err)
    print(f"MEASURE beam {what} {name}: {err:.3e} (bar {SCORE_BAR})")
    assert same and err <= SCORE_BAR, f"{name} {what}: rel err {err:.3e} (bar {SCORE_BAR}), non-finite as ref {same}"


def _check(st, p, path, step, o, name):
    n, V = st["logits"].shape
    B, beam = st["B"], p.beam_size
    ref = _ref(st, p, step)
    scale, lp_scale = _scale(st, p, step)
    sc = ref["sc"]
    tok, pred = o["tok"][step, :n].long(), o["pred"][step, :n].long()
    # selection: rank by rank, a different candidate only inside a near-tie group (never an exact float64 tie)
    for u in range(B):
        for k in range(beam):
            i = u * beam + k
            a, b = (int(pred[i]), int(tok[i])), (int(ref["pred"][i]), int(ref["tok"][i]))
            if a == b:
                continue
            assert 0 <= a[0] - u * beam < beam and 0 <= a[1] < V, f"{name}: rank {k} of utt {u}: {a} outside the utterance"
            x, y = sc[a], sc[b]
            tol = SCORE_BAR * (scale[a] + scale[b] + x.abs() + y.abs())
            assert torch.isfinite(x) and torch.isfinite(y) and x != y and (x - y).abs() <= tol, \
                f"{name}: rank {k} of utt {u}: kernel {a} ({float(x)}) vs reference {b} ({float(y)})"
        sel = set(zip(pred[u * beam:(u + 1) * beam].tolist(), tok[u * beam:(u + 1) * beam].tolist()))
        assert len(sel) == beam, f"{name}: utt {u} selected a candidate twice"
    # scores, log-probs and next sequence scores of the kernel's own candidates (a near-tie swap keeps its own score)
    idx = (pred, tok)
    lp_full = torch.log_softmax(st["logits"].double() / p.temperature, -1) * (1.0 - p.ctc_weight)
    mul = (step + 1) if p.length_normalization else 1
    _close(o["score"][step, :n], sc[idx], scale[idx], "score", name)
    _close(o["lp"][step, :n], lp_full[idx], lp_scale[idx], "lp", name)
    seq_next = torch.where(tok == p.eos, torch.full_like(sc[idx], NEG), sc[idx] * mul)
    _close(o["seq"][(step + 1) & 1, :n], seq_next, scale[idx] * mul, "seq", name)
    # exact outputs of that selection
    exact = _bookkeeping(st, step, tok, pred, beam, p.eos)
    assert torch.equal(o["lin"][(step + 1) & 1][:, :step + 2].long(), exact["lineage"][:, :step + 2]), f"{name}: lineage"
    assert torch.equal(o["lin"][(step + 1) & 1][:, step + 2:], st["lin"][(step + 1) & 1][:, step + 2:]), f"{name}: lineage sentinels"
    assert torch.equal(o["lin"][step & 1], st["lin"][step & 1]), f"{name}: the read lineage table changed"
    assert torch.equal(o["fin"][:B].long(), exact["finished"]) and int(o["fin"][B]) == ISENT, f"{name}: finished"
    assert int(o["n_full"][0]) == 3 + exact["n_full"], f"{name}: n_full {int(o['n_full'][0])}, expected {3 + exact['n_full']}"
    assert (o["step"][:n] == step + 1).all() and int(o["step"][n]) == ISENT, f"{name}: step counters"
    x_ref = exact["x"]
    assert float(((o["x"][:n].double() - x_ref).abs() / (x_ref.abs() + 1.0)).max()) <= 1e-6 and (o["x"][n] == SENT).all(), \
        f"{name}: x_next"
    if st["lm"] is not None:
        lx = exact["lm_x"]
        assert float(((o["lm_x"][:n].double() - lx).abs() / (lx.abs() + 1.0)).max()) <= 1e-6, f"{name}: LM x"
        l16 = exact["lm_x16"]
        assert float(((o["lm_x16"][:n].double() - l16).abs() / (l16.abs() + 1e-3)).max()) <= 2.0 ** -11, f"{name}: LM x16"
        tc = o["tok_cache"]
        assert torch.equal(tc[:n, step + 1].long(), tok), f"{name}: token cache"
        others = [c for c in range(st["S_max"]) if c != step + 1]
        assert (tc[:, others] == ISENT).all() and (tc[n] == ISENT).all(), f"{name}: token cache sentinels"
    assert torch.equal(_bits(o["seq"][step & 1, :n]), _bits(st["seq"])), f"{name}: the read seq_scores changed"
    assert (o["seq"][:, n] == SENT).all(), f"{name}: seq_scores sentinel"
    for k in ("tok", "pred", "score", "lp"):
        others = [s for s in range(o[k].shape[0]) if s != step]
        assert (o[k][others] == (ISENT if k in ("tok", "pred") else SENT)).all() and (o[k][:, n] == (
            ISENT if k in ("tok", "pred") else SENT)).all(), f"{name}: history {k} of other steps"
    return ref


def _bookkeeping(st, step, tok, pred, beam, eos):
    """lineage, finished, n_full, x_next and the LM outputs of a given selection"""
    n = tok.shape[0]
    B = n // beam
    lin_in = st["lin"][step & 1].long()
    lin = st["lin"][(step + 1) & 1].long().clone()
    lin[:, :step] = lin_in[pred, :step]
    lin[:, step] = pred
    lin[:, step + 1] = torch.arange(n)
    before = st["finished"].long()
    after = torch.clamp(before + (tok == eos).view(B, beam).sum(1), max=beam)
    out = {"lineage": lin, "finished": after, "n_full": int(((before < beam) & (after >= beam)).sum()),
           "x": st["emb"].double()[tok] * math.sqrt(16) + st["pe"].double()[step + 1]}
    if st["lm"] is not None:
        e, pe = st["lm"]
        out["lm_x"] = e.double()[tok] * math.sqrt(64) + pe.double()[step + 1]
        out["lm_x16"] = out["lm_x"].clamp(-DK.FP16_MAX, DK.FP16_MAX)
    return out


def _alone(st, u, beam):
    """the inputs of utterance u alone"""
    sl = slice(u * beam, (u + 1) * beam)
    one = dict(st)
    one["B"] = 1
    one["logits"], one["seq"] = st["logits"][sl].contiguous(), st["seq"][sl].contiguous()
    one["finished"] = st["finished"][u:u + 1].clone()
    one["lin"] = torch.zeros(2, beam, st["S_max"], dtype=torch.int32)
    one["add"] = None if st["add"] is None else st["add"][sl].contiguous()
    one["add_row"] = None if st["add_row"] is None else st["add_row"][sl].contiguous()
    return one


def _case(st, p, paths, step, dev, name, alone=True):
    """every check of one input state on the given paths; -> {path: outputs}"""
    n, B, beam = st["logits"].shape[0], st["B"], p.beam_size
    outs = {}
    for path in paths:
        nm = f"{name} path={path}"
        rc, o = _run(st, p, path, step, dev)
        assert rc == 0, nm
        _check(st, p, path, step, o, nm)
        rc, o2 = _run(st, p, path, step, dev)
        assert rc == 0 and all(torch.equal(_bits(o[k]), _bits(o2[k])) for k in o), f"{nm}: rerun differs"
        if alone and B > 1:
            u = B - 1
            rc, o1 = _run(_alone(st, u, beam), p, path, step, dev)
            sl = slice(u * beam, (u + 1) * beam)
            assert rc == 0
            same = (torch.equal(_bits(o1["score"][step, :beam]), _bits(o["score"][step, sl]))
                    and torch.equal(_bits(o1["lp"][step, :beam]), _bits(o["lp"][step, sl]))
                    and torch.equal(o1["tok"][step, :beam], o["tok"][step, sl])
                    and torch.equal(o1["pred"][step, :beam] + u * beam, o["pred"][step, sl])
                    and torch.equal(_bits(o1["seq"][(step + 1) & 1, :beam]), _bits(o["seq"][(step + 1) & 1, sl]))
                    and torch.equal(_bits(o1["x"][:beam]), _bits(o["x"][sl]))
                    and int(o1["fin"][0]) == int(o["fin"][u]))
            assert same, f"{nm}: utterance {u} alone differs"
        outs[path] = o
    if len(outs) == 2:   # the two paths: the same selections up to near-tie swaps (each checked against the reference)
        a, b = outs[1], outs[2]
        sa, sb = a["score"][step, :n].double(), b["score"][step, :n].double()
        f = torch.isfinite(sa) & torch.isfinite(sb)
        assert torch.equal(torch.isnan(sa), torch.isnan(sb)) and torch.equal(sa[torch.isinf(sa)], sb[torch.isinf(sb)])
        err = float(((sa[f] - sb[f]).abs() / (sa[f].abs() + 1.0)).max()) if f.any() else 0.0
        print(f"MEASURE beam paths {name}: {err:.3e}")
        assert err <= 2 * SCORE_BAR, f"{name}: paths apart {err:.3e}"
    return outs


SMALL = [1, 2, 3, 10, 15, 16]
LARGE = [17, 32, 66, 80, 127, 128]
VOCABS = [None, 31, 255, 256, 257, 1024, 5000, 5120]   # None: V = beam


def _vocabs(beam):
    return [v if v is not None else beam for v in VOCABS if v is None or v >= beam]


@pytest.mark.parametrize("beam", SMALL + LARGE)
def test_beam_step_widths(dev, beam):
    """every vocabulary at this width, batches 1 / 3 (32 at V = 1024), diffuse and peaked logits at step 0 and at step 37
    with finished rows, ties inside and across rows, the LM outputs at every other vocabulary"""
    paths = (1, 2) if beam <= 16 else (2,)
    for vi, V in enumerate(_vocabs(beam)):
        for B in ((1, 3, 32) if V == 1024 and beam <= 32 else (1, 3)):
            for step, kind in ((0, "diffuse"), (37, "peaked")):
                seed = beam * 1009 + V * 7 + B * 3 + step
                st = _state(B, beam, V, step, seed, kind, ties=True, cross_ties=step > 0, dead=step > 0, lm=vi % 2 == 0)
                p = _params(beam, eos=2 if V > 2 and vi % 2 else V - 1)
                _case(st, p, paths, step, dev, f"beam={beam} V={V} B={B} step={step} {kind}")


# (name, state kwargs, params kwargs, step)
SCENARIOS = [
    ("flat row at step 0", dict(flat_row=True), dict(), 0),
    ("length norm step 1", dict(dead=True), dict(), 1),
    ("length norm step 499", dict(dead=True, kind="peaked"), dict(), 499),
    ("no length norm", dict(dead=True), dict(ln=False), 5),
    ("min_steps above", dict(), dict(min_steps=3), 2),
    ("min_steps below", dict(), dict(min_steps=2), 3),
    ("eos threshold", dict(), dict(thr=True), 4),
    ("eos threshold temperature", dict(), dict(thr=True, T=1.7), 4),
    ("ctc blank 0", dict(add=True), dict(ctc=0.3, blank=0), 3),
    ("ctc blank V-1", dict(add=True, add_row=True), dict(ctc=0.3, blank=-1, lw=0.6), 3),
    ("coverage and length", dict(add_row=True, lm=True), dict(lw=-0.4), 6),
    ("eos wins", dict(eos_win=True), dict(), 2),
    ("NaN rows", dict(nan_rows=(0, 4)), dict(), 3),
    ("NaN utterance", dict(nan_utt=1), dict(), 0),
    ("NaN utterance later", dict(nan_utt=0), dict(thr=True), 7),
    ("few finite", dict(few=True), dict(minus_inf=NEG), 0),
    ("few finite eos", dict(few=True), dict(minus_inf=NEG, min_steps=5, eos=0), 0),
]


@pytest.mark.parametrize("beam", [1, 3, 10, 16, 17, 66, 128])
@pytest.mark.parametrize("V", [257, 5000])
def test_beam_step_scenarios(dev, beam, V):
    """the edge states of SCENARIOS at B = 3 on both paths where they apply"""
    paths = (1, 2) if beam <= 16 else (2,)
    for i, (name, skw, pkw, step) in enumerate(SCENARIOS):
        pkw = dict(pkw)
        if pkw.get("blank") == -1:
            pkw["blank"] = V - 1
        st = _state(3, beam, V, step, beam * 131 + V + i, **skw)
        if "eos threshold" in name:   # eos log-prob 1.2 x max (kept) in rows 0, 3, ..., 1.8 x max (masked) elsewhere
            lg, eos, Tm = st["logits"], 2, pkw.get("T", 1.0)
            c = torch.where(torch.arange(lg.shape[0]) % 3 == 0, 1.2, 1.8).double()
            other = torch.arange(V) != eos
            for _ in range(6):   # the eos logit moves the log-sum-exp: iterate to the fixed point
                lse = torch.logsumexp(lg.double() / Tm, -1)
                m = (lg.double()[:, other] / Tm).max(-1).values - lse
                lg[:, eos] = ((c * m + lse) * Tm).float()
            lp = torch.log_softmax(lg.double() / Tm, -1)
            margin = float((lp[:, eos] - 1.5 * lp.max(-1).values).abs().min())
            assert margin > 1e-3, f"eos-threshold margin {margin:.2e}"
        p = _params(beam, **pkw)
        _case(st, p, paths, step, dev, f"{name} beam={beam} V={V}")


def test_beam_step_rejects_bad_arguments(dev):
    """host checks: beam outside [1, 128] or above V, path 1 past beam 16, an unknown path, rows of an utterance at
    different steps, step + 1 >= S_max, step >= n_hist, a lineage entry outside [0, n_bh): an error, nothing written"""
    beam, V, step = 4, 40, 2
    st = _state(2, beam, V, step, 5)
    p = _params(beam)
    assert _run(st, p, 2, step, dev)[0] == 0

    def rejected(st_, p_, path=2, step_=step, n_hist=None, mutate=None):
        s2 = dict(st_)
        if mutate:
            mutate(s2)
        rc, o = _run(s2, p_, path, step_, dev, n_hist=n_hist)
        untouched = (o["tok"][:, :-1] == ISENT).all() and (o["x"] == SENT).all() and (o["step"][:-1] == step_).all()
        return rc != 0 and bool(untouched)

    assert rejected(st, _params(0)) and rejected(st, _params(129))
    big = _state(1, 17, 17, step, 6)
    assert rejected(big, _params(17), path=1) and rejected(st, p, path=3) and rejected(st, p, path=-1)
    assert rejected(_state(1, 4, 3, step, 7), _params(4))                   # beam > V
    assert rejected(st, p, step_=st["S_max"] - 1)                           # step + 1 >= S_max
    assert rejected(st, p, n_hist=step)                                     # step >= n_hist

    def bad_lin(s2):
        s2["lin"] = s2["lin"].clone()
        s2["lin"][1, 3, 4] = 8
    assert rejected(st, p, mutate=bad_lin)

    def neg_lin(s2):
        s2["lin"] = s2["lin"].clone()
        s2["lin"][0, 0, 0] = -1
    assert rejected(st, p, mutate=neg_lin)
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    # rows of one utterance at different steps
    n = 2 * beam
    stp = torch.full((n,), step, dtype=torch.int32, device=dev)
    stp[1] = step + 1
    buf = lambda *s: torch.full(s, SENT, device=dev)  # noqa: E731
    ibuf = lambda *s: torch.full(s, ISENT, dtype=torch.int32, device=dev)  # noqa: E731
    tok = ibuf(step + 2, n)
    rc = lib().sbk_beam_step_test(ctypes.byref(p), 2, 2, V, st["S_max"], step + 2, ptr(st["logits"].to(dev)), ptr(buf(2, n)),
                                  ptr(st["lin"].to(dev)), ptr(stp), ptr(ibuf(2)), ptr(ibuf(1)), ptr(tok), ptr(ibuf(step + 2, n)),
                                  ptr(buf(step + 2, n)), ptr(buf(step + 2, n)), None, None, ptr(st["emb"].to(dev)),
                                  ptr(st["pe"].to(dev)), 16, ptr(buf(n, 16)), None, None, 0, None, None, None, stream_ptr(dev))
    assert rc != 0 and (tok == ISENT).all() and int(stp[1]) == step + 1


# ------------------------------------------------------------------------------------------------ coverage
def _cov_run(q, K, layout, lens, rpu, cov, hist_pred, step, thr, w, dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    U, T, H, dh = K.shape
    d = H * dh
    if layout == "head":
        buf = K.permute(0, 2, 1, 3).contiguous()
        us, ks, hs = T * d, 64, T * 64
    else:
        buf = torch.cat([K.reshape(U, T, d), torch.zeros_like(K).reshape(U, T, d)], dim=-1).contiguous()
        us, ks, hs = T * 2 * d, 2 * d, 64
    n = q.shape[0]
    steps = torch.full((n,), step, dtype=torch.int32, device=dev)
    out = torch.full((n + 1,), SENT, device=dev)
    rc = lib().sbk_coverage_score_test(ptr(q), d, ptr(buf), ctypes.c_longlong(us), ks, hs, ptr(lens), rpu, T, H, ptr(cov),
                                       ptr(hist_pred), ptr(steps), n, ctypes.c_float(thr), ctypes.c_float(w), ptr(out),
                                       stream_ptr(dev))
    torch.cuda.synchronize(dev)
    return rc, out.cpu(), cov.cpu()


@pytest.mark.parametrize("layout", ["head", "row"])
@pytest.mark.parametrize("T", [1, 251, 2500, 12288])
def test_coverage_score(dev, T, layout):
    """4 utterances with enc_len {T, ragged, 1, 0}, rows_per_utt {1, 10, 66}, 8 heads of 64, steps 0 and 5 (predecessors
    never the row itself); the coverage written, the score within the bar, NaN exactly for the utterance with no frame;
    the coverage table of the other parity untouched; reruns bit-identical"""
    H, dh, U = 8, 64, 4
    for rpu in (1, 10, 66):
        for step in (0, 5):
            name = f"coverage T={T} {layout} rows_per_utt={rpu} step={step}"
            g = torch.Generator().manual_seed(T * 13 + rpu * 7 + step + len(layout))
            n = U * rpu
            lens = torch.tensor([T, max(1, (2 * T) // 3), 1, 0], dtype=torch.int32)
            K = torch.randn(U, T, H, dh, generator=g).half()
            q = ((3.0 / 8.0) * torch.randn(n, H, dh, generator=g)).half()
            rr = torch.arange(n)
            pred = ((rr + 1 + torch.randint(0, max(n - 1, 1), (n,), generator=g)) % n) if n > 1 else rr
            hist_pred = torch.full((6, n), ISENT, dtype=torch.int32)
            hist_pred[max(step - 1, 0)] = pred.to(torch.int32)
            cov0 = torch.full((2, n, T), SENT)
            prev = torch.rand(n, T, generator=g) * 0.3
            cov0[step & 1] = prev
            thr, w = 0.5, 0.8
            rc, out, cov = _cov_run(q.to(dev), K.to(dev), layout, lens.to(dev), rpu, cov0.clone().to(dev),
                                    hist_pred.to(dev), step, thr, w, dev)
            assert rc == 0, name
            att = DK.cross_attention_probs(q.view(n, H, dh), K, lens, rpu)
            cprev = torch.zeros(n, T, dtype=torch.float64) if step == 0 else prev.double()[pred.long()]
            c_ref, s_ref = DK.coverage_ref(att, cprev, step, thr, w)
            nan = torch.isnan(s_ref)
            assert torch.equal(torch.isnan(out[:n]), nan) and bool(nan[3 * rpu:].all()) and not bool(nan[:3 * rpu].any()), \
                f"{name}: NaN rows {torch.isnan(out[:n]).nonzero().flatten().tolist()}"
            f = ~nan
            scl = (c_ref[f].abs().clamp_min(thr).sum(-1) + T * thr) * w / (step + 1)
            err = float(((out[:n][f].double() - s_ref[f]).abs() / scl).max())
            cerr = float(((cov[(step + 1) & 1][f].double() - c_ref[f]).abs() / (c_ref[f].abs() + 1.0 / max(T, 1))).max())
            WORST["cov"] = max(WORST["cov"], err, cerr)
            print(f"MEASURE coverage {name}: score {err:.3e}, coverage {cerr:.3e} (bar {COV_BAR})")
            assert err <= COV_BAR and cerr <= COV_BAR, f"{name}: score {err:.3e} coverage {cerr:.3e} (bar {COV_BAR})"
            assert torch.isnan(cov[(step + 1) & 1][nan]).all(), f"{name}: coverage of the empty utterance"
            assert torch.equal(_bits(cov[step & 1]), _bits(cov0[step & 1])) and float(out[n]) == SENT, f"{name}: sentinels"
            rc, out2, cov2 = _cov_run(q.to(dev), K.to(dev), layout, lens.to(dev), rpu, cov0.clone().to(dev),
                                      hist_pred.to(dev), step, thr, w, dev)
            assert rc == 0 and torch.equal(_bits(out), _bits(out2)) and torch.equal(_bits(cov), _bits(cov2)), \
                f"{name}: rerun differs"


# ------------------------------------------------------------------------------------------------ engine level
@pytest.fixture(scope="module")
def small_asr(dev):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    cfg = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=2)
    sd = seeded_asr_state(cfg, 0)
    return cfg, sd, AsrEngine(cfg, sd, device=dev)


def _utt_hist(h, u, beam, n):
    """utterance u's columns of a device history, predecessors relative to the utterance"""
    tok, pred, score, lp = h
    sl = slice(u * beam, (u + 1) * beam)
    return tok[:n, sl], pred[:n, sl] - u * beam, score[:n, sl], lp[:n, sl]


@pytest.mark.parametrize("beam", [10, 66])
def test_beam_zero_length_utterance(dev, small_asr, beam):
    """wav_lens [1.0, 0.0, 0.6] at beam 10 (rows + merge) and 66 (radix select): the empty utterance's NaN logits do not
    reach the others, whose histories and replayed hypotheses, scores and log-probs are bit-identical to a run without
    it; a second run is bit-identical"""
    from speechbrain_b200.decoders.seq2seq import replay_beam_history
    cfg, sd, eng = small_asr
    T, steps = 40, 12
    g = torch.Generator().manual_seed(8 + beam)
    enc = torch.randn(3, T, cfg["d_model"], generator=g)
    wl = torch.tensor([1.0, 0.0, 0.6])
    h = eng.beam_from_enc(enc.to(dev), wl.to(dev), beam, steps, 0, 1, 2)
    h2 = eng.beam_from_enc(enc.to(dev), wl.to(dev), beam, steps, 0, 1, 2)
    assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(h, h2)), "rerun differs"
    hs = eng.beam_from_enc(enc[[0, 2]].contiguous().to(dev), wl[[0, 2]].to(dev), beam, steps, 0, 1, 2)
    n = min(h[0].shape[0], hs[0].shape[0])
    assert n >= 1
    for u, us in ((0, 0), (2, 1)):
        a, b = _utt_hist(h, u, beam, n), _utt_hist(hs, us, beam, n)
        assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(a, b)), f"utterance {u} differs"
        ra = replay_beam_history(tuple(x.contiguous() for x in _utt_hist(h, u, beam, h[0].shape[0])), 1, beam, 2)
        rb = replay_beam_history(tuple(x.contiguous() for x in _utt_hist(hs, us, beam, hs[0].shape[0])), 1, beam, 2)
        assert all(torch.equal(_bits(x.float()), _bits(y.float())) for x, y in zip(ra, rb)), f"utterance {u} replay differs"
    assert torch.isnan(h[2][:n, beam:2 * beam]).any()
