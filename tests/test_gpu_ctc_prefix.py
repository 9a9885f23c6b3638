"""-m gpu: the CTC prefix scorer kernels (csrc/ctc_scorer.cu) on their own, through the sbk_ctc_prefix_test hook, vs the
float64 oracle (oracle.ctc_prefix_scores, pinned to the reference's CTCPrefixScore by tests/test_ctc_prefix_golden.py) on
every (row, token) of every step of a forced search history.

Comparison, on the extensions of every prefix the reference calls possible (psi_prev > -1e19):
  - an entry is impossible (<= -1e19: the blank column, extensions past the last frame) in the kernel iff in the oracle;
  - every other entry: |kernel - oracle| <= ATOL + RTOL * (|psi| + |psi_prev|).  The RTOL term is the fp32 rounding of
    forward variables of magnitude ~T log V, which the reference's own fp32 run carries too (printed beside it where
    the full-tensor oracle fits in memory).
Cases cover every compiled group width R (checked with the width the hook reports), the bulk-copy and the per-thread-load
paths (V % 4), the log-domain fallback (peaked posteriors: the oracle counts the entries whose every term lies more than
69 + log T nats below the row maximum), blank 0 and V - 1, T from 1 to 10240, ragged enc_len down to 0, steps past enc_len
and up to T, and scores accumulated onto LM addends.  Cases at T >= 2458 need more than 48 KB of dynamic shared memory in
the state-update kernel (T >= 6145 in the init kernel); they run in a fresh interpreter, because whether the kernel
attribute is set can depend on what ran earlier in a process.  So do the end-to-end beam searches at T = 3000 and 6200."""
import ctypes
import json
import math
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
pytestmark = pytest.mark.gpu

ATOL, RTOL = 2e-4, 4e-6
BOS, EOS = 1, 2


def _case(name, B, T, V, beam, blank=0, regime="diffuse", n_steps=4, enc_len=None, weight=0.4, accumulate=False, seed=0):
    return dict(name=name, B=B, T=T, V=V, beam=beam, blank=blank, regime=regime, n_steps=n_steps,
                enc_len=enc_len if enc_len is not None else [T] * B, weight=weight, accumulate=accumulate, seed=seed)


# (beam, T) pairs that reach every compiled group width; V = 5000 (the recipe), 5001, 256, 61, 31
CASES = [
    _case("b16_T1216_V257", 1, 1216, 257, 16, regime="peaked", n_steps=3, seed=1),
    _case("b12_V5000_peaked", 2, 300, 5000, 12, regime="peaked", n_steps=4, enc_len=[300, 211], seed=2),
    _case("b11_V5001_blankV-1", 1, 251, 5001, 11, blank=5000, n_steps=4, seed=3),
    _case("b10_recipe", 2, 251, 5000, 10, regime="peaked", n_steps=5, enc_len=[251, 150], seed=4),
    _case("b8_V61_blankV-1_to_T", 2, 40, 61, 8, blank=60, regime="peaked", n_steps=41, enc_len=[40, 17], seed=5),
    _case("b6_V31_to_T", 3, 37, 31, 6, n_steps=38, enc_len=[37, 1, 20], seed=6),
    _case("b5_T5", 2, 5, 61, 5, regime="peaked", n_steps=6, enc_len=[5, 2], seed=7),
    _case("b4_T1001_V256", 1, 1001, 256, 4, regime="peaked", n_steps=4, seed=8),
    _case("b3_T3_blankV-1", 2, 3, 31, 3, blank=30, n_steps=4, enc_len=[3, 1], seed=9),
    _case("b2_T2", 2, 2, 64, 2, n_steps=3, enc_len=[2, 1], seed=10),
    _case("b7_T1", 1, 1, 61, 7, regime="peaked", n_steps=2, seed=11),
    _case("b7_T251_V5000", 1, 251, 5000, 7, regime="peaked", n_steps=4, seed=12),
    _case("enc_len0", 2, 24, 64, 4, regime="peaked", n_steps=6, enc_len=[24, 0], seed=13),
    _case("acc_w0.4", 2, 60, 300, 4, n_steps=4, enc_len=[60, 33], accumulate=True, seed=14),
    _case("acc_w1.0_peaked", 2, 60, 5000, 4, regime="peaked", n_steps=4, weight=1.0, accumulate=True, seed=15),
]
# more than 48 KB of dynamic shared memory in ctc_update (T >= 2458) / ctc_init (T >= 6145); first in a fresh process
LONG_CASES = [
    _case("T2458_b4", 1, 2458, 256, 4, regime="peaked", n_steps=3, seed=20),
    _case("T2500_b66", 1, 2500, 61, 66, regime="peaked", n_steps=3, seed=21),
    _case("T2500_b128", 1, 2500, 64, 128, n_steps=2, seed=22),
    _case("T6145_b2", 1, 6145, 32, 2, regime="peaked", n_steps=3, seed=23),
    _case("T10240_b2", 2, 10240, 31, 2, regime="peaked", n_steps=3, enc_len=[10240, 7000], seed=24),
]


def _logits(c):
    """diffuse: random logits at scale 1.  peaked (a trained CTC head): logits at scale 30, the blank +12, and on 40 % of
    the frames one token +30 -- most tokens sit about 100 nats below the frame's best, which sends their sums (every term
    below e^-69 of the row maximum) to the log-domain fallback."""
    g = torch.Generator().manual_seed(1000 + c["seed"])
    B, T, V = c["B"], c["T"], c["V"]
    if c["regime"] == "diffuse":
        return torch.randn(B, T, V, generator=g)
    x = torch.randn(B, T, V, generator=g) * 30.0
    x[:, :, c["blank"]] += 12.0
    spike = torch.rand(B, T, generator=g) < 0.4
    tok = torch.randint(0, V, (B, T), generator=g)
    x.scatter_add_(2, tok.unsqueeze(-1), (30.0 * spike.float()).unsqueeze(-1))
    return x


def _hook(logits, enc_len, beam, blank, weight, hist_tok, hist_pred, n_steps, addend=None):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    B, T, V = logits.shape
    dev = torch.device("cuda:0")
    lg, el = logits.contiguous().to(dev), enc_len.to(torch.int32).to(dev)
    ht, hp = hist_tok.to(torch.int32).contiguous().to(dev), hist_pred.to(torch.int32).contiguous().to(dev)
    out = addend.clone().to(dev) if addend is not None else torch.full((n_steps, B * beam, V), float("nan"), device=dev)
    width = ctypes.c_int(-1)
    check(lib().sbk_ctc_prefix_test(ptr(lg), ptr(el), B, T, V, beam, blank, BOS, EOS, ctypes.c_float(weight),
                                    1 if addend is not None else 0, ptr(ht), ptr(hp), n_steps, ptr(out), ctypes.byref(width),
                                    stream_ptr(dev)), "sbk_ctc_prefix_test")
    return out.cpu(), width.value


def _errors(score, ref, psi, psi_prev):
    """(max |err|, max |err| / bar, compared entries, mask of compared entries); asserts the impossible-entry pattern."""
    live = (psi_prev > -1e19).unsqueeze(-1).expand_as(ref)
    dead = ref <= -1e19
    kdead = score <= -1e19
    bad = (dead != kdead) & live
    assert not bad.any(), f"impossible-entry pattern differs at {bad.nonzero()[:5].tolist()}"
    m = live & ~dead
    err = (score - ref).abs()
    bar = ATOL + RTOL * (psi.abs() + psi_prev.abs().unsqueeze(-1))
    assert torch.isfinite(score[m]).all()
    return float(err[m].max()), float((err / bar)[m].max()), int(m.sum()), m


def _fp32_reference_error(c, logits, enc_len, ht, hp, o):
    """The reference's own fp32 error on this case: oracle.ctc_prefix_step (a restatement of CTCPrefixScore that is
    pinned to the reference at float64) run in float32, or None when its (T, 2, n_bh, V) state would not fit."""
    from oracle import asr_oracle as O
    B, T, V, beam = c["B"], c["T"], c["V"], c["beam"]
    if T * 2 * B * beam * V > 40_000_000 or c["n_steps"] * T > 20000:
        return None
    st = O.ctc_prefix_reset(torch.log_softmax(logits, -1), enc_len.long(), c["blank"], EOS)
    inp = torch.full((B * beam,), BOS, dtype=torch.long)
    mem, out = None, []
    for s in range(c["n_steps"]):
        sc, mem = O.ctc_prefix_step(st, inp, mem, beam)
        out.append(sc.double())
        if s + 1 < c["n_steps"]:
            loc = hp[s].long() - (torch.arange(B * beam) // beam) * beam
            mem = O.ctc_prefix_permute(st, mem, (loc * V + ht[s].long()).view(B, beam))
            inp = ht[s].long()
    return _errors(torch.stack(out), o["score"], o["psi"], o["psi_prev"])[:2]


def _run_case(c):
    from oracle import asr_oracle as O
    B, T, V, beam, n_steps = c["B"], c["T"], c["V"], c["beam"], c["n_steps"]
    logits = _logits(c)
    enc_len = torch.tensor(c["enc_len"], dtype=torch.int32)
    ht = torch.zeros(n_steps, B * beam, dtype=torch.int32)
    hp = torch.zeros(n_steps, B * beam, dtype=torch.int32)
    with torch.no_grad():
        o = O.ctc_prefix_scores(logits, enc_len, beam, c["blank"], BOS, EOS, ht, hp, n_steps,
                                pick=O.ctc_history_picker(B, beam, V, c["blank"], EOS, c["seed"]))
    addend = None
    if c["accumulate"]:
        addend = torch.randn(n_steps, B * beam, V, generator=torch.Generator().manual_seed(c["seed"])) * 5.0
    out, width = _hook(logits, enc_len, beam, c["blank"], c["weight"], ht, hp, n_steps, addend)
    score = out.double()
    if addend is not None:
        score = score - addend.double()
    score = score / c["weight"]
    err, margin, n, m = _errors(score, o["score"], o["psi"], o["psi_prev"])
    n_low = int((o["low"] & m).sum())
    with torch.no_grad():
        ref32 = _fp32_reference_error(c, logits, enc_len, ht, hp, o)
    r = dict(name=c["name"], R=width, bulk=V % 4 == 0, compared=n, fallback_entries=n_low, err=err, margin=margin,
             fp32_ref_err=ref32[0] if ref32 else None)
    print(json.dumps(r))
    assert n > 0
    if c["regime"] == "peaked":
        assert n_low > 0, "the peaked case no longer reaches the log-domain fallback"
    assert margin <= 1.0, r
    return r


def test_ctc_prefix_hook_vs_reference_fixture():
    """The fixture written from the reference's CTCPrefixScore (float64), through the hook."""
    gold = torch.load(os.path.join(GOLDEN, "ctc_prefix.pt"))
    for name, c in gold.items():
        out, width = _hook(c["logits"], c["enc_len"], c["beam"], c["blank"], 1.0, c["hist_tok"], c["hist_pred"], c["n_steps"])
        score = out.double()
        ref, prev = c["score"], c["psi_prev"]
        psi = ref + prev.unsqueeze(-1)
        err, margin, n, _ = _errors(score, ref, psi, prev)
        print(f"[fixture {name}] R={width} compared {n} entries: max abs err {err:.2e}, worst err / bar {margin:.3f}")
        assert margin <= 1.0


def test_ctc_prefix_hook_sweep():
    """Every compiled group width, both load paths, the fallback, blank 0 / V - 1, short T, ragged and zero enc_len, steps
    up to T, accumulated scores at weights 0.4 and 1.0."""
    results, failed = [], []
    for c in CASES:
        try:
            results.append(_run_case(c))
        except AssertionError as e:
            print(f"FAILED {c['name']}: {str(e)[:300]}")
            failed.append(c["name"])
    assert not failed, failed
    widths = {r["R"] for r in results}
    assert widths >= {16, 12, 11, 10, 8, 6, 5, 4, 3, 2, 1}, sorted(widths)
    assert any(r["bulk"] for r in results) and not all(r["bulk"] for r in results)
    assert sum(r["fallback_entries"] for r in results) > 0


LONG_SCRIPT = r"""
import json, sys
sys.path.insert(0, %r); sys.path.insert(0, %r)
import test_gpu_ctc_prefix as t
for c in t.LONG_CASES:
    t._run_case(c)
print("LONG_OK")
""" % (ROOT, os.path.join(ROOT, "tests"))


def test_ctc_prefix_hook_long_T_fresh_process():
    """T = 2458 .. 10240 (beam 66 and 128 at T = 2500, where shared memory caps the group width) as the first CTC work of
    a process."""
    p = subprocess.run([sys.executable, "-c", LONG_SCRIPT], capture_output=True, text=True, timeout=1500, cwd=ROOT)
    print(p.stdout[-4000:])
    assert p.returncode == 0 and "LONG_OK" in p.stdout, p.stdout[-2000:] + p.stderr[-3000:]


E2E_SCRIPT = r"""
import json, sys, torch
sys.path.insert(0, %r)
import bench
from oracle import asr_oracle as O
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
T, steps = int(sys.argv[1]), 4
cfg = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=1)
sd = seeded_asr_state(cfg, 0)
dev = torch.device("cuda:0")
asr = bench.build_product_asr(cfg, sd, dev, decoder="beam", beam=4, ctc=True)
bs = asr.mods["decoder"]
bs.max_decode_ratio = (steps + 0.5) / T
bs.return_topk, bs.topk = True, 4
enc = torch.randn(1, T, cfg["d_model"], generator=torch.Generator().manual_seed(T))
lens = torch.ones(1)
hyps, hlens, scores, _ = bs(enc.to(dev), lens.to(dev))
hyps, hlens, scores = hyps.cpu(), hlens.cpu(), scores.cpu()
n = int(torch.round(hlens[0, 0] * hyps.shape[2])) + 1
toks = hyps[0, 0, :n].tolist()
with torch.no_grad():
    o = O.beam_search(enc, lens, sd, dict(cfg), sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], 1, 2, beam_size=1,
                      prefix="Transformer.", ctc=dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=0.4, blank_index=0),
                      forced=[toks], temperature=1.15, using_eos_threshold=False, length_normalization=True)
print(json.dumps(dict(T=T, tokens=toks, score=float(scores[0, 0]), oracle=float(o[0]))))
""" % ROOT


@pytest.mark.parametrize("T", [3000, 6200])
def test_ctc_beam_search_long_T_fresh_process(T):
    """A CTC beam search through sbk_asr_beam_from_enc (the captured per-step graph) at T = 3000 and 6200 as the first CTC
    search of a process: it completes, and the oracle scores the best hypothesis as the search did (within 3e-2, the
    bar of the beam goldens)."""
    p = subprocess.run([sys.executable, "-c", E2E_SCRIPT, str(T)], capture_output=True, text=True, timeout=1500, cwd=ROOT)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-3000:]
    r = json.loads(p.stdout.strip().splitlines()[-1])
    print(r)
    assert len(r["tokens"]) >= 1 and math.isfinite(r["score"])
    assert abs(r["score"] - r["oracle"]) < 3e-2


def test_ctc_only_beam16_vs_oracle_search():
    """beam 16 (the widest score-kernel group, R = 16) with the CTC scorer alone on the 2 s golden, vs the oracle's own
    search, judged like the beam goldens (near-tied alternatives scored by the oracle walked along our tokens)."""
    from oracle import asr_oracle as O
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    from test_gpu_bench_shapes import _cfg, _run_beam_case
    g = torch.load(os.path.join(GOLDEN, "conformer_large_rope.pt"))
    cfg = _cfg(g)
    sd = seeded_asr_state(cfg, 0)
    kw = dict(beam_size=16, using_eos_threshold=False, temperature=1.15, min_decode_ratio=0.0)
    mdr = 0.20588235294117646
    with torch.no_grad():
        hyps, lens, scores, lp = O.beam_search(g["enc_out"], g["wav_lens"], sd, dict(g["cfg"]), sd["seq_lin.w.weight"],
                                               sd["seq_lin.w.bias"], 1, 2, prefix="Transformer.", max_decode_ratio=mdr,
                                               ctc=dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=0.4,
                                                        blank_index=0), topk=16, return_topk=True, **kw)
    gb = dict(kwargs=kw, eos_bias=0.0, max_decode_ratio=mdr, with_lm=False, with_ctc=True, hyps=hyps, lens=lens, scores=scores)
    _run_beam_case(torch.device("cuda:0"), g, gb, "ctc_beam16")
