"""The float64 decode-step references of decoder_kernels_oracle.py against the CPU oracle (oracle.asr_oracle), which
make_goldens.py pins to the running reference.  A KV-cached decoder and a KV-cached TransformerLM built from proj_ref and
dec_attention_ref, one position at a time as the device steps run, must give the oracle's whole-prefix outputs at every
position; attention through a lineage table must equal attention over caches reordered the way the reference's beam search
moves its memory.  So the references are the reference's maths, not a restatement of the kernels."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import decoder_kernels_oracle as DK  # noqa: E402
from oracle import asr_oracle as O  # noqa: E402

TOL = 1e-10


def _r(g, *s, scale=1.0):
    return scale * torch.randn(*s, generator=g, dtype=torch.float64)


def _linear(sd, key, n_out, n_in, g):
    sd[key + "weight"] = _r(g, n_out, n_in, scale=1.0 / math.sqrt(n_in))
    sd[key + "bias"] = _r(g, n_out, scale=0.1)


def _norm(sd, key, d, g):
    sd[key + "weight"] = 1.0 + _r(g, d, scale=0.1)
    sd[key + "bias"] = _r(g, d, scale=0.1)


def _decoder_state(d, F_, V, n_layers, g):
    sd = {"custom_tgt_module.layers.0.emb.Embedding.weight": _r(g, V, d, scale=0.3)}
    for j in range(n_layers):
        p = f"decoder.layers.{j}."
        for n in ("norm1.norm.", "norm2.norm.", "norm3.norm."):
            _norm(sd, p + n, d, g)
        for a in ("self_attn.att.", "multihead_attn.att."):
            sd[p + a + "in_proj_weight"] = _r(g, 3 * d, d, scale=1.0 / math.sqrt(d))
            sd[p + a + "in_proj_bias"] = _r(g, 3 * d, scale=0.1)
            _linear(sd, p + a + "out_proj.", d, d, g)
        _linear(sd, p + "pos_ffn.ffn.0.", F_, d, g)
        _linear(sd, p + "pos_ffn.ffn.3.", d, F_, g)
    _norm(sd, "decoder.norm.norm.", d, g)
    return sd


def _decoder_steps(tgt, enc, enc_len, sd, cfg):
    """the KV-cached decoder of the device, position by position, from the references: [n, S, d]"""
    n, S = tgt.shape
    d, H, L = cfg["d_model"], cfg["nhead"], cfg["num_decoder_layers"]
    dh = d // H
    T = enc.shape[1]
    act = "f16_gelu" if cfg["decoder_activation"] == "gelu" else "f16_relu"
    emb = sd["custom_tgt_module.layers.0.emb.Embedding.weight"]
    pe = O.sine_pe(S, d).double()
    kc = [torch.zeros(n, S, d, dtype=torch.float64) for _ in range(L)]
    vc = [torch.zeros(n, S, d, dtype=torch.float64) for _ in range(L)]
    outs = []
    for s in range(S):
        x = emb[tgt[:, s]] * math.sqrt(d) + pe[s]
        for j in range(L):
            p = f"decoder.layers.{j}."
            w = lambda k: sd[p + k]  # noqa: E731
            wi, bi = DK.fold_query_scale(w("self_attn.att.in_proj_weight"), w("self_attn.att.in_proj_bias"), d, dh)
            q, kc[j], vc[j] = DK.proj_ref(None, wi, bi, "qkv_cache", X=x, ln_g=w("norm1.norm.weight"),
                                          ln_b=w("norm1.norm.bias"), kcache=kc[j], vcache=vc[j], step=s)
            att = DK.dec_attention_ref(q.view(n, H, dh), kc[j].view(n, S, H, dh), vc[j].view(n, S, H, dh), s + 1)
            x = DK.proj_ref(att.reshape(n, d), w("self_attn.att.out_proj.weight"), w("self_attn.att.out_proj.bias"), "resid",
                            out=x)
            wc, bc = w("multihead_attn.att.in_proj_weight"), w("multihead_attn.att.in_proj_bias")
            wq, bq = DK.fold_query_scale(wc[:d], bc[:d], d, dh)
            q = DK.proj_ref(None, wq, bq, "f16", X=x, ln_g=w("norm2.norm.weight"), ln_b=w("norm2.norm.bias"))
            kx = (enc @ wc[d:2 * d].T + bc[d:2 * d]).view(n, T, H, dh)   # the per-utterance cross K / V projection
            vx = (enc @ wc[2 * d:].T + bc[2 * d:]).view(n, T, H, dh)
            att = DK.dec_attention_ref(q.view(n, H, dh), kx, vx, enc_len)
            x = DK.proj_ref(att.reshape(n, d), w("multihead_attn.att.out_proj.weight"), w("multihead_attn.att.out_proj.bias"),
                            "resid", out=x)
            h = DK.proj_ref(None, w("pos_ffn.ffn.0.weight"), w("pos_ffn.ffn.0.bias"), act, X=x, ln_g=w("norm3.norm.weight"),
                            ln_b=w("norm3.norm.bias"))
            x = DK.proj_ref(h, w("pos_ffn.ffn.3.weight"), w("pos_ffn.ffn.3.bias"), "resid", out=x)
        outs.append(DK.layer_norm_ref(x, sd["decoder.norm.norm.weight"], sd["decoder.norm.norm.bias"]))
    return torch.stack(outs, dim=1)


@pytest.mark.parametrize("H,act", [(2, "gelu"), (4, "relu"), (4, "gelu")])
def test_decoder_step_vs_oracle(H, act):
    """d = 32, 2 layers, ragged enc_len {T, 5, 1}: the cached step's output at every position equals O.decode over the
    whole prefix."""
    d, F_, V, L, T, S, n = 32, 64, 11, 2, 9, 7, 3
    g = torch.Generator().manual_seed(H * 10 + len(act))
    cfg = dict(d_model=d, nhead=H, num_decoder_layers=L, decoder_activation=act)
    sd = _decoder_state(d, F_, V, L, g)
    enc = _r(g, n, T, d)
    enc_len = torch.tensor([T, 5, 1])
    tgt = torch.randint(0, V, (n, S), generator=g)
    tgt[:, 0] = 1
    out = _decoder_steps(tgt, enc, enc_len, sd, cfg)
    for s in range(S):
        ref, _ = O.decode(tgt[:, :s + 1], enc, enc_len, sd, cfg)
        assert torch.isfinite(ref).all()
        assert float((out[:, s] - ref[:, -1]).abs().max()) <= TOL, f"position {s}"


def _lm_state(d, F_, V, n_layers, g):
    sd = {"custom_src_module.emb.Embedding.weight": _r(g, V, d, scale=0.3)}
    for i in range(n_layers):
        p = f"encoder.layers.{i}."
        sd[p + "self_att.att.in_proj_weight"] = _r(g, 3 * d, d, scale=1.0 / math.sqrt(d))
        sd[p + "self_att.att.in_proj_bias"] = _r(g, 3 * d, scale=0.1)
        _linear(sd, p + "self_att.att.out_proj.", d, d, g)
        _norm(sd, p + "norm1.norm.", d, g)
        _norm(sd, p + "norm2.norm.", d, g)
        _linear(sd, p + "pos_ffn.ffn.0.", F_, d, g)
        _linear(sd, p + "pos_ffn.ffn.3.", d, F_, g)
    _norm(sd, "encoder.norm.norm.", d, g)
    _linear(sd, "output_proj.layers.0.w.", d, d, g)
    _norm(sd, "output_proj.layers.1.norm.", d, g)
    _linear(sd, "output_proj.layers.2.w.", V, d, g)
    return sd


def _lm_steps(tokens, sd, cfg):
    """the KV-cached TransformerLM step of the device (post-norm layers, pad mask on id 0), position by position: logits
    [n, s, V]"""
    n, S = tokens.shape
    d, H, L = cfg["d_model"], cfg["nhead"], cfg["num_encoder_layers"]
    dh = d // H
    act = "f16_gelu" if cfg["activation"] == "gelu" else "f16_relu"
    pe = O.sine_pe(S, d).double()
    kc = [torch.zeros(n, S, d, dtype=torch.float64) for _ in range(L)]
    vc = [torch.zeros(n, S, d, dtype=torch.float64) for _ in range(L)]
    ln = lambda x, k: DK.layer_norm_ref(x, sd[k + "weight"], sd[k + "bias"])  # noqa: E731
    outs = []
    for s in range(S):
        x = sd["custom_src_module.emb.Embedding.weight"][tokens[:, s]] * math.sqrt(d) + pe[s]
        for i in range(L):
            p = f"encoder.layers.{i}."
            w = lambda k: sd[p + k]  # noqa: E731
            wi, bi = DK.fold_query_scale(w("self_att.att.in_proj_weight"), w("self_att.att.in_proj_bias"), d, dh)
            q, kc[i], vc[i] = DK.proj_ref(x, wi, bi, "qkv_cache", kcache=kc[i], vcache=vc[i], step=s)
            att = DK.dec_attention_ref(q.view(n, H, dh), kc[i].view(n, S, H, dh), vc[i].view(n, S, H, dh), s + 1,
                                       tok=tokens, pad_tok=0)
            x = ln(DK.proj_ref(att.reshape(n, d), w("self_att.att.out_proj.weight"), w("self_att.att.out_proj.bias"), "resid",
                               out=x), p + "norm1.norm.")
            h = DK.proj_ref(x, w("pos_ffn.ffn.0.weight"), w("pos_ffn.ffn.0.bias"), act)
            x = ln(DK.proj_ref(h, w("pos_ffn.ffn.3.weight"), w("pos_ffn.ffn.3.bias"), "resid", out=x), p + "norm2.norm.")
        x = ln(x, "encoder.norm.norm.")
        x = ln(DK.proj_ref(x, sd["output_proj.layers.0.w.weight"], sd["output_proj.layers.0.w.bias"], "f32"),
               "output_proj.layers.1.norm.")
        outs.append(DK.proj_ref(x, sd["output_proj.layers.2.w.weight"], sd["output_proj.layers.2.w.bias"], "f32"))
    return torch.stack(outs, dim=1)


@pytest.mark.parametrize("n_layers,act", [(1, "gelu"), (2, "relu")])
def test_lm_self_attention_vs_oracle(n_layers, act):
    """tokens with pad id 0 inside the prefix (positions 2, 4 and 5 of row 0, 1 of row 1) and at the end (row 2): the
    cached LM step's logits at every position equal O.transformer_lm_forward over the whole prefix."""
    d, F_, V, H, S = 32, 64, 13, 4, 8
    g = torch.Generator().manual_seed(n_layers * 7 + len(act))
    cfg = dict(d_model=d, nhead=H, num_encoder_layers=n_layers, activation=act)
    sd = _lm_state(d, F_, V, n_layers, g)
    tokens = torch.randint(1, V, (3, S), generator=g)
    tokens[0, [2, 4, 5]] = 0
    tokens[1, 1] = 0
    tokens[2, 6:] = 0
    out = _lm_steps(tokens, sd, cfg)
    for s in range(S):
        ref = O.transformer_lm_forward(tokens[:, :s + 1], sd, cfg)
        assert torch.isfinite(ref).all()
        assert float((out[:, s] - ref[:, -1]).abs().max()) <= TOL, f"position {s}"


@pytest.mark.parametrize("with_tokens", [False, True])
@pytest.mark.parametrize("R", [2, 5])
def test_lineage_vs_reordered_caches(R, with_tokens):
    """Self-attention through lineage_from_history's table over the physical caches (row r writes position s at row r)
    equals attention over caches that are physically reordered by index_select along the same predecessor history after
    every step, as the reference's beam search moves its memory (and its token memory, for the LM's pad mask)."""
    H, dh, S = 2, 8, 9
    g = torch.Generator().manual_seed(R * 3 + with_tokens)
    kp, vp = _r(g, R, S, H, dh), _r(g, R, S, H, dh)
    tp = torch.randint(0, 3, (R, S), generator=g)     # physical token cache: id 0 (pad) about a third of the time
    tp[:, 0] = 1
    hist = torch.randint(0, R, (S - 1, R), generator=g)
    k_log, v_log, t_log = kp[:, :1].clone(), vp[:, :1].clone(), tp[:, :1].clone()
    for s in range(S - 1):
        q = _r(g, R, H, dh)
        lin = DK.lineage_from_history(hist[:s], S)[s & 1]
        tok = tp if with_tokens else None
        got = DK.dec_attention_ref(q, kp, vp, s + 1, lineage=lin, tok=tok)
        ref = DK.dec_attention_ref(q, k_log, v_log, s + 1, tok=t_log if with_tokens else None)
        assert float((got - ref).abs().max()) <= TOL, f"step {s}"
        # the reference's beam step: reorder by predecessor, then the next step appends its own K / V / token
        k_log = torch.cat([k_log[hist[s]], kp[:, s + 1:s + 2]], dim=1)
        v_log = torch.cat([v_log[hist[s]], vp[:, s + 1:s + 2]], dim=1)
        t_log = torch.cat([t_log[hist[s]], tp[:, s + 1:s + 2]], dim=1)


def test_zero_length_utterance_oracle():
    """An utterance with no encoder frame: the reference's cross-attention masks every key, nn.MultiheadAttention gives NaN,
    and the decoder output of that utterance is NaN at every position while the others stay finite.  Greedy search then
    takes torch's arg-max of a NaN row, its first index: token 0 at every step, with NaN scores."""
    d, F_, V, L, T, S = 32, 64, 11, 2, 6, 4
    g = torch.Generator().manual_seed(5)
    cfg = dict(d_model=d, nhead=4, num_decoder_layers=L, decoder_activation="gelu")
    sd = _decoder_state(d, F_, V, L, g)
    enc = _r(g, 3, T, d)
    tgt = torch.randint(3, V, (3, S), generator=g)
    tgt[:, 0] = 1
    enc_len = torch.tensor([T, 0, 4])
    ref, _ = O.decode(tgt, enc, enc_len, sd, cfg)
    assert torch.isnan(ref[1]).all() and torch.isfinite(ref[[0, 2]]).all()
    out = _decoder_steps(tgt, enc, enc_len, sd, cfg)
    assert torch.isnan(out[1]).all() and float((out[[0, 2]] - ref[[0, 2]]).abs().max()) <= TOL
    seq_w, seq_b = _r(g, V, d, scale=1.0 / math.sqrt(d)), _r(g, V, scale=0.1)
    hyps, _, scores, _ = O.greedy_search(enc, torch.tensor([1.0, 0.0, 0.6]), sd, cfg, seq_w, seq_b, 1, 2)
    assert hyps[1] == [0] * T and torch.isnan(scores[1, 0]).all()
    assert torch.isfinite(scores[0, 0]).all() and torch.isfinite(scores[2, 0]).all()


# ------------------------------------------------------------------------------------------------ beam step
@pytest.fixture(scope="module")
def small_model():
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state
    cfg = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=2)
    return cfg, seeded_asr_state(cfg, 0)


def _beam_by_steps(enc, wav_len, sd, cfg, beam, max_steps, ctc=None, length_weight=0.0, coverage=None):
    """oracle.asr_oracle.beam_search's loop with every step's selection and bookkeeping from DK.beam_step_ref (and the
    coverage from DK.coverage_ref): -> (history [(tok, pred, score, lp)], smallest gap between the beam-th and the
    (beam + 1)-th candidate of any utterance and step, relative to the scores' scale)"""
    B, T, _ = enc.shape
    V, n_bh = sd["seq_lin.w.weight"].shape[0], B * beam
    enc_lens = torch.round(T * wav_len).int()
    enc_r, enc_l = enc.repeat_interleave(beam, dim=0), enc_lens.repeat_interleave(beam, dim=0)
    seq = torch.full((n_bh,), float("-inf"), dtype=torch.float64)
    seq[::beam] = 0.0
    memory = torch.full((n_bh, 1), 1, dtype=torch.long)
    finished = torch.zeros(B, dtype=torch.long)
    cov = torch.zeros(n_bh, T, dtype=torch.float64)
    kw = {}
    if ctc is not None:
        kw = dict(ctc_weight=ctc["weight"], blank=ctc["blank_index"])
        st = O.ctc_prefix_reset(torch.log_softmax(enc @ ctc["w"].T + ctc["b"], dim=-1), enc_lens, ctc["blank_index"], 2)
        mem = None
    hist, gap = [], float("inf")
    for step in range(max_steps):
        if bool((finished == beam).all()):
            break
        pred_out, attn = O.decode(memory, enc_r, enc_l, sd, cfg, "Transformer.")
        logits = pred_out[:, -1] @ sd["seq_lin.w.weight"].T + sd["seq_lin.w.bias"]
        add = add_row = None
        if ctc is not None:
            score, mem = O.ctc_prefix_step(st, memory[:, -1], mem, beam)
            add = ctc["weight"] * score
        if coverage is not None:
            c, add_row = DK.coverage_ref(attn[:, -1], cov, step, coverage["threshold"], coverage["weight"])
        r = DK.beam_step_ref(logits, seq, step, beam, 2, using_eos_threshold=True, eos_threshold=1.5, add_scores=add,
                             add_row=add_row, length_weight=length_weight, finished=finished, **kw)
        flat = r["sc"].view(B, -1)
        top = flat.topk(beam + 1, dim=-1).values
        scale = top[:, 0].abs().clamp_min(1.0)
        gap = min(gap, float(((top[:, beam - 1] - top[:, beam]) / scale).min()))
        if ctc is not None:
            mem = O.ctc_prefix_permute(st, mem, ((r["pred"] % beam) * V + r["tok"]).view(B, beam))
        if coverage is not None:
            cov = c[r["pred"]]
        memory = torch.cat([memory[r["pred"]], r["tok"].view(n_bh, 1)], dim=1)
        seq, finished = r["seq"], r["finished"]
        hist.append((r["tok"], r["pred"], r["score"], r["lp"]))
    return hist, gap


BEAM_SCORERS = ["none", "ctc", "length", "coverage"]
SEED_SHIFT = {(20, "ctc"): 300}   # the first seed of this case has a near-tie at the beam boundary


@pytest.mark.parametrize("scorer", BEAM_SCORERS)
@pytest.mark.parametrize("beam", [4, 20])
def test_beam_step_vs_oracle(small_model, beam, scorer):
    """Conformer-L with 2 decoder layers (seeded), 2 utterances of 12 and 7 frames, 6 steps: DK.beam_step_ref driven one
    step at a time reproduces O.beam_search's history, tokens and predecessors exactly and scores and log-probs within fp32
    rounding (the oracle runs in fp32), on a case whose beam boundary has no near-tie."""
    cfg, sd = small_model
    g = torch.Generator().manual_seed(beam * 7 + len(scorer) + SEED_SHIFT.get((beam, scorer), 0))
    enc = torch.randn(2, 12, cfg["d_model"], generator=g)
    wl = torch.tensor([1.0, 0.6])
    steps = 6
    ctc = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=0.4, blank_index=0) if scorer == "ctc" else None
    cov = dict(weight=0.5, threshold=0.3) if scorer == "coverage" else None
    lw = 0.7 if scorer == "length" else 0.0
    with torch.no_grad():
        *_, ref = O.beam_search(enc, wl, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], 1, 2, beam, 0.0,
                                (steps + 0.5) / 12, prefix="Transformer.", return_history=True, ctc=ctc, length_weight=lw,
                                coverage=cov)
        got, gap = _beam_by_steps(enc, wl, sd, cfg, beam, steps, ctc=ctc, length_weight=lw, coverage=cov)
    assert gap > 1e-5, f"near-tie at the beam boundary ({gap:.2e}): the case would pin fp32 noise"
    assert len(got) == len(ref) and len(ref) >= 1
    for s, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a[0], b[0].long()) and torch.equal(a[1], b[1].long()), f"step {s}"
        for x, y, what in ((a[2], b[2], "score"), (a[3], b[3], "lp")):
            fin = torch.isfinite(y)
            assert torch.equal(fin, torch.isfinite(x)), f"step {s} {what}"
            err = float(((x[fin] - y[fin].double()).abs() / y[fin].double().abs().clamp_min(1.0)).max()) if fin.any() else 0.0
            assert err <= 2e-5, f"step {s} {what}: {err:.2e}"


def test_beam_step_ref_order():
    """candidate_order: NaN (either sign) first, lowest index first among NaN, among equal scores and among -inf"""
    nan, inf = float("nan"), float("inf")
    neg_nan = -torch.tensor(nan)
    sc = torch.tensor([[1.0, nan, 2.0, float(neg_nan), 2.0, -inf, inf, -inf]], dtype=torch.float64)
    assert DK.candidate_order(sc)[0].tolist() == [1, 3, 6, 2, 4, 0, 5, 7]
    r = DK.beam_step_ref(torch.full((2, 5), -inf), torch.tensor([0.0, -inf]), 0, 2, 2)   # every log-prob NaN
    assert r["tok"].tolist() == [0, 1] and r["pred"].tolist() == [0, 0] and torch.isnan(r["score"]).all()
    lg = torch.tensor([[0.0, 0.0, -inf, -inf], [0.0, 0.0, 0.0, 0.0]])
    r = DK.beam_step_ref(lg, torch.tensor([0.0, -inf]), 0, 2, 3, length_normalization=False, minus_inf=-inf)
    assert r["tok"].tolist() == [0, 1]
    r = DK.beam_step_ref(lg, torch.tensor([-inf, -inf]), 3, 2, 3, finished=torch.tensor([1]))   # only -inf candidates
    assert r["tok"].tolist() == [0, 1] and r["pred"].tolist() == [0, 0] and r["finished"].tolist() == [1]


def test_coverage_ref_empty_row():
    """a row with no visible key: NaN coverage and score; others finite; coverage accumulates over the predecessor's"""
    g = torch.Generator().manual_seed(3)
    q, K = torch.randn(4, 2, 8, generator=g), torch.randn(2, 5, 2, 8, generator=g)
    att = DK.cross_attention_probs(q, K, torch.tensor([5, 0]), 2)
    assert torch.isnan(att[2:]).all() and torch.allclose(att[:2].sum(-1), torch.ones(2, dtype=torch.float64))
    cov, s = DK.coverage_ref(att, torch.zeros(4, 5), 0, 0.5, 1.0)
    assert torch.isnan(s[2:]).all() and torch.isfinite(s[:2]).all()
    cov2, s2 = DK.coverage_ref(att, cov[[1, 0, 3, 2]], 1, 0.5, 1.0)
    assert torch.allclose(cov2[0], att[0] + att[1]) and torch.isnan(s2[2:]).all()
