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
