"""float64 references of the decode-step kernels that the device hooks expose alone:

- proj_ref: one step Linear (sbk_step_proj_test) on either back end, the weight-streaming skinny_gemm_kernel (with the
  decoder pre-norm fused into it or not) and the wgmma gemm_f16_small, with every step epilogue;
- dec_attention_ref: dec_attention_kernel<64 / 128> and dec_attention_generic_kernel (sbk_dec_attention_test), the
  self-attention over the KV cache with a beam lineage table and the TransformerLM's pad-token mask, and the
  cross-attention over the encoder states;
- lineage_from_history: the [2][rows][S_max] cache-row table that beam_reset and beam_step leave after a search history;
- beam_step_ref: one beam-search step (sbk_beam_step_test) with every output of the kernels, in the candidate order both
  selection paths follow (candidate_order: NaN first, score descending, lowest index first);
- cross_attention_probs and coverage_ref: the CoverageScorer step (sbk_coverage_score_test).

They take the inputs the kernels receive (fp16 activations and weights, fp32 LayerNorm inputs and biases) in float64 and
work on whatever device those tensors are on.  test_decoder_kernels_oracle.py pins them to oracle.asr_oracle.decode,
greedy_search and transformer_lm_forward (which make_goldens.py pins to the running reference) to 1e-10, and
beam_step_ref / coverage_ref to beam_search within its fp32 rounding."""
import math

import torch
import torch.nn.functional as F

FP16_MAX = 65504.0
EPILOGUES = ("f16", "f16_gelu", "f16_relu", "f32", "resid", "qkv_cache")   # the hook's epilogue codes, in order


def layer_norm_ref(x, gamma, beta, eps=1e-6):
    """the decoder pre-norm: LayerNorm over the last dim in float64"""
    return F.layer_norm(x.double(), (x.shape[-1],), gamma.double(), beta.double(), eps)


def proj_ref(A, W, bias, epilogue, out=None, X=None, ln_g=None, ln_b=None, kcache=None, vcache=None, step=0):
    """y = A W^T + bias in float64, A [rows, K] (or A = LayerNorm(X; ln_g, ln_b, eps 1e-6) when X is given), W [N, K].

    epilogue 'f16' / 'f16_gelu' (exact erf) / 'f16_relu': y (activated) clamped to +-65504, the saturating fp16 store;
    'f32': y; 'resid': out + y; 'qkv_cache': y = [q | k | v] of width N / 3: returns (q clamped, kcache, vcache) with row r
    of k / v written at position `step` of the caches [rows, S_max, N / 3] (copies in float64; every other entry kept)."""
    a = layer_norm_ref(X, ln_g, ln_b) if X is not None else A.double()
    y = a @ W.double().T
    if bias is not None:
        y = y + bias.double()
    sat = lambda t: t.clamp(-FP16_MAX, FP16_MAX)  # noqa: E731
    if epilogue == "f16":
        return sat(y)
    if epilogue == "f16_gelu":
        return sat(F.gelu(y))
    if epilogue == "f16_relu":
        return sat(F.relu(y))
    if epilogue == "f32":
        return y
    if epilogue == "resid":
        return out.double() + y
    if epilogue == "qkv_cache":
        d = y.shape[-1] // 3
        kc, vc = kcache.double().clone(), vcache.double().clone()
        kc[:, step], vc[:, step] = sat(y[:, d:2 * d]), sat(y[:, 2 * d:])
        return sat(y[:, :d]), kc, vc
    raise ValueError(epilogue)


def dec_attention_ref(q, k, v, n_keys, rows_per_block=1, lineage=None, tok=None, pad_tok=0):
    """One query per row: q [R, H, dh] (the 1/sqrt(dh) scale already folded in), keys / values k, v [blocks, S, H, dh] ->
    [R, H, dh] float64.

    Row r attends to keys j < n (n = n_keys, or n_keys[b] per block b = r // rows_per_block: enc_len), read from block b, or
    with a lineage table [R, >= n] from block lineage[r, j] (the cache row of the ancestor that wrote position j).  With
    tok [blocks, S]: key j is masked when the token of the block it is read from, tok[src, j], is pad_tok
    (TransformerLM.make_masks).  A row with no visible key is NaN, as nn.MultiheadAttention gives it."""
    R, H, dh = q.shape
    q, k, v = q.double(), k.double(), v.double()
    out = torch.empty(R, H, dh, dtype=torch.float64, device=q.device)
    for r in range(R):
        blk = r // rows_per_block
        n = int(n_keys) if not torch.is_tensor(n_keys) else int(n_keys[blk])
        if n == 0:
            out[r] = float("nan")
            continue
        j = torch.arange(n, device=q.device)
        src = lineage[r, :n].to(q.device).long() if lineage is not None else torch.full_like(j, blk)
        s = torch.einsum("hd,nhd->hn", q[r], k[src, j])
        if tok is not None:
            s = s.masked_fill((tok.to(q.device)[src, j] == pad_tok).view(1, n), float("-inf"))
        out[r] = torch.einsum("hn,nhd->hd", torch.softmax(s, dim=-1), v[src, j])
    return out


def lineage_from_history(hist_pred, S_max):
    """[2][R][S_max] int64 cache-row table after len(hist_pred) beam steps, hist_pred [n_steps, R] the predecessor row of
    every new hypothesis.  beam_reset: position 0 of row r lives in row r (table 0).  Step s (beam_step_kernel) fills table
    (s + 1) % 2 from table s % 2: positions p < s come from the predecessor's entries, position s from the predecessor itself
    (its K/V were written there), position s + 1 from the row itself (the next step writes there).  The self-attention of
    step s reads table s % 2."""
    n_steps, R = hist_pred.shape
    lin = torch.zeros(2, R, S_max, dtype=torch.long)
    lin[0, :, 0] = torch.arange(R)
    for s in range(n_steps):
        lin_in, lin_out = lin[s & 1], lin[(s + 1) & 1]
        pred = hist_pred[s].long()
        lin_out[:, :s] = lin_in[pred, :s]
        lin_out[:, s] = pred
        lin_out[:, s + 1] = torch.arange(R)
    return lin


def candidate_order(sc):
    """sc [B, n] -> the candidates of each row in the beam step's order: NaN first whatever its sign, then score descending,
    then the lowest index first (torch.topk leaves the order among equal scores unspecified)."""
    nan = torch.isnan(sc)
    order = torch.sort(sc.masked_fill(nan, float("inf")), dim=-1, descending=True, stable=True).indices
    return order.gather(-1, torch.sort(nan.gather(-1, order).to(torch.int8), dim=-1, descending=True, stable=True).indices)


def beam_step_ref(logits, seq, step, beam, eos, min_steps=0, temperature=1.0, using_eos_threshold=False, eos_threshold=1.5,
                  length_normalization=True, minus_inf=-1e20, ctc_weight=0.0, blank=-1, add_scores=None, add_row=None,
                  length_weight=0.0, finished=None, lineage=None, emb=None, pe=None, lm_emb=None, lm_pe=None):
    """One iteration of oracle.asr_oracle.beam_search (S2SBeamSearcher.search_step) in float64, the scorers' scores
    precomputed: logits [n_bh, V] of the hypotheses, seq [n_bh] their sequence scores, every row at `step`.  In order: the
    decoder weight 1 - ctc_weight, the log-probs kept for the history, eos -> minus_inf while step < min_steps, the eos
    threshold, the CTC blank -> minus_inf, + add_scores [n_bh, V] + add_row [n_bh] + length_weight, / (step + 1) under length
    normalisation, then the first `beam` of each utterance's beam * V candidates in candidate_order.

    Returns a dict: the full scores 'sc' [n_bh, V], the history row 'tok', 'pred' (global row), 'score', 'lp', the next
    sequence scores 'seq' (-inf after eos), and with the matching arguments 'finished' [B] (capped at beam) and
    'n_full' (utterances whose counter reaches beam at this step), 'lineage' (the next parity's [n_bh, S] table from this
    parity's `lineage`, as lineage_from_history builds it), 'x' = emb[tok] * sqrt(d) + pe[step + 1], and for the LM 'lm_x',
    'lm_x16' (fp16 saturation) and 'tok_cache' (the token written at position step + 1)."""
    n_bh, V = logits.shape
    B = n_bh // beam
    lp = torch.log_softmax(logits.double() / temperature, dim=-1)
    if ctc_weight != 0.0:
        lp = (1.0 - ctc_weight) * lp
    hist_lp = lp.clone()
    if step < min_steps:
        lp[:, eos] = minus_inf
    if using_eos_threshold:
        cond = lp[:, eos] > eos_threshold * lp.max(dim=-1).values
        lp[:, eos] = torch.where(cond, lp[:, eos], torch.full_like(lp[:, eos], minus_inf))
    if ctc_weight != 0.0:
        lp[:, blank] = minus_inf
    if add_scores is not None:
        lp = lp + add_scores.double()
    if add_row is not None:
        lp = lp + add_row.double().view(n_bh, 1)
    lp = lp + length_weight
    sc = seq.double().view(n_bh, 1) + lp
    if length_normalization:
        sc = sc / (step + 1)
    flat = sc.view(B, beam * V)
    cand = candidate_order(flat)[:, :beam]
    score = flat.gather(1, cand).reshape(n_bh)
    tok = (cand % V).reshape(n_bh)
    pred = (cand // V + (torch.arange(B, device=cand.device) * beam).view(B, 1)).reshape(n_bh)
    out = {"sc": sc, "tok": tok, "pred": pred, "score": score, "lp": hist_lp[pred, tok]}
    nxt = score * (step + 1) if length_normalization else score.clone()
    out["seq"] = nxt.masked_fill(tok == eos, float("-inf"))
    if finished is not None:
        before = finished.long().cpu()
        after = torch.clamp(before + (tok.cpu() == eos).view(B, beam).sum(1), max=beam)
        out["finished"], out["n_full"] = after, int(((before < beam) & (after >= beam)).sum())
    if lineage is not None:
        lin = lineage.long().cpu().clone()
        p = pred.cpu()
        lin[:, :step] = lineage.long().cpu()[p, :step]
        lin[:, step] = p
        lin[:, step + 1] = torch.arange(n_bh)
        out["lineage"] = lin
    t = tok.cpu()
    if emb is not None:
        out["x"] = emb.double().cpu()[t] * math.sqrt(emb.shape[1]) + pe.double().cpu()[step + 1]
    if lm_emb is not None:
        out["lm_x"] = lm_emb.double().cpu()[t] * math.sqrt(lm_emb.shape[1]) + lm_pe.double().cpu()[step + 1]
        out["lm_x16"] = out["lm_x"].clamp(-FP16_MAX, FP16_MAX)
        out["tok_cache"] = t
    return out


def cross_attention_probs(q, K, enc_len, rows_per_utt):
    """the head-averaged cross-attention distribution of one query per row: q [R, H, dh] (scale folded in), keys K [U, T, H,
    dh], row r reads utterance r // rows_per_utt and its first enc_len[u] frames -> [R, T] float64, 0 past enc_len, NaN for a
    row with no visible key (nn.MultiheadAttention's attention weights, averaged over heads)."""
    R, H, dh = q.shape
    T = K.shape[1]
    out = torch.zeros(R, T, dtype=torch.float64)
    q, K = q.double().cpu(), K.double().cpu()
    for r in range(R):
        u = r // rows_per_utt
        n = int(enc_len[u])
        if n == 0:
            out[r] = float("nan")
            continue
        s = torch.einsum("hd,thd->ht", q[r], K[u, :n])
        out[r, :n] = torch.softmax(s, dim=-1).mean(0)
    return out


def coverage_ref(att, cov_prev, step, threshold, weight):
    """CoverageScorer.score (scorer.py:880-922) one step at a time: the coverage of a hypothesis is this step's head-averaged
    attention att [R, T] plus its predecessor's coverage cov_prev [R, T] (already gathered; zeros at step 0) -> (coverage,
    weight * -(sum_t max(coverage_t, threshold) - T * threshold) / (step + 1)).  NaN attention stays NaN (torch.maximum)."""
    cov = att.double() + cov_prev.double()
    T = cov.shape[-1]
    pen = torch.maximum(cov, torch.full_like(cov, threshold)).sum(-1) - T * threshold
    return cov, weight * (-pen / (step + 1))


def fold_query_scale(w, b, d, dh):
    """the packed weights' query scale: rows [0, d) of a q (or [q | k | v]) projection times 1 / sqrt(dh)"""
    w, b = w.clone(), b.clone()
    w[:d] *= 1.0 / math.sqrt(dh)
    b[:d] *= 1.0 / math.sqrt(dh)
    return w, b
