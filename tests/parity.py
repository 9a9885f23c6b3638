"""The comparison rules the parity tests judge the device against a reference with, written once.

Test modules import from here the way they import the oracles (tests/ on sys.path); a GPU test module imports the `dev`
fixture into its globals (``from parity import dev  # noqa: F401``), where pytest finds it.

Bars shared by every model:
- greedy search: tokens identical up to the first decision whose reference top-1/top-2 margin is below GREEDY_MARGIN
  (fp16 operands move logits by ~1e-3), chosen log-probs within GREEDY_LOGPROB;
- beam search: best score and every n-best rank within BEAM_TOL; a best hypothesis other than the reference's must
  score, by the oracle walked along our tokens, within BEAM_TOL of ours and no worse than the reference's best - BEAM_TOL;
- CTC arg-max: log-probs within GREEDY_LOGPROB, the arg-max equal wherever the reference's margin is GREEDY_MARGIN or more.
"""
import os

import pytest
import torch

from oracle.goldens import rel, seeded_wav  # noqa: F401  (the writers' waveform rule and rel-L2, re-exported)

GREEDY_MARGIN = 5e-3
GREEDY_LOGPROB = 2e-2
BEAM_TOL = 3e-2


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def case_wav(case):
    """seeded_wav of a fixture case: its wav_seed and wav_shape, and its wav_lens and wav_checksum where it stores them"""
    return seeded_wav(case["wav_seed"], case["wav_shape"], case.get("wav_lens"), case.get("wav_checksum"))


def check_summary(tag, x, norms, idx, rows, bar):
    """x [B, T, d] against a fixture's summary of the reference's: every row's L2 norm and the sampled rows x[idx[:, 0],
    idx[:, 1]], each within rel-L2 bar; returns both errors"""
    idx = idx.long()
    e_norm = rel(x.double().norm(dim=-1), norms)
    e_rows = rel(x[idx[:, 0], idx[:, 1]], rows)
    print(f"MEASURE {tag} vs reference summary: row norms rel-L2 {e_norm:.3e}, sampled rows {e_rows:.3e} (bar {bar})")
    assert e_norm < bar and e_rows < bar, tag
    return e_norm, e_rows


def check_encoder(tag, enc, ref, abs_len, bar):
    """encoder states [B, T, d]: finite, rel-L2 below bar over all frames and over each utterance's abs_len[b] valid frames"""
    r_all = rel(enc, ref)
    per = [rel(enc[b, :int(abs_len[b])], ref[b, :int(abs_len[b])]) for b in range(enc.shape[0])]
    print(f"[{tag}] encoder rel-L2 {r_all:.3e} (valid frames per utterance {['%.3e' % x for x in per]}) "
          f"max abs {(enc - ref).abs().max():.3e} (bar {bar})")
    assert torch.isfinite(enc).all() and r_all < bar and max(per) < bar


def check_greedy(tag, pred, score, tokens, margin, chosen_lp=None, stop_at=None, min_compared=None):
    """Greedy tokens pred [B, S] against the reference's tokens [B, S'] (S' <= S compared): identical up to the first
    decision whose reference margin is below GREEDY_MARGIN; up to there, |score - chosen_lp| within GREEDY_LOGPROB
    (both [B, S] chosen log-probs, or [B, S, V] whole distributions: the largest difference counts).  stop_at: a row
    stops after the reference emits this token; min_compared: the fraction of the B S' decisions that must be compared.
    Returns the number of decisions compared."""
    B, S = tokens.shape
    compared, worst, stops = 0, 0.0, []
    for b in range(B):
        for s in range(S):
            if int(pred[b, s]) != int(tokens[b, s]):
                assert float(margin[b, s]) < GREEDY_MARGIN, \
                    f"[{tag}] token mismatch at b={b} s={s}, reference margin {float(margin[b, s]):.4f}"
                stops.append((b, s))
                break
            if chosen_lp is not None:
                d = float((score[b, s].double() - chosen_lp[b, s].double()).abs().max())
                worst = max(worst, d)
                assert d < GREEDY_LOGPROB, f"[{tag}] log-prob err {d} at b={b} s={s}"
            compared += 1
            if stop_at is not None and int(tokens[b, s]) == stop_at:
                break
    print(f"[{tag}] greedy: {compared}/{B * S} decisions compared identical, max log-prob err {worst:.2e}, "
          f"near-tie stops {stops}")
    if min_compared is not None:
        assert compared >= min_compared * B * S, "too few decisions comparable"
    return compared


def check_beam(tag, hyps, scores, ref_hyps, ref_scores, rescore_forced):
    """Beam search against the reference: hyps / ref_hyps are best hypotheses as token lists, scores / ref_scores [B, k]
    n-best scores (rank 0 the best).  rescore_forced(indices, token_lists) returns the oracle's scores of those utterances
    walked along those tokens."""
    scores, ref_scores = scores.cpu(), ref_scores.cpu()
    B, diverged = len(hyps), []
    for b in range(B):
        assert abs(float(scores[b, 0]) - float(ref_scores[b, 0])) < BEAM_TOL, \
            f"[{tag}] best score {float(scores[b, 0])} vs reference {float(ref_scores[b, 0])}"
        if list(hyps[b]) != list(ref_hyps[b]):
            diverged.append((b, list(hyps[b])))
    k = min(scores.shape[1], ref_scores.shape[1])
    nbest_err = (scores[:, :k] - ref_scores[:, :k]).abs().max().item()
    print(f"[{tag}] beam: best scores {scores[:, 0].tolist()} ref {ref_scores[:, 0].tolist()}; identical best hypothesis for "
          f"{B - len(diverged)}/{B}; max |n-best score - reference| over {k} ranks {nbest_err:.2e}")
    assert nbest_err < BEAM_TOL
    if diverged:
        o = rescore_forced([b for b, _ in diverged], [t for _, t in diverged])
        for (b, toks), osc in zip(diverged, [float(x) for x in o]):
            print(f"   utterance {b}: our hypothesis ({len(toks)} tokens) scores {float(scores[b, 0]):.5f}, the oracle gives it "
                  f"{osc:.5f}; reference best {float(ref_scores[b, 0]):.5f}")
            assert abs(osc - float(scores[b, 0])) < BEAM_TOL, "our score for our own hypothesis is off"
            assert osc > float(ref_scores[b, 0]) - BEAM_TOL, "the search returned a clearly worse hypothesis than the reference"


def best_tokens(hyps, lens):
    """each utterance's best hypothesis, as a token list with its EOS, of a padded n-best [B, k, L] with relative lengths
    [B, k]"""
    hyps, lens = hyps.cpu(), lens.cpu()
    return [hyps[b, 0, :int(torch.round(lens[b, 0] * hyps.shape[2])) + 1].tolist() for b in range(hyps.shape[0])]


def check_alone_vs_batch(encode, wav, lens, bar, relative=False):
    """encode(wav, lens) -> encoder states, or a tuple of outputs with the states first: a rerun is bit-identical, and
    utterance 0 (relative length 1.0, so the same T) alone equals its rows in the padded batch within bar, as max |d| or,
    relative, as max |d| / max |x|"""
    def run(w, ln):
        out = encode(w, ln)
        return tuple(t.cpu() for t in out) if isinstance(out, tuple) else (out.cpu(),)
    batch = run(wav, lens)
    assert all(torch.equal(x, y) for x, y in zip(batch, run(wav, lens))), "rerun differs"
    alone = run(wav[:1].contiguous(), lens[:1].contiguous())[0]
    d = float((alone[0] - batch[0][0]).abs().max())
    if relative:
        d /= float(batch[0][0].abs().max())
    print(f"utterance 0 alone vs in the batch: max |d|{' / max |x|' if relative else ''} {d:.2e}")
    assert d <= bar


def check_ctc_argmax(tag, lp, ref_lp, ref_argmax, margin, lens, blank, ref_hyps):
    """EncoderASR CTC log-posteriors lp [B, T, V] against the reference's: the stored ref_lp [B, T, V' <= V] within
    GREEDY_LOGPROB, the per-frame arg-max equal to the reference's on valid frames whose margin is GREEDY_MARGIN or more,
    and greedy decoding of our arg-max, with the near-tie frames taken from the reference, equal to ref_hyps"""
    from speechbrain_b200.decoders.ctc import greedy_from_argmax
    e = float((lp[..., :ref_lp.shape[-1]] - ref_lp).abs().max())
    am = lp.argmax(-1)
    T = lp.shape[1]
    bad = 0
    for b in range(lp.shape[0]):
        n = int(torch.round(lens[b] * T))
        strong = margin[b, :n] >= GREEDY_MARGIN
        bad += int((am[b, :n][strong] != ref_argmax[b, :n].long()[strong]).sum())
    patched = torch.where(margin >= GREEDY_MARGIN, am, ref_argmax.long())
    print(f"[{tag}] CTC log-prob max err {e:.2e}; strong-margin frames with another arg-max: {bad}")
    assert e < GREEDY_LOGPROB and bad == 0 and greedy_from_argmax(patched, lens, blank) == ref_hyps


def module_list_ckpt(sd):
    """A seeded ASR state as the recipes' asr.ckpt: the keys of torch.nn.ModuleList([CNN, Transformer, seq_lin, ctc_lin])"""
    prefix = {"CNN.": "0.", "Transformer.": "1.", "seq_lin.": "2.", "ctc_lin.": "3."}
    return {q + k[len(p):]: v for k, v in sd.items() for p, q in prefix.items() if k.startswith(p)}


def normalizer_ckpt(sd):
    return {"count": 1, "glob_mean": sd["normalize.glob_mean"], "glob_std": sd["normalize.glob_std"]}


def write_pretrained_dir(path, yaml, ckpts):
    """A pretrained-model directory for from_hparams: <name>.ckpt for each entry of ckpts, and hyperparams.yaml with
    <save_dir> replaced by path"""
    path = str(path)
    for name, state in ckpts.items():
        torch.save(state, os.path.join(path, name + ".ckpt"))
    with open(os.path.join(path, "hyperparams.yaml"), "w") as f:
        f.write(yaml.replace("<save_dir>", path))
    return path


def lm_scorer(vocab=5000):
    """The recipes' 12-layer, 768-wide TransformerLM with seeded weights (seed 1): the scorer of the beam-search tests"""
    from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    lm = TransformerLM(vocab=vocab, d_model=768, nhead=12, num_encoder_layers=12, num_decoder_layers=0, d_ffn=3072,
                       dropout=0.0, activation=torch.nn.GELU, normalize_before=False)
    lm.load_state_dict(seeded_state_dict(lm, seed=1))
    return lm


def lm_scorer_state(vocab=5000):
    return lm_scorer(vocab).state_dict()


def oracle_lm(weight, temperature, vocab=5000):
    """the oracle's lm= argument for lm_scorer(vocab) at this weight and temperature"""
    return dict(sd=lm_scorer_state(vocab), cfg=dict(d_model=768, nhead=12, num_encoder_layers=12, d_ffn=3072, activation="gelu"),
                weight=weight, temperature=temperature)
