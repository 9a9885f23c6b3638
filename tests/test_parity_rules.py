"""The shared comparison rules of parity.py on small synthetic inputs, no GPU needed: for each rule, an input just inside
its bar passes and one just outside it raises AssertionError."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import parity as P  # noqa: E402

INSIDE, OUTSIDE = 0.99, 1.01
MARGIN, LOGPROB, TOL = 5e-3, 2e-2, 3e-2  # the bars the rules are stated with, written here again on purpose


def _judge(ok, call):
    if ok:
        call()
    else:
        with pytest.raises(AssertionError):
            call()


@pytest.mark.parametrize("f", [INSIDE, OUTSIDE])
def test_check_summary(f):
    ref = torch.randn(2, 5, 4, generator=torch.Generator().manual_seed(0))
    idx = torch.tensor([[0, 1], [1, 3]])
    x = ref * (1 + f * 1e-3)  # both the row norms and the sampled rows off by f * 1e-3
    _judge(f < 1, lambda: P.check_summary("t", x, ref.double().norm(dim=-1), idx, ref[idx[:, 0], idx[:, 1]], 1e-3))


@pytest.mark.parametrize("case,f", [("all", INSIDE), ("all", OUTSIDE), ("utterance", INSIDE), ("utterance", OUTSIDE),
                                    ("nonfinite", INSIDE)])
def test_check_encoder(case, f):
    ref = torch.randn(2, 6, 4, generator=torch.Generator().manual_seed(1))
    enc = ref.clone()
    if case == "all":  # an error on utterance 1's padded frames only: the all-frames figure alone sees it
        d = ref[1, 3:]
        enc[1, 3:] = d + d / d.norm() * f * 1e-3 * ref.norm()
    elif case == "utterance":  # utterance 1 has 3 valid frames: an error there is diluted in the all-frames figure
        enc[1, :3] = ref[1, :3] * (1 + f * 1e-3)
    else:
        enc[1, 5, 0] = float("nan")
    _judge(case != "nonfinite" and f < 1, lambda: P.check_encoder("t", enc, ref, [6, 3], 1e-3))


@pytest.mark.parametrize("case,f", [("margin", INSIDE), ("margin", OUTSIDE), ("logprob", INSIDE), ("logprob", OUTSIDE),
                                    ("min_compared", INSIDE), ("min_compared", OUTSIDE), ("stop_at", INSIDE)])
def test_check_greedy(case, f):
    tokens = torch.tensor([[5, 6, 7, 8], [5, 6, 2, 9]])
    margin = torch.ones(2, 4)
    lp = -torch.ones(2, 4)
    pred, score, kw = tokens.clone(), lp.clone(), {}
    if case == "margin":  # a different token where the reference's margin is f times the near-tie bar
        pred[0, 2], margin[0, 2] = 3, f * MARGIN
    elif case == "logprob":
        score[1, 1] += f * LOGPROB
    elif case == "min_compared":  # a near tie at step 1 leaves 5 of 8 decisions compared
        pred[0, 1], margin[0, 1] = 3, 0.0
        kw = dict(min_compared=f * 5 / 8)
    else:  # a row stops at the reference's EOS (2): what follows is not compared
        pred[1, 3] = 3
        kw = dict(stop_at=2)
    _judge(f < 1, lambda: P.check_greedy("t", pred, score, tokens, margin, lp, **kw))


@pytest.mark.parametrize("case,f", [("best", INSIDE), ("best", OUTSIDE), ("nbest", INSIDE), ("nbest", OUTSIDE),
                                    ("own_score", INSIDE), ("own_score", OUTSIDE), ("worse", INSIDE), ("worse", OUTSIDE)])
def test_check_beam(case, f):
    tol = TOL
    ref_scores = torch.tensor([[-5.0, -5.5, -6.0], [-3.0, -3.2, -4.0]])
    scores = ref_scores.clone()
    ref_hyps, hyps = [[4, 5, 2], [6, 2]], [[4, 5, 2], [6, 2]]
    rescored = {}
    if case == "best":
        scores[1, 0] += f * tol
    elif case == "nbest":
        scores[0, 2] -= f * tol
    else:  # utterance 0 returned another best hypothesis; the oracle rescores it along our tokens
        hyps[0] = [4, 7, 2]
        if case == "own_score":
            rescored[0] = float(scores[0, 0]) + f * tol
        else:  # our score half a tolerance below the reference's best, the oracle's f tolerances below it
            scores[0, 0] -= 0.5 * tol
            rescored[0] = float(ref_scores[0, 0]) - f * tol
    _judge(f < 1, lambda: P.check_beam("t", hyps, scores, ref_hyps, ref_scores, lambda idx, toks: [rescored[b] for b in idx]))


@pytest.mark.parametrize("case,f", [("abs", INSIDE), ("abs", OUTSIDE), ("relative", INSIDE), ("relative", OUTSIDE),
                                    ("rerun", INSIDE)])
def test_check_alone_vs_batch(case, f):
    batch = torch.randn(2, 5, 3, generator=torch.Generator().manual_seed(2)) * 4.0
    scale = float(batch[0].abs().max()) if case == "relative" else 1.0
    alone = batch[:1].clone()
    alone[0, 2, 1] += f * 1e-5 * scale
    calls = []

    def encode(wav, lens):
        calls.append(wav.shape[0])
        if wav.shape[0] == 1:
            return alone
        return (batch + (1e-7 if case == "rerun" and len(calls) > 1 else 0.0), torch.arange(3))

    _judge(case != "rerun" and f < 1,
           lambda: P.check_alone_vs_batch(encode, torch.zeros(2, 8), torch.ones(2), 1e-5, relative=case == "relative"))


@pytest.mark.parametrize("case,f", [("logprob", INSIDE), ("logprob", OUTSIDE), ("argmax", INSIDE), ("argmax", OUTSIDE),
                                    ("padding", OUTSIDE)])
def test_check_ctc_argmax(case, f):
    from speechbrain_b200.decoders.ctc import greedy_from_argmax
    ref_lp = torch.log_softmax(torch.randn(2, 6, 5, generator=torch.Generator().manual_seed(3)) * 3.0, -1)
    lens = torch.tensor([1.0, 0.5])  # utterance 1: 3 valid frames
    margin = torch.ones(2, 6)
    if case == "logprob":
        ref_argmax = ref_lp.argmax(-1)
        lp = ref_lp.clone()
        lp[1, 2, int(ref_argmax[1, 2])] += f * LOGPROB
    else:  # a near tie the device breaks the other way, on a valid frame or on a padded one (never judged)
        b, t = (1, 4) if case == "padding" else (0, 3)
        top, other = ref_lp[b, t].topk(2).indices.tolist()
        ref_lp[b, t, other] = ref_lp[b, t, top] - 1e-3
        ref_argmax = ref_lp.argmax(-1)
        lp = ref_lp.clone()
        lp[b, t, other] += 2e-3
        margin[b, t] = f * MARGIN
    ref_hyps = greedy_from_argmax(ref_argmax, lens, 0)
    _judge(f < 1 or case == "padding", lambda: P.check_ctc_argmax("t", lp, ref_lp, ref_argmax, margin, lens, 0, ref_hyps))
