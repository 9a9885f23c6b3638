"""-m gpu tests of the early-exit poll (sbk_asr_set_poll_interval).  Greedy and beam search read the device's count of
finished rows every `poll` steps and stop at the first poll that finds the search over, so a search that is over after n
steps runs min(max_steps, ceil(n / poll) * poll) steps, and its outputs are the first steps of the fixed-length run
(poll 0, no early exit)."""
import pytest
import torch

from speechbrain_b200.engine import AsrEngine
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state

pytestmark = pytest.mark.gpu
CFG = dict(CONFORMER_LARGE, num_encoder_layers=1, num_decoder_layers=2)
S = 40    # max_steps
BOS = 1


@pytest.fixture(scope="module")
def setup():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    dev = torch.device("cuda:0")
    eng = AsrEngine(CFG, seeded_asr_state(CFG, 0), device=dev)
    g = torch.Generator().manual_seed(0)
    enc = torch.randn(4, 60, CFG["d_model"], generator=g).to(dev)
    lens = torch.tensor([1.0, 0.9, 0.75, 0.6], device=dev)
    # eos candidates: the tokens a fixed-length run emits, the one that every row emits soonest first
    eng.set_poll_interval(0)
    pred = eng.greedy_from_enc(enc, lens, S, BOS, 2)[0].cpu()
    first = {}
    for v in pred.unique().tolist():
        hit = pred == v
        ends = torch.where(hit.any(1), hit.int().argmax(1) + 1, S + 1)
        first[v] = int(ends.max())
    return eng, enc, lens, sorted(first, key=lambda v: (first[v], v))


def _expected(n, poll):
    return min(S, -(-n // poll) * poll)


def test_greedy_steps_done_per_poll_interval(setup):
    eng, enc, lens, cands = setup
    for eos in cands[:8]:
        eng.set_poll_interval(0)
        pred0, score0, _, done0 = eng.greedy_from_enc(enc, lens, S, BOS, eos)
        assert done0 == S
        hit = (pred0 == eos).cpu()
        if hit.any(1).all():
            break
    else:
        pytest.fail("no candidate eos ends every row within max_steps")
    n = int((hit.int().argmax(1) + 1).max())  # the step after which every row has ended
    assert n < S
    for poll in (1, 3, 8):
        eng.set_poll_interval(poll)
        pred, score, _, done = eng.greedy_from_enc(enc, lens, S, BOS, eos)
        assert done == _expected(n, poll), (poll, n, done)
        assert torch.equal(pred[:, :done], pred0[:, :done]) and torch.equal(score[:, :done], score0[:, :done])
    eng.set_poll_interval(0)


def test_beam_steps_done_per_poll_interval(setup):
    eng, enc, lens, cands = setup
    beam = dict(beam_size=2, max_steps=S, min_steps=0, bos=BOS, using_eos_threshold=False)
    eng.set_poll_interval(1)  # polls after every step: the step the search is over
    for eos in cands[:8]:
        hist1 = eng.beam_from_enc(enc, lens, eos=eos, **beam)
        if len(hist1[0]) < S:
            break
    else:
        pytest.fail("no candidate eos ends the search within max_steps")
    n = len(hist1[0])
    eng.set_poll_interval(0)
    hist0 = eng.beam_from_enc(enc, lens, eos=eos, **beam)
    assert len(hist0[0]) == S
    for poll in (1, 3, 8):
        eng.set_poll_interval(poll)
        hist = eng.beam_from_enc(enc, lens, eos=eos, **beam)
        done = len(hist[0])
        assert done == _expected(n, poll), (poll, n, done)
        assert all(torch.equal(a, b[:done]) for a, b in zip(hist, hist0))
    eng.set_poll_interval(0)
