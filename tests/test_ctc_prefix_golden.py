"""CPU test (-m "not gpu"): the float64 CTC prefix-score oracle (oracle.ctc_prefix_scores, which the GPU tests of
sbk_ctc_prefix_test compare against) vs the REFERENCE's CTCPrefixScore fixture (tests/golden/ctc_prefix.pt, written by
tools/make_ctc_prefix_golden.py from the running reference in float64), and vs the older full-tensor oracle
(oracle.ctc_prefix_step / ctc_prefix_permute, which the beam-search oracle uses) on the same inputs.

Fixture cases: blank 0 with beam 7 and blank = V - 1 with beam 3, V = 61, ragged enc_len including 1 and T, every step up to
prefix_length = T, histories with repeated last tokens and parents with several children."""
import os

import torch

from oracle import asr_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _compare(score, ref, ref_prev):
    """Max |score - ref| over the extensions of possible prefixes (psi_prev > -1e19), after checking that both sides call
    the same extensions impossible (<= -1e19)."""
    live = (ref_prev > -1e19).unsqueeze(-1).expand_as(ref)
    dead = ref <= -1e19
    assert torch.equal(dead[live], (score <= -1e19)[live]), "impossible-extension pattern differs"
    m = live & ~dead
    return float((score - ref)[m].abs().max()), int(m.sum())


def _full_tensor_oracle(c):
    """ctc_prefix_step + ctc_prefix_permute along the fixture's history, float64."""
    logits, beam, n_steps = c["logits"], c["beam"], c["n_steps"]
    B, T, V = logits.shape
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        st = O.ctc_prefix_reset(torch.log_softmax(logits.double(), -1), c["enc_len"].long(), c["blank"], c["eos"])
        inp = torch.full((B * beam,), c["bos"], dtype=torch.long)
        mem, out = None, []
        for s in range(n_steps):
            score, mem = O.ctc_prefix_step(st, inp, mem, beam)
            out.append(score)
            if s + 1 < n_steps:
                loc = c["hist_pred"][s].long() - (torch.arange(B * beam) // beam) * beam
                mem = O.ctc_prefix_permute(st, mem, (loc * V + c["hist_tok"][s].long()).view(B, beam))
                inp = c["hist_tok"][s].long()
    finally:
        torch.set_default_dtype(old)
    return torch.stack(out)


def test_ctc_prefix_oracle_vs_reference_golden():
    gold = torch.load(os.path.join(GOLDEN, "ctc_prefix.pt"))
    assert {c["blank"] for c in gold.values()} >= {0, 60} and 7 in {c["beam"] for c in gold.values()}
    assert any(1 in c["enc_len"].tolist() for c in gold.values())
    for name, c in gold.items():
        B, T, V = c["logits"].shape
        assert V % 4 != 0 and V < 256 and T in c["enc_len"].tolist() and c["n_steps"] == T + 1
        ht = c["hist_tok"][: c["n_steps"] - 1]
        # the history repeats last tokens and gives some parents several children
        assert (ht[1:] == ht[:-1].gather(1, c["hist_pred"][1:c["n_steps"] - 1].long())).any()
        assert any(len(set(r.tolist())) < r.numel() for r in c["hist_pred"])
        o = O.ctc_prefix_scores(c["logits"], c["enc_len"], c["beam"], c["blank"], c["bos"], c["eos"], c["hist_tok"],
                                c["hist_pred"], c["n_steps"])
        err, n = _compare(o["score"], c["score"], c["psi_prev"])
        prev_err = float((o["psi_prev"] - c["psi_prev"]).abs().max())
        print(f"[{name}] fp64 oracle vs reference: {n} entries, max abs err {err:.2e}, psi_prev err {prev_err:.2e}")
        assert n > 1000 and err < 1e-9 and prev_err < 1e-9
        full = _full_tensor_oracle(c)
        err2, n2 = _compare(full, o["score"], o["psi_prev"])
        print(f"[{name}] ctc_prefix_step (float64) vs ctc_prefix_scores: {n2} entries, max abs err {err2:.2e}")
        assert n2 == n and err2 < 1e-9
