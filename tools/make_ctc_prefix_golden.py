"""Generate tests/golden/ctc_prefix.pt by RUNNING THE REFERENCE's CTCPrefixScore (decoders/ctc.py:26-295) in float64.

Run it the way oracle/make_goldens.py's docstring describes (reference package and hyperpyyaml stub on PYTHONPATH).

Each case drives CTCPrefixScore.forward_step + permute_mem along a forced search history (the way ScorerBuilder /
S2SBeamSearcher drive it: inp_tokens = the previous step's tokens, permute_mem(memory, candidates)) for every step up to
prefix_length = T, the last step the reference defines.  The history comes from oracle.ctc_history_picker (parents with
several children and with none, repeated last tokens, the best and random tokens).  Cases: blank 0 and a nonzero blank,
V = 61 (not a multiple of 4, below one 256-token CTA), ragged enc_len including 1 and T, beam 7.  The script checks
oracle.ctc_prefix_scores against the reference on every entry, then stores the inputs and the reference's psi - psi_prev.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import asr_oracle as O  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "ctc_prefix.pt")
# name: (B, T, V, beam, blank, bos, eos, enc_len, seed)
CASES = {
    "blank0_beam7": (3, 14, 61, 7, 0, 1, 2, [14, 1, 9], 11),
    "blank_nonzero": (2, 12, 61, 3, 60, 1, 2, [12, 5], 12),
}


def reference_scores(logits, enc_len, beam, blank, bos, eos, hist_tok, hist_pred, n_steps):
    from speechbrain.decoders.ctc import CTCPrefixScore
    B, T, V = logits.shape
    x = torch.log_softmax(logits.double(), dim=-1)
    sc = CTCPrefixScore(x.clone(), enc_len.long(), blank, eos)
    inp = torch.full((B * beam,), bos, dtype=torch.long)
    mem, out, prev = None, [], [torch.zeros(B * beam)]
    for s in range(n_steps):
        score, mem = sc.forward_step(inp, mem)
        out.append(score.clone())
        if s + 1 == n_steps:
            break
        loc = hist_pred[s].long() - (torch.arange(B * beam) // beam) * beam
        cand = (loc * V + hist_tok[s].long()).view(B, beam)
        mem = sc.permute_mem(mem, cand)
        prev.append(mem[1][:, 0].clone())
        inp = hist_tok[s].long()
    return torch.stack(out), torch.stack(prev)


def compare(score, ref, ref_prev):
    """Max |score - ref| over the entries whose prefix is possible (psi_prev > -1e19: the difference of two minus_inf-sized
    values is rounding noise in any precision), after checking that both sides call the same extensions impossible."""
    live = (ref_prev > -1e19).unsqueeze(-1).expand_as(ref)
    dead = ref <= -1e19
    assert torch.equal(dead[live], (score <= -1e19)[live]), "impossible-extension pattern differs"
    m = live & ~dead
    return float((score - ref)[m].abs().max()), int(m.sum())


def main():
    torch.set_default_dtype(torch.float64)   # CTCPrefixScore allocates its state with the default dtype
    gold = {}
    for name, (B, T, V, beam, blank, bos, eos, lens, seed) in CASES.items():
        g = torch.Generator().manual_seed(seed)
        logits = (torch.randn(B, T, V, generator=g) * 3.0).float()   # the fp32 the CUDA hook takes, stored as is
        enc_len = torch.tensor(lens, dtype=torch.int32)
        n_steps = T + 1
        ht = torch.zeros(n_steps, B * beam, dtype=torch.int32)
        hp = torch.zeros(n_steps, B * beam, dtype=torch.int32)
        ours = O.ctc_prefix_scores(logits, enc_len, beam, blank, bos, eos, ht, hp, n_steps,
                                   pick=O.ctc_history_picker(B, beam, V, blank, eos, seed))
        with torch.no_grad():
            ref, ref_prev = reference_scores(logits, enc_len, beam, blank, bos, eos, ht, hp, n_steps)
        err, n_cmp = compare(ours["score"], ref, ref_prev)
        print(f"[{name}] steps {n_steps}, entries {ref.numel()}, compared {n_cmp}, oracle max abs err {err:.2e}")
        assert err < 1e-9 and (ours["psi_prev"] - ref_prev).abs().max() < 1e-9
        gold[name] = dict(logits=logits, enc_len=enc_len, beam=beam, blank=blank, bos=bos, eos=eos, n_steps=n_steps,
                          hist_tok=ht, hist_pred=hp, score=ref.clone(), psi_prev=ref_prev.clone())
    torch.save(gold, OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
