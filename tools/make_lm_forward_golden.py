"""Generate tests/golden/lm_forward.pt by RUNNING THE REFERENCE's TransformerLM.forward (TransformerLM.py:127-169).

Run it the way oracle/make_goldens.py's docstring describes (reference package and hyperpyyaml stub on PYTHONPATH).

The recipe-size LM (12 x 768, 12 heads, d_ffn 3072, vocab 5000, seed 1 -- the weights of oracle/make_goldens.py's
rescore_case, regenerated from the seed, not stored) runs on a ragged batch padded with token 0, bos = 1, where some
sequences also hold id 0 inside their valid length (SentencePiece's <unk> in the recipes), so make_masks' key-padding mask
removes keys that real positions would otherwise see.  The script checks oracle.transformer_lm_forward against the
reference on every position, pad positions included, then stores a small fixture: the tokens and lengths, per position the
logsumexp of the logits and the top-8 logits / ids, and the full logit rows of a few sampled positions.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import asr_oracle as O  # noqa: E402
from speechbrain_b200.utils.seeded_init import seeded_state_dict  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "lm_forward.pt")
LENGTHS = [80, 1, 37, 64, 65, 12]  # one of length 1, one of the full s = 80, one across the 64-key attention block
INTERIOR_PAD = [(0, 5), (0, 40), (0, 70), (3, 20), (4, 64)]  # (sequence, position) holding id 0 inside the valid length


def main():
    from speechbrain.lobes.models.transformer.TransformerLM import TransformerLM
    lm = TransformerLM(vocab=5000, d_model=768, nhead=12, num_encoder_layers=12, num_decoder_layers=0, d_ffn=3072,
                       dropout=0.0, activation=torch.nn.GELU, normalize_before=False)
    sd = seeded_state_dict(lm, seed=1)
    lm.load_state_dict(sd)
    lm.eval()
    cfg = dict(d_model=768, nhead=12, num_encoder_layers=12, d_ffn=3072, activation="gelu")
    g = torch.Generator().manual_seed(2024)
    n, s = len(LENGTHS), max(LENGTHS)
    tokens = torch.zeros(n, s, dtype=torch.long)
    for i, L in enumerate(LENGTHS):
        tokens[i, 0] = 1  # bos
        if L > 1:
            tokens[i, 1:L] = torch.randint(3, 5000, (L - 1,), generator=g)
    for i, p in INTERIOR_PAD:
        tokens[i, p] = 0
    with torch.no_grad():
        ref = lm(tokens)
        ours = O.transformer_lm_forward(tokens, sd, cfg)
    lens = torch.tensor(LENGTHS)
    err = max(float((ours[i] - ref[i]).norm() / ref[i].norm()) for i in range(n))
    print(f"[lm_forward] logits {tuple(ref.shape)} oracle rel err (worst sequence, all positions) {err:.2e}")
    assert err < 1e-5 and torch.isfinite(ref).all()
    top_v, top_i = ref.topk(8, dim=-1)
    # sampled positions: the last valid position of every sequence, the first and the middle of the longest one, the
    # positions right after an interior id 0, and two pad positions
    pos = sorted({(i, L - 1) for i, L in enumerate(LENGTHS)} | {(0, 0), (0, LENGTHS[0] // 2), (0, 41), (3, 21), (1, 40),
                                                                 (5, 79)})
    sample_idx = torch.tensor(pos, dtype=torch.long)
    sample_logits = ref[sample_idx[:, 0], sample_idx[:, 1]].clone()
    torch.save(dict(tokens=tokens.to(torch.int32), lengths=lens.to(torch.int32), logsumexp=ref.logsumexp(-1).clone(),
                    top_values=top_v.clone(), top_ids=top_i.to(torch.int32), sample_idx=sample_idx.to(torch.int32),
                    sample_logits=sample_logits, vocab=5000, seed=1, bos=1, pad=0), OUT)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
