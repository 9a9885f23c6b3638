"""CPU test (-m "not gpu"): oracle.transformer_lm_forward vs the REFERENCE's TransformerLM.forward fixture
(tests/golden/lm_forward.pt, written by tools/make_lm_forward_golden.py from the running reference): recipe-size LM, seed 1,
a ragged batch padded with token 0 that also holds id 0 inside some valid lengths.  Every position is compared, pad
positions included: their logits depend on the key-padding mask too."""
import os

import torch

from oracle import asr_oracle as O
from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
from speechbrain_b200.utils.seeded_init import seeded_state_dict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_lm_forward_oracle_vs_reference_golden():
    gold = torch.load(os.path.join(GOLDEN, "lm_forward.pt"))
    lm = TransformerLM(vocab=5000, d_model=768, nhead=12, num_encoder_layers=12, num_decoder_layers=0, d_ffn=3072, dropout=0.0,
                       activation=torch.nn.GELU, normalize_before=False)
    sd = seeded_state_dict(lm, seed=gold["seed"])
    cfg = dict(d_model=768, nhead=12, num_encoder_layers=12, d_ffn=3072, activation="gelu")
    tokens, lens = gold["tokens"], gold["lengths"]
    assert tokens.shape[0] >= 6 and 1 in lens.tolist() and int(lens.max()) == tokens.shape[1]
    with torch.no_grad():
        logits = O.transformer_lm_forward(tokens, sd, cfg)
    valid = torch.arange(tokens.shape[1]).unsqueeze(0) < lens.unsqueeze(1)
    assert ((tokens == 0) & valid).sum() >= 3  # interior id 0: masked keys inside the valid length
    assert torch.isfinite(logits).all()
    assert (logits.logsumexp(-1) - gold["logsumexp"]).abs().max() < 1e-3
    top_v, top_i = logits.topk(8, dim=-1)
    assert (top_v - gold["top_values"]).abs().max() < 1e-3
    margin = gold["top_values"][..., 0] - gold["top_values"][..., 1]
    sure = margin >= 5e-3
    assert torch.equal(top_i[..., 0][sure], gold["top_ids"][..., 0][sure].long())
    idx = gold["sample_idx"].long()
    sample = logits[idx[:, 0], idx[:, 1]]
    assert float((sample - gold["sample_logits"]).norm() / gold["sample_logits"].norm()) < 1e-5
