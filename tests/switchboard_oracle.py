"""CPU restatement of the Switchboard recipe's TransformerLM (d_model 264, 12 heads of 22, d_embedding 128): the
embedding is NormalizedEmbedding(128) (times sqrt(128)) followed by embedding_proj = Linear(128, 264)
(TransformerLM.py:102-112, 140-143), the rest is oracle/asr_oracle.py's post-norm transformer_lm_forward.  The projected
table is handed to that function divided by sqrt(d_model), which it multiplies back.  The ASR part of the recipe is
tests/transformer_oracle.py at d_model 256.  Test infrastructure only: tools/make_switchboard_golden.py asserts that it
equals the running reference."""
import math

import torch

from oracle import asr_oracle as O

CFG = dict(d_model=264, nhead=12, num_encoder_layers=12, d_ffn=1024, activation="relu")


def projected_table(sd, prefix=""):
    """[vocab, d_model] = embedding_proj(sqrt(d_embedding) E), in E's dtype"""
    E = sd[prefix + "custom_src_module.emb.Embedding.weight"]
    return torch.nn.functional.linear(E * math.sqrt(E.shape[1]), sd[prefix + "embedding_proj.w.weight"],
                                      sd[prefix + "embedding_proj.w.bias"])


def plain_state(sd, prefix=""):
    """sd with the projection folded into a d_model-wide table for transformer_lm_forward"""
    out = {k: v for k, v in sd.items() if not k.startswith(prefix + "embedding_proj.")}
    out[prefix + "custom_src_module.emb.Embedding.weight"] = projected_table(sd, prefix) / math.sqrt(CFG["d_model"])
    return out


def lm_forward(tokens, sd):
    """TransformerLM.forward: tokens [n, s] (pad id 0) -> logits [n, s, vocab]"""
    return O.transformer_lm_forward(tokens, plain_state(sd), CFG)
