"""TransformerLM -- parameter container mirroring speechbrain.lobes.models.transformer.TransformerLM.TransformerLM
(TransformerLM.py:22-187) for its use as a shallow-fusion scorer inside the H100 beam search: same constructor kwargs and
state_dict keys (so ``lm.ckpt`` loads unchanged); the forward pass runs inside the engine with a KV cache
(csrc/engine.cu enqueue_lm_step), so calling the module directly is not part of the hot path."""
import torch

from ....utils.param_tree import _Node, build_param_tree, default_init
from ....utils.shapes import transformer_lm_shapes
from .TransformerASR import _sine_table


class TransformerLM(torch.nn.Module):
    def __init__(self, vocab, d_model=512, nhead=8, num_encoder_layers=12, num_decoder_layers=0, d_ffn=2048, dropout=0.1,
                 activation=torch.nn.ReLU, positional_encoding="fixed_abs_sine", normalize_before=False, d_embedding=None,
                 max_length=2500, causal=True, attention_type="regularMHA", decoder_use_memory=False):
        super().__init__()
        bad = []
        if num_decoder_layers != 0:
            bad.append("num_decoder_layers != 0")
        if normalize_before:
            bad.append("normalize_before=True")
        if d_embedding is not None and d_embedding != d_model:
            bad.append("d_embedding != d_model")
        if attention_type != "regularMHA" or positional_encoding != "fixed_abs_sine" or not causal:
            bad.append("attention_type / positional_encoding / causal other than the recipe's")
        if d_model % nhead or d_model // nhead != 64 or d_model % 128:
            bad.append("head_dim != 64 or d_model % 128 != 0")
        act = getattr(activation, "__name__", str(activation))
        if act not in ("GELU", "ReLU"):
            bad.append(f"activation {act}")
        if bad:
            raise NotImplementedError("speechbrain_b200.TransformerLM: not built: " + ", ".join(bad))
        self.vocab, self.d_model, self.nhead, self.num_encoder_layers, self.d_ffn = vocab, d_model, nhead, num_encoder_layers, d_ffn
        self.activation = "gelu" if act == "GELU" else "relu"
        build_param_tree(self, transformer_lm_shapes(vocab, d_model, nhead, num_encoder_layers, d_ffn), default_init)
        self.positional_encoding = _Node()
        self.positional_encoding.register_buffer("pe", _sine_table(max_length, d_model))

    def engine_cfg(self):
        return dict(d_model=self.d_model, nhead=self.nhead, num_encoder_layers=self.num_encoder_layers, d_ffn=self.d_ffn,
                    activation=self.activation)

    def forward(self, src):
        raise NotImplementedError("speechbrain_b200.TransformerLM runs inside the beam search engine (TransformerLMScorer)")
