"""TransformerLM -- mirror of speechbrain.lobes.models.transformer.TransformerLM.TransformerLM (TransformerLM.py:22-187):
same constructor kwargs and state_dict keys (so ``lm.ckpt`` loads unchanged).  ``forward(src)`` runs the whole-sequence
(prefill) pass on the device (csrc/engine.cu run_lm_forward); the beam search's shallow fusion and the n-best rescorer
keep the KV-cached step (enqueue_lm_step).

Built: head width 64 with d_model a multiple of 128, and the Switchboard recipe's LM (d_model 264, 12 heads of 22,
d_embedding 128, whose embedding_proj the device folds into the embedding table)."""
SWITCHBOARD_LM_SHAPE = (264, 12, 128)  # (d_model, nhead, d_embedding) of Switchboard/LM/hparams/transformer.yaml
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
        switchboard = (d_model, nhead, d_embedding) == SWITCHBOARD_LM_SHAPE
        if d_embedding is not None and d_embedding != d_model and not switchboard:
            bad.append("d_embedding other than d_model (or 128 with the Switchboard LM's d_model 264 and 12 heads)")
        if attention_type != "regularMHA" or positional_encoding != "fixed_abs_sine" or not causal:
            bad.append("attention_type / positional_encoding / causal other than the recipe's")
        if not switchboard and (d_model % nhead or d_model // nhead != 64 or d_model % 128):
            bad.append("head_dim != 64 or d_model % 128 != 0")
        act = getattr(activation, "__name__", str(activation))
        if act not in ("GELU", "ReLU"):
            bad.append(f"activation {act}")
        if bad:
            raise NotImplementedError("speechbrain_b200.TransformerLM: not built: " + ", ".join(bad))
        self.vocab, self.d_model, self.nhead, self.num_encoder_layers, self.d_ffn = vocab, d_model, nhead, num_encoder_layers, d_ffn
        self.activation = "gelu" if act == "GELU" else "relu"
        self.max_length = max_length
        self.d_embedding = d_embedding if switchboard else None  # (d_embedding == d_model builds no projection)
        build_param_tree(self, transformer_lm_shapes(vocab, d_model, nhead, num_encoder_layers, d_ffn, self.d_embedding),
                         default_init)
        self.positional_encoding = _Node()
        self.positional_encoding.register_buffer("pe", _sine_table(max_length, d_model))
        self._slot = None

    def engine_cfg(self):
        return dict(d_model=self.d_model, nhead=self.nhead, num_encoder_layers=self.num_encoder_layers, d_ffn=self.d_ffn,
                    activation=self.activation)

    def _engine_base_cfg(self):
        # an LM-only engine: the ASR fields are placeholders the "lm" part does not read (as TransformerLMRescorer's)
        return dict(n_fft=400, hop=160, n_mels=80, cnn_channels=(64, 32), input_size=640, d_model=512, nhead=8,
                    num_encoder_layers=0, num_decoder_layers=0, d_ffn=2048, vocab=self.vocab, attention_type="RoPEMHA",
                    max_length=self.max_length)

    def _get_engine(self, device):
        if self._slot is None:
            from ....engine_cache import EngineSlot
            self._slot = EngineSlot(self._engine_base_cfg)
        return self._slot.get(device, ("lm",), {"lm.": self})

    @torch.no_grad()
    def forward(self, src):
        """src [n, s] int64 / int32 CUDA token ids (0 = padding) -> logits [n, s, vocab] fp32 CUDA (TransformerLM.py:127-169:
        causal self-attention with make_masks' look-ahead and key-padding masks)."""
        if not src.is_cuda:
            raise RuntimeError("speechbrain_b200.TransformerLM.forward: expected a CUDA tensor (no CPU path)")
        if src.dim() != 2 or src.dtype not in (torch.int64, torch.int32):
            raise ValueError(f"TransformerLM.forward: expected [n, s] int64/int32 token ids, got {src.dtype} {tuple(src.shape)}")
        n, s = src.shape
        if s > self.max_length:
            raise ValueError(f"TransformerLM.forward: {s} positions exceed max_length={self.max_length}")
        if n == 0 or s == 0:
            return torch.empty(n, s, self.vocab, device=src.device, dtype=torch.float32)
        lo, hi = torch.aminmax(src)
        if int(lo) < 0 or int(hi) >= self.vocab:  # F.embedding raises on such ids
            raise IndexError(f"TransformerLM.forward: token ids must be in [0, {self.vocab}), got [{int(lo)}, {int(hi)}]")
        return self._get_engine(src.device).lm_forward(src)
