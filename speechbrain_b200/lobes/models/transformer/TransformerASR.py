"""TransformerASR -- drop-in for speechbrain.lobes.models.transformer.TransformerASR.TransformerASR
(TransformerASR.py:167-675) restricted to what the Conformer, HyperConformer and Branchformer ASR recipes instantiate:
encoder_module="conformer" with attention_type in {"RoPEMHA", "RelPosMHAXL", "hypermixing"} and normalize_before=True
(head width d_model / nhead of 64, 36 or 32, and 80 with RelPosMHAXL: the d_model 640 conformer_large recipes;
hypermixing: HyperMixing token mixing, nnet/hypermixing.py, with head width d_model / nhead of 32 or 64 and
d_ffn / nhead a multiple of 16 up to 256), or encoder_module="branchformer" with attention_type="RelPosMHAXL"
(Branchformer.py:92-410), or encoder_module="transformer" with attention_type="regularMHA",
positional_encoding="fixed_abs_sine" and normalize_before=True (Transformer.py:311-490, head width 64 or 128); causal=False.
The decoder's FFN activation is GELU, ReLU or Swish / SiLU; the Conformer's (conformer_activation) is Swish / SiLU or
torch.nn.GELU (exact erf, the Loquacious recipes).

Same constructor kwargs, same state_dict keys (incl. the positional buffers), ``encode()`` on the sm_90a
kernels.  ``decode()`` / ``forward()`` run teacher-forced on the KV-cached decoder step (the searchers in
speechbrain_b200.decoders drive the same step one token at a time).
"""
import math

import torch

from ...._lib import require_cuda
from ....utils.param_tree import _Node, build_param_tree, default_init
from ....utils.shapes import transformer_asr_shapes


HYPERMIXING_MAX_FRAMES = 3000  # HyperMixing(max_length=3000) (hypermixing.py:60): longer inputs fail in the reference


def _sine_table(max_len, d):
    """Transformer.py:252-303 PositionalEncoding buffer ``pe`` (1, max_len, d)."""
    pe = torch.zeros(max_len, d)
    pos = torch.arange(0, max_len).unsqueeze(1).float()
    den = torch.exp(torch.arange(0, d, 2).float() * -(math.log(10000.0) / d))
    pe[:, 0::2] = torch.sin(pos * den)
    pe[:, 1::2] = torch.cos(pos * den)
    return pe.unsqueeze(0)


class TransformerASR(torch.nn.Module):
    def __init__(self, tgt_vocab, input_size, d_model=512, nhead=8, num_encoder_layers=6, num_decoder_layers=6,
                 d_ffn=2048, dropout=0.1, activation=torch.nn.ReLU, positional_encoding="fixed_abs_sine",
                 normalize_before=False, kernel_size=31, bias=True, encoder_module="transformer",
                 conformer_activation=None, branchformer_activation=None, attention_type="regularMHA",
                 max_length=2500, causal=None, csgu_linear_units=3072, gate_activation=None,
                 use_linear_after_conv=False, output_hidden_states=False, layerdrop_prob=0.0):
        super().__init__()
        # same argument validation as Transformer.py:141-147,206-212
        assert attention_type in ["regularMHA", "RelPosMHAXL", "hypermixing", "RoPEMHA"]
        assert positional_encoding in ["fixed_abs_sine", None]
        assert num_encoder_layers + num_decoder_layers > 0, \
            "number of encoder layers and number of decoder layers cannot both be 0!"
        if encoder_module == "conformer":
            assert normalize_before, "normalize_before must be True for Conformer"
        if causal is None:
            causal = True  # the reference warns and assumes True (TransformerASR.py:274-282)
        unsupported = []
        if encoder_module not in ("conformer", "branchformer", "transformer"):
            unsupported.append(f"encoder_module={encoder_module!r}")
        if encoder_module == "transformer":
            if attention_type != "regularMHA":
                unsupported.append(f"Transformer encoder with attention_type={attention_type!r} (regularMHA only)")
            if not normalize_before:
                unsupported.append("Transformer encoder with normalize_before=False (post-norm)")
            if positional_encoding != "fixed_abs_sine":
                unsupported.append(f"Transformer encoder with positional_encoding={positional_encoding!r}")
            if d_model % nhead or d_model // nhead not in (128, 64):
                unsupported.append(f"Transformer encoder head_dim={d_model // max(nhead, 1)} (128 or 64)")
        elif attention_type not in ("RoPEMHA", "RelPosMHAXL", "hypermixing"):
            unsupported.append(f"attention_type={attention_type!r}")
        if attention_type == "hypermixing" and encoder_module == "conformer":
            if d_model % nhead or d_model // nhead not in (64, 32):
                unsupported.append(f"hypermixing head width d_model / nhead = {d_model / max(nhead, 1):g} (32 or 64)")
            if d_ffn % nhead or (d_ffn // nhead) % 16 or d_ffn // nhead > 256:
                unsupported.append(f"hypermixing d_ffn / nhead = {d_ffn / max(nhead, 1):g} (a multiple of 16 up to 256)")
        bf_act = "gelu"
        if encoder_module == "branchformer":
            if attention_type != "RelPosMHAXL":
                unsupported.append(f"Branchformer with attention_type={attention_type!r} (RelPosMHAXL only)")
            name = getattr(branchformer_activation, "__name__", "GELU") if branchformer_activation is not None else "GELU"
            if name not in ("GELU", "ReLU"):
                unsupported.append(f"branchformer_activation={name} (GELU or ReLU)")
            bf_act = "relu" if name == "ReLU" else "gelu"
            if gate_activation is not None and getattr(gate_activation, "__name__", "") != "Identity":
                unsupported.append("gate_activation other than Identity")
            if use_linear_after_conv:
                unsupported.append("use_linear_after_conv=True")
            if kernel_size % 2 == 0 or kernel_size > 31:
                unsupported.append(f"Branchformer kernel_size={kernel_size} (odd, <= 31)")
            if csgu_linear_units % 2 or (csgu_linear_units // 2) % 8:
                unsupported.append(f"csgu_linear_units={csgu_linear_units} (even, with csgu_linear_units / 2 a multiple of 8)")
        if causal:
            unsupported.append("causal=True (streaming / chunked masks)")
        if not bias:
            unsupported.append("bias=False")
        if output_hidden_states:
            unsupported.append("output_hidden_states=True")
        conf_act = "swish"
        if encoder_module == "conformer" and conformer_activation is not None:
            # torch.nn.GELU itself is the exact erf form; a partial or subclass (e.g. approximate="tanh") is another function
            if conformer_activation is torch.nn.GELU:
                conf_act = "gelu"
            elif getattr(conformer_activation, "__name__", "") not in ("Swish", "SiLU"):
                unsupported.append("conformer_activation other than Swish or torch.nn.GELU")
        if encoder_module != "transformer" and (d_model % nhead or d_model // nhead not in (64, 36, 32)):
            if not (encoder_module == "conformer" and attention_type == "RelPosMHAXL" and d_model == 80 * nhead):
                unsupported.append(f"head_dim={d_model // max(nhead, 1)} (64, 36 or 32; 80 for the Conformer with RelPosMHAXL)")
        if d_model % 16:
            unsupported.append("d_model not a multiple of 16")
        if unsupported:
            raise NotImplementedError("speechbrain_b200.TransformerASR: not built: " + ", ".join(unsupported))
        act_name = getattr(activation, "__name__", str(activation))
        dec_acts = {"GELU": "gelu", "ReLU": "relu", "Swish": "swish", "SiLU": "swish"}
        if act_name not in dec_acts:
            raise NotImplementedError(f"speechbrain_b200.TransformerASR: decoder activation {act_name} not built")
        self.decoder_activation = dec_acts[act_name]
        self.tgt_vocab, self.input_size, self.d_model, self.nhead = tgt_vocab, input_size, d_model, nhead
        self.num_encoder_layers, self.num_decoder_layers, self.d_ffn = num_encoder_layers, num_decoder_layers, d_ffn
        self.kernel_size, self.attention_type, self.max_length, self.causal = kernel_size, attention_type, max_length, causal
        self.positional_encoding_type = positional_encoding
        self.encoder_module, self.csgu_linear_units, self.branchformer_activation = encoder_module, csgu_linear_units, bf_act
        self.conformer_activation = conf_act
        build_param_tree(self, transformer_asr_shapes(tgt_vocab, input_size, d_model, nhead, num_encoder_layers,
                                                      num_decoder_layers, d_ffn, kernel_size, attention_type, encoder_module,
                                                      csgu_linear_units), default_init)
        # buffers the reference keeps in its state_dict (Transformer.py:150-163)
        if attention_type == "RelPosMHAXL":
            self.positional_encoding = _Node()
            inv = torch.exp(torch.arange(0, d_model, 2, dtype=torch.float32) * -(math.log(10000.0) / d_model))
            self.positional_encoding.register_buffer("inv_freq", inv)
        elif positional_encoding == "fixed_abs_sine":
            self.positional_encoding = _Node()
            self.positional_encoding.register_buffer("pe", _sine_table(max_length, d_model))
        if attention_type == "hypermixing":
            # no positional_encoding_decoder: the decoder adds positional_encoding (TransformerASR.py:455-466), the same
            # table the engine computes; every HyperMixing layer keeps its own 3000-row table (hypermixing.py:74-81),
            # one shared tensor here
            pe_hm = _sine_table(HYPERMIXING_MAX_FRAMES, d_model)
            for i in range(num_encoder_layers):
                getattr(self.encoder.layers, str(i)).mha_layer.add_module("positional_encoding", _Node())
                getattr(self.encoder.layers, str(i)).mha_layer.positional_encoding.register_buffer("pe", pe_hm)
        elif attention_type != "regularMHA":  # with regularMHA the decoder adds positional_encoding, as HyperMixing's does
            self.positional_encoding_decoder = _Node()
            self.positional_encoding_decoder.register_buffer("pe", _sine_table(max_length, d_model))
        # engine slots (plain dict, not sub-modules): one shared device engine per set of modules wired to this model
        object.__setattr__(self, "_slots", {})

    def engine_cfg(self):
        # the front-end each encoder's recipes pair it with: for the Transformer the LibriSpeech recipes' 3-block one, or
        # AISHELL-1's 2-block one with 256 channels (20 x 256 = 5120 features at 80 mels); else the 2-block (64, 32) one
        tfm = self.encoder_module == "transformer"
        cnn3 = tfm and self.input_size != 5120
        return dict(n_fft=400, hop=160, win=400, n_mels=80,
                    cnn_channels=(64, 64) if cnn3 else (256, 256) if tfm else (64, 32),
                    cnn_blocks=3 if cnn3 else 2, input_size=self.input_size,
                    d_model=self.d_model, nhead=self.nhead, num_encoder_layers=self.num_encoder_layers,
                    num_decoder_layers=self.num_decoder_layers, d_ffn=self.d_ffn, vocab=self.tgt_vocab,
                    kernel_size=self.kernel_size, attention_type=self.attention_type,
                    decoder_activation=self.decoder_activation, max_length=self.max_length,
                    encoder_module=self.encoder_module, csgu_linear_units=self.csgu_linear_units,
                    branchformer_activation=self.branchformer_activation,
                    conformer_activation=self.conformer_activation)

    def prefixed_state(self, prefix="Transformer."):
        return {prefix + k: v for k, v in self.state_dict().items()}

    def engine_slot(self, key=()):
        """The shared ``EngineSlot`` for the modules identified by ``key`` (ids of the output head / LM / CTC head wired to
        this model by a searcher); every mirror using the same modules gets the same repacked device engine."""
        from ....engine_cache import EngineSlot
        if key not in self._slots:
            slot = EngineSlot(self.engine_cfg)
            slot.sources["Transformer."] = self
            self._slots[key] = slot
        return self._slots[key]

    def invalidate_engines(self):
        """Drop every cached device engine (needed only after edits through ``param.data``; ``load_state_dict``, ``.to()``
        and in-place ops on the parameters are detected)."""
        for slot in self._slots.values():
            slot.invalidate()

    def _get_engine(self, device):
        """Engine for ``encode``: any slot that already holds the encoder (e.g. the one EncoderDecoderASR or a searcher
        built), else an encoder-only one."""
        for slot in self._slots.values():
            if "encoder" in slot.parts and slot.engine is not None:
                return slot.get(device, ("encoder",))
        return self.engine_slot().get(device, ("encoder",))

    @torch.no_grad()
    def encode(self, src, wav_len=None, pad_idx=0, dynchunktrain_config=None):
        """src [B, T, F] or [B, T, F', C] -> encoder_out [B, T, d_model] (TransformerASR.py:475-544).

        ``dynchunktrain_config`` (a ``DynChunkTrainConfig``): chunked attention + Dynamic Chunk Convolution, i.e. the masked
        evaluation mode whose outputs equal chunk-by-chunk streaming (TransformerASR.py:46-105, Conformer.py:190-313).
        The Branchformer has no such mode (an AssertionError, like Branchformer.py:369) and needs more than
        (kernel_size - 1) / 2 frames: its reflect-padded CSGU convolution fails on shorter inputs in the reference.
        HyperMixing ignores the chunked attention mask and mixes the whole utterance, so the masked mode would not equal
        streaming (NotImplementedError), and it takes at most 3000 frames: its positional table fails to broadcast on
        longer inputs in the reference (RuntimeError, raised here before any device work)."""
        if src.dim() == 4:
            bz, t, ch1, ch2 = src.shape
            src = src.reshape(bz, t, ch1 * ch2)
        if self.encoder_module == "transformer" and dynchunktrain_config is not None:
            raise NotImplementedError("TransformerASR: the Transformer encoder's chunked (streaming-equivalent) mode is not built")
        if self.encoder_module == "branchformer":
            assert dynchunktrain_config is None, "Dynamic Chunk Training unsupported for this encoder"
            halo = (self.kernel_size - 1) // 2
            if src.shape[1] <= halo:
                raise RuntimeError(f"TransformerASR.encode: the Branchformer's reflect padding ({halo} frames) needs more than "
                                   f"{halo} frames, got {src.shape[1]}")
        if self.attention_type == "hypermixing":
            if dynchunktrain_config is not None:
                raise NotImplementedError("TransformerASR: HyperMixing has no chunked (streaming-equivalent) mode: it "
                                          "ignores the attention mask and mixes the whole utterance")
            if src.shape[1] > HYPERMIXING_MAX_FRAMES:
                raise RuntimeError(f"TransformerASR.encode: HyperMixing's positional table has {HYPERMIXING_MAX_FRAMES} "
                                   f"rows, got {src.shape[1]} frames")
        require_cuda(src, "TransformerASR.encode")
        if wav_len is not None and float(wav_len.max()) < 1.0 - 1e-6:
            # the reference builds its mask with width max(abs_len) and then fails to broadcast (dataio.py:836)
            raise ValueError("wav_len: the longest utterance must have relative length 1.0")
        eng = self._get_engine(src.device)
        if dynchunktrain_config is None:
            return eng.encode_from_cnn(src, wav_len)
        if dynchunktrain_config.chunk_size <= 0:
            raise ValueError("DynChunkTrainConfig.chunk_size must be > 0")
        eng.set_dynchunk(dynchunktrain_config.chunk_size, dynchunktrain_config.left_context_size)
        try:
            return eng.encode_from_cnn(src, wav_len)
        finally:
            eng.set_dynchunk(0)

    # ------------------------------------------------------------------ streaming (TransformerASR.py:546-670)
    def _check_streaming(self):
        if self.encoder_module == "transformer":
            raise NotImplementedError("TransformerASR: streaming for the Transformer encoder is not built")
        if self.encoder_module == "branchformer":
            raise NotImplementedError("TransformerASR: the Branchformer encoder has no streaming mode")
        if self.attention_type == "hypermixing":
            raise NotImplementedError("TransformerASR: HyperMixing has no streaming mode")
        if self.d_model // self.nhead == 80:
            raise NotImplementedError("TransformerASR: streaming is not built for head width 80")

    def make_streaming_context(self, dynchunktrain_config):
        """Streaming context for ``encode_streaming`` (TransformerASR.py:645-670).  An infinite left context
        (``left_context_size=None``) is accepted: the context then keeps every frame (with RelPosMHAXL, up to max_length)."""
        self._check_streaming()
        if dynchunktrain_config is None or dynchunktrain_config.chunk_size <= 0:
            raise ValueError("make_streaming_context needs a DynChunkTrainConfig with chunk_size > 0")
        return TransformerASRStreamingContext(dynchunktrain_config, ConformerEncoderStreamingContext(
            dynchunktrain_config, self.num_encoder_layers, self.nhead))

    @torch.no_grad()
    def encode_streaming(self, src, context):
        """Encoder output for one more chunk of ``src`` [B, n <= chunk_size, F] (TransformerASR.py:546-643).

        The context keeps, per layer, the projected keys / values of the left context and the Dynamic Chunk Convolution's
        last (kernel_size - 1) / 2 inputs on the device, so every chunk costs the same however long the stream.  The outputs
        equal the masked full-sequence run ``encode(..., dynchunktrain_config)`` (tests/unittests/test_conformer.py).  The B
        streams of a batch advance together; only the last chunk of a stream may be shorter than chunk_size."""
        self._check_streaming()
        require_cuda(src, "TransformerASR.encode_streaming")
        if src.dim() == 4:
            src = src.reshape(src.shape[0], src.shape[1], -1)
        ec = context.encoder_context
        eng = ec.slot.get(src.device, ("encoder",)) if ec.slot is not None else self._get_engine(src.device)
        out = ec.ensure_stream(eng, src.shape[0]).encode_chunk(src)
        ec.frames += src.shape[1]
        return out

    def _decoder_engine(self, device):
        """Engine for ``decode``: a searcher's slot when one is wired to this model (its engine already holds the decoder),
        else a decoder-only engine without the output head."""
        for slot in self._slots.values():
            if "seq_lin." in slot.sources:
                return slot.get(device, ("decoder",))
        return self.engine_slot().get(device, ("decoder",))

    @torch.no_grad()
    def decode(self, tgt, encoder_out, enc_len=None):
        """TransformerASR.py:426-473: tgt [n, s] token ids (bos first), encoder_out [n, T, d], enc_len [n] ABSOLUTE frame
        counts -> (prediction [n, s, d] = decoder.norm(decoder(...)), None).

        Runs teacher-forced on the KV-cached decoder step: position s attends to positions <= s (the reference's causal
        mask) and to the first enc_len frames of the memory.  The reference's second value (last layer's head-averaged
        cross-attention weights [n, s, T]) is not produced by the device decoder and is returned as None."""
        require_cuda(encoder_out, "TransformerASR.decode")
        if self.num_decoder_layers == 0:
            raise ValueError("TransformerASR.decode: the model has no decoder layers")
        out = self._decoder_engine(encoder_out.device).decode_teacher_forced(tgt.long(), encoder_out, enc_len)
        return out, None

    @torch.no_grad()
    def forward(self, src, tgt, wav_len=None, pad_idx=0):
        """TransformerASR.py:326-424 for inference: (encoder_out, decoder_out).  Target positions holding ``pad_idx`` lie
        behind every real token of their row, so the causal decoder gives the real positions the reference's values; the
        padded positions (ignored by every consumer) are computed as if the pads were tokens."""
        enc = self.encode(src, wav_len, pad_idx)
        enc_len = torch.round(wav_len.to(enc.device).float() * enc.shape[1]).int() if wav_len is not None else None
        dec, _ = self.decode(tgt, enc, enc_len)
        return enc, dec


class ConformerEncoderLayerStreamingContext:
    """One layer's streaming state (Conformer.py:27-60), read from the device caches on access."""

    def __init__(self, parent, index, mha_left_context_size):
        self._parent, self._index = parent, index
        self.mha_left_context_size = mha_left_context_size

    def _caches(self):
        st = self._parent.stream
        return None if st is None or self._parent.frames == 0 else st.layer_context(self._index)

    @property
    def mha_left_context(self):
        """The projected keys of the cached frames [B, frames, d_model] (fp16; RoPE keys rotated by stream position), or
        None before the first chunk.  The shape is the reference's, the values are not: the reference keeps the layer
        inputs of the same frames and projects them again for every chunk."""
        c = self._caches()
        if c is None:
            return None
        kv = c[0]
        B, n, _ = kv.shape
        H = self._parent.nhead
        return kv.view(B, n, H, 2, kv.shape[2] // (2 * H))[:, :, :, 0].reshape(B, n, kv.shape[2] // 2)

    @property
    def dcconv_left_context(self):
        """The depthwise convolution's inputs of the last (kernel_size - 1) / 2 frames [B, (kernel_size - 1) / 2, d_model]
        (fp32, after the GLU; LayerNorm, pointwise conv and GLU act per frame), or None before the first chunk."""
        c = self._caches()
        return None if c is None else c[1]


class ConformerEncoderStreamingContext:
    """Streaming state of a Conformer encoder (Conformer.py:63-80): ``layers[i]`` per layer, backed by one device stream."""

    def __init__(self, dynchunktrain_config, num_layers, nhead):
        cfg = dynchunktrain_config
        # frames of left context per layer; None: every frame so far (the reference has no such mode)
        size = None if cfg.is_infinite_left_context() else cfg.left_context_size * cfg.chunk_size
        self.config = cfg
        self.stream = None  # speechbrain_b200.engine.EncoderStream, created by the first chunk
        self.frames = 0
        self.started = False  # the streaming front end has taken a chunk since the last reset
        self.nhead = nhead
        self.slot = None  # the EngineSlot whose engine runs the stream (StreamingASR: the one that also holds the front end)
        self.layers = [ConformerEncoderLayerStreamingContext(self, i, size) for i in range(num_layers)]

    def ensure_stream(self, eng, B):
        """The device stream of B rows on ``eng``, created on first use (and again when the batch size or the weights
        changed before the stream took any chunk)."""
        if self.stream is None or self.stream.engine is not eng or self.stream.B != B:
            if self.stream is not None and (self.frames > 0 or self.started):
                raise ValueError("encode_streaming: the batch size or the model's weights changed inside a stream")
            cfg = self.config
            left = None if cfg.is_infinite_left_context() else cfg.left_context_size * cfg.chunk_size
            self.stream = eng.stream_create(B, cfg.chunk_size, left)
        return self.stream

    def reset(self):
        """Back to an empty context (the device buffers are kept for the next stream of the same batch size)."""
        if self.stream is not None:
            self.stream.reset()
        self.frames = 0
        self.started = False


class TransformerASRStreamingContext:
    """Mutable streaming state (TransformerASR.py:26-43): the DynChunkTrainConfig and the encoder's per-layer context."""

    def __init__(self, dynchunktrain_config, encoder_context):
        self.dynchunktrain_config = dynchunktrain_config
        self.encoder_context = encoder_context

    def reset(self):
        """Forget the stream: the next chunk starts a new one, with the same configuration."""
        self.encoder_context.reset()

    @property
    def history(self):
        """The frames the context retains (layer 0's left context [B, frames, d_model]), or None before the first chunk."""
        return self.encoder_context.layers[0].mha_left_context if self.encoder_context.layers else None


class EncoderWrapper(torch.nn.Module):
    """TransformerASR.py:678-714: calls ``transformer.encode`` so the model can sit at the end of a Sequential."""

    def __init__(self, transformer, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.transformer = transformer

    def forward(self, x, wav_lens=None, pad_idx=0, **kwargs):
        return self.transformer.encode(x, wav_lens, pad_idx, **kwargs)

    def forward_streaming(self, x, context):
        """TransformerASR.py:716-737: one chunk through ``encode_streaming``."""
        return self.transformer.encode_streaming(x, context)

    def make_streaming_context(self, *args, **kwargs):
        return self.transformer.make_streaming_context(*args, **kwargs)
