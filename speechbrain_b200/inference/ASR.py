"""EncoderDecoderASR -- drop-in for speechbrain.inference.ASR.EncoderDecoderASR (inference/ASR.py:35-173) for the
Conformer encoder-decoder recipes: ``encode_batch`` / ``transcribe_batch`` / ``forward`` with the reference's signatures.

Two module layouts are accepted:

* the reference's (``MODULES_NEEDED = ["encoder", "decoder"]``): ``encoder`` is a ``LengthsCapableSequential`` of
  Fbank -> InputNormalization -> ConvolutionFrontEnd [-> EncoderWrapper(TransformerASR)], ``decoder`` a
  ``S2STransformerGreedySearcher`` or ``S2STransformerBeamSearcher`` (+ ``ScorerBuilder``), and with
  ``hparams["transformer_beam_search"]`` the model itself sits under ``modules["transformer"]`` -- i.e. what
  ``speechbrain/asr-conformer-transformerlm-librispeech``'s hyperparams.yaml builds (``from_hparams`` loads such a file
  from a local directory, see ``speechbrain_b200.utils.hparams``);
* the Conformer-Transducer layout (``hparams["transducer_beam_search"]``): ``encoder`` ends in the ``proj_enc`` Linear and
  ``decoder`` is a ``TransducerBeamSearcher`` (greedy, decoders/transducer.py) that gets every frame of the batch;
* the flat layout the recipes' training YAML uses (compute_features, normalize, CNN, Transformer, seq_lin, decoder).

The waveform -> encoder states part runs as ONE fused device pipeline (Fbank + CMVN + CNN + Conformer encoder, C ABI
``sbk_asr_transcribe_greedy_*`` / ``sbk_asr_encode``); a greedy decoder stays inside the same call (one CUDA-graph-able
pipeline wav -> token ids), a beam decoder runs ``sbk_asr_beam_from_enc`` on the states.  One repacked engine is shared
by every mirror involved (engine_cache.py)."""
import types
from dataclasses import dataclass
from typing import Any, List, Optional

import torch

from ..decoders.seq2seq import (S2STransformerBeamSearcher, S2STransformerGreedySearcher, greedy_exit_step, greedy_outputs)
from ..lobes.features import Fbank
from ..lobes.models.convolution import ConvolutionFrontEnd
from ..lobes.models.transformer.TransformerASR import EncoderWrapper, TransformerASR
from ..processing.features import InputNormalization


def _find(mods, cls):
    """First module of type ``cls`` among ``mods`` and their direct children (the reference nests the front end in a
    LengthsCapableSequential)."""
    for m in mods:
        if isinstance(m, cls):
            return m
    for m in mods:
        if isinstance(m, torch.nn.Module):
            for c in m.children():
                if isinstance(c, cls):
                    return c
    return None


class EncoderDecoderASR(torch.nn.Module):
    HPARAMS_NEEDED = ["tokenizer"]
    MODULES_NEEDED = ["encoder", "decoder"]

    def __init__(self, modules=None, hparams=None, run_opts=None, freeze_params=True):
        super().__init__()
        modules = dict(modules or {})
        if "decoder" not in modules:
            raise ValueError("Need modules['decoder']")
        if "encoder" not in modules and not {"compute_features", "normalize", "CNN", "Transformer"} <= set(modules):
            raise ValueError("Need modules['encoder'] (or the flat compute_features / normalize / CNN / Transformer layout)")
        self.mods = torch.nn.ModuleDict(modules)
        self.hparams = dict(hparams) if isinstance(hparams, dict) else (dict(vars(hparams)) if hparams is not None else {})
        self.tokenizer = self.hparams.get("tokenizer")
        self.transformer_beam_search = bool(self.hparams.get("transformer_beam_search", False))
        self.transducer_beam_search = bool(self.hparams.get("transducer_beam_search", False))
        self.device = torch.device((run_opts or {}).get("device", "cuda:0"))
        dec = self.mods["decoder"]
        if self.transducer_beam_search:
            self._init_transducer()
            return
        if not isinstance(dec, (S2STransformerGreedySearcher, S2STransformerBeamSearcher)):
            raise NotImplementedError("EncoderDecoderASR: the decoder must be a speechbrain_b200 S2STransformerGreedySearcher "
                                      "or S2STransformerBeamSearcher")
        vals = list(self.mods.values())
        wrap = _find(vals, EncoderWrapper)
        # plain attributes (not sub-modules: they already live under self.mods)
        for name, m in (("fbank", _find(vals, Fbank)), ("normalize", _find(vals, InputNormalization)),
                        ("cnn", _find(vals, ConvolutionFrontEnd)),
                        ("transformer", _find(vals, TransformerASR) or (wrap.transformer if wrap is not None else None) or dec.model)):
            object.__setattr__(self, name, m)
        if self.transformer is not dec.model:
            raise ValueError("EncoderDecoderASR: the decoder's model is not the encoder's TransformerASR")
        missing = [n for n, m in (("Fbank", self.fbank), ("InputNormalization", self.normalize), ("ConvolutionFrontEnd", self.cnn))
                   if m is None]
        if missing:
            raise ValueError(f"EncoderDecoderASR: could not find {missing} among the modules")
        if self.normalize.norm_type != "global":
            raise NotImplementedError("EncoderDecoderASR: fused pipeline needs InputNormalization(norm_type='global')")

    def _init_transducer(self):
        """The Conformer-Transducer layout: ``encoder`` = LengthsCapableSequential(Fbank, InputNormalization,
        ConvolutionFrontEnd, EncoderWrapper(TransformerASR), Linear proj_enc), ``decoder`` = TransducerBeamSearcher."""
        from ..decoders.transducer import TransducerBeamSearcher
        from ..nnet.linear import Linear
        if not isinstance(self.mods["decoder"], TransducerBeamSearcher):
            raise NotImplementedError("EncoderDecoderASR(transducer_beam_search=True): the decoder must be a "
                                      "speechbrain_b200 TransducerBeamSearcher")
        if "encoder" not in self.mods:
            raise ValueError("EncoderDecoderASR(transducer_beam_search=True): need modules['encoder']")
        vals = list(self.mods["encoder"].children()) if isinstance(self.mods["encoder"], torch.nn.Module) else []
        wrap = _find(vals, EncoderWrapper)
        tr = _find(vals, TransformerASR) or (wrap.transformer if wrap is not None else None)
        for name, m in (("fbank", _find(vals, Fbank)), ("normalize", _find(vals, InputNormalization)),
                        ("cnn", _find(vals, ConvolutionFrontEnd)), ("transformer", tr), ("proj_enc", _find(vals, Linear))):
            if m is None:
                raise ValueError(f"EncoderDecoderASR: could not find the {name} module in modules['encoder']")
            object.__setattr__(self, name, m)
        if self.normalize.norm_type != "global":
            raise NotImplementedError("EncoderDecoderASR: fused pipeline needs InputNormalization(norm_type='global')")

    @classmethod
    def from_hparams(cls, source, hparams_file="hyperparams.yaml", overrides=None, savedir=None, run_opts=None, **kwargs):
        """inference/interfaces.py:385-489 for a LOCAL directory: loads ``source/hparams_file`` with the HyperPyYAML-subset
        loader (speechbrain.* dotted names are mapped onto this package), runs the ``pretrainer`` parameter transfer on the
        checkpoint files found in ``source`` and builds the interface.  There is no hub download (no network)."""
        from ..utils.hparams import load_pretrained_interface
        return load_pretrained_interface(cls, source, hparams_file, overrides or {}, run_opts or {})

    # ------------------------------------------------------------------ engine
    def engine(self):
        dec = self.mods["decoder"]
        src = {"fbank": self.fbank, "normalize": self.normalize, "CNN.": self.cnn}
        if self.transducer_beam_search:
            return self.transformer.engine_slot(("transducer",)).get(self.device, ("fbank", "cnn", "encoder"), src)
        return dec._get_engine(self.device, parts=("fbank", "cnn", "encoder"), extra_sources=src)

    def _steps(self, n_samples):
        dec = self.mods["decoder"]
        _, T = self.engine().num_frames(n_samples)
        return max(0, int(T * dec.max_decode_ratio) - int(T * dec.min_decode_ratio))

    # ------------------------------------------------------------------ reference API
    @torch.no_grad()
    def encode_batch(self, wavs, wav_lens):
        """inference/ASR.py:100-128: wavs [B, L] (+ relative lengths) -> encoder states [B, T, d]."""
        wavs = wavs.float().to(self.device)
        wav_lens = wav_lens.to(self.device)
        if self.transducer_beam_search:  # the fused wav -> encoder pipeline, then proj_enc on the wgmma GEMM
            return self.proj_enc(self.engine().encode_wav(wavs, wav_lens))
        dec = self.mods["decoder"]
        _, _, enc, _ = self.engine().transcribe_greedy_dev(wavs, wav_lens, 0, dec.bos_index, dec.eos_index, want_enc=True)
        return enc

    @torch.no_grad()
    def transcribe_batch(self, wavs, wav_lens):
        """inference/ASR.py:131-169: -> (predicted_words list[str], predicted_tokens list[list[int]])."""
        dec = self.mods["decoder"]
        if self.transducer_beam_search:
            # inference/ASR.py:160-164: the search gets every frame of the padded batch (no lengths), as the reference's
            # does, so a short utterance is also decoded over its padded frames
            hyps = dec(self.encode_batch(wavs, wav_lens))[0]
        elif isinstance(dec, S2STransformerBeamSearcher):
            enc = self.encode_batch(wavs, wav_lens)
            hyps = dec(enc, wav_lens.to(self.device))[0]
            if dec.return_topk:  # padded (B, topk, L) tensor: the best hypothesis of every utterance, like hyps[0]
                raise NotImplementedError("EncoderDecoderASR.transcribe_batch: build the searcher with return_topk=False")
        else:
            n = self._steps(wavs.shape[1])
            if wavs.is_cuda:
                pred, _, _, done = self.engine().transcribe_greedy_dev(wavs, wav_lens.to(wavs.device), n, dec.bos_index,
                                                                       dec.eos_index)
                pred = pred[:, :done].cpu()
            else:  # host buffers: H2D / D2H inside the C-ABI call
                pred, done = self.engine().transcribe_greedy_host(wavs, wav_lens, n, dec.bos_index, dec.eos_index)
                pred = pred[:, :done]
            pred = pred[:, :greedy_exit_step(pred, dec.eos_index)]
            hyps, _, _, _ = greedy_outputs(pred, torch.zeros_like(pred, dtype=torch.float32), None, dec.eos_index)
        if self.tokenizer is not None:
            words = [self.tokenizer.decode_ids(h) for h in hyps]
        else:
            words = [" ".join(map(str, h)) for h in hyps]
        return words, hyps

    def forward(self, wavs, wav_lens):
        return self.transcribe_batch(wavs, wav_lens)

    # ------------------------------------------------------------------ extension: several batches per call
    @torch.no_grad()
    def transcribe_batches_async(self, wavs_host, lens_host, preds_host, preds_dev=None):
        """Throughput form of ``transcribe_batch`` for a greedy decoder: G pinned host batches ([B, L] fp32, [B] fp32) are
        copied, encoded batch by batch and decoded together (one greedy loop over G*B rows); token ids land in the pinned
        ``preds_host`` [B, steps] int32 tensors.  Only enqueues on the current stream -- synchronise it, then pass each
        ``preds_host[g]`` to ``tokens_to_words``."""
        dec = self.mods["decoder"]
        if not isinstance(dec, S2STransformerGreedySearcher):
            raise NotImplementedError("transcribe_batches_async needs a greedy decoder")
        n = self._steps(wavs_host[0].shape[1])
        if any(p.shape[1] != n for p in preds_host):
            raise ValueError(f"preds_host tensors must be [B, {n}]")
        return self.engine().transcribe_greedy_group_host_async(wavs_host, lens_host, n, dec.bos_index, dec.eos_index,
                                                                preds_host, preds_dev)

    def tokens_to_words(self, pred):
        dec = self.mods["decoder"]
        pred = pred[:, :greedy_exit_step(pred, dec.eos_index)]
        hyps, _, _, _ = greedy_outputs(pred, torch.zeros_like(pred, dtype=torch.float32), None, dec.eos_index)
        words = [self.tokenizer.decode_ids(h) for h in hyps] if self.tokenizer is not None else [" ".join(map(str, h)) for h in hyps]
        return words, hyps


class EncoderASR(torch.nn.Module):
    """Drop-in for speechbrain.inference.ASR.EncoderASR (inference/ASR.py:176-389) with a Conformer encoder + CTC head and
    greedy decoding: ``encode_batch`` returns the log-posteriors [B, T, V] the reference's ``encoder`` Sequential ends in,
    ``transcribe_batch`` runs wav -> encoder -> ctc_lin -> per-frame arg-max on the device (one fused pipeline + the CTC head
    GEMM + ``rows_logsoftmax_argmax_kernel``) and the CTC merge / blank filter on the host.

    ``modules["encoder"]``: ``LengthsCapableSequential`` of Fbank, InputNormalization, ConvolutionFrontEnd,
    ``EncoderWrapper(TransformerASR)``, the CTC ``Linear`` and a log-softmax (``torch.nn.LogSoftmax`` /
    ``speechbrain_b200.nnet.activations.Softmax(apply_log=True)``); ``hparams["decoding_function"]`` is a
    ``functools.partial`` of ``ctc_greedy_decode`` or the ``CTCBeamSearcher`` / ``CTCPrefixBeamSearcher`` class
    (inference/ASR.py:212-282), which is instantiated with ``hparams["test_beam_search"]`` (or no keywords) and the
    tokenizer's vocabulary; the log-posteriors then stay on the device and go to the beam search kernel (csrc/ctc_beam.cu,
    csrc/ctc_prefix_beam.cu).  TorchAudioCTCPrefixBeamSearch is not built."""
    HPARAMS_NEEDED = ["tokenizer", "decoding_function"]
    MODULES_NEEDED = ["encoder"]

    def __init__(self, modules=None, hparams=None, run_opts=None, freeze_params=True):
        super().__init__()
        import functools

        from ..decoders.ctc import CTCBaseSearcher, ctc_greedy_decode
        from ..nnet.linear import Linear
        modules = dict(modules or {})
        if "encoder" not in modules:
            raise ValueError("Need modules['encoder']")
        self.mods = torch.nn.ModuleDict(modules)
        self.hparams = dict(hparams) if isinstance(hparams, dict) else (dict(vars(hparams)) if hparams is not None else {})
        for k in self.HPARAMS_NEEDED:
            if k not in self.hparams:
                raise ValueError(f"Need hparams['{k}']")
        self.tokenizer = self.hparams["tokenizer"]
        fn = self.hparams["decoding_function"]
        self.beam_search = isinstance(fn, type) and issubclass(fn, CTCBaseSearcher)
        if self.beam_search:
            opts = dict(self.hparams.get("test_beam_search") or {})
            self.decoding_function = fn(**opts, vocab_list=self._vocab_list())
        elif isinstance(fn, functools.partial) and fn.func is ctc_greedy_decode:
            self.decoding_function = fn
            self.blank_id = fn.keywords.get("blank_id", -1)
        else:
            raise NotImplementedError("speechbrain_b200.EncoderASR: decoding_function must be functools.partial(ctc_greedy_decode, "
                                      "blank_id=...), CTCBeamSearcher or CTCPrefixBeamSearcher (TorchAudioCTCPrefixBeamSearch "
                                      "is not built)")
        self.device = torch.device((run_opts or {}).get("device", "cuda:0"))
        vals = list(self.mods.values())
        wrap = _find(vals, EncoderWrapper)
        tr = _find(vals, TransformerASR) or (wrap.transformer if wrap is not None else None)
        for name, m in (("fbank", _find(vals, Fbank)), ("normalize", _find(vals, InputNormalization)),
                        ("cnn", _find(vals, ConvolutionFrontEnd)), ("transformer", tr), ("ctc_lin", _find(vals, Linear))):
            if m is None:
                raise ValueError(f"EncoderASR: could not find the {name} module in modules['encoder']")
            object.__setattr__(self, name, m)
        if self.normalize.norm_type != "global":
            raise NotImplementedError("EncoderASR: fused pipeline needs InputNormalization(norm_type='global')")

    def _vocab_list(self):
        """inference/ASR.py:240-255: the beam searcher's vocab_list from a sentencepiece model or a label encoder."""
        tok = self.tokenizer
        try:
            import sentencepiece
        except ImportError:
            sentencepiece = None
        if sentencepiece is not None and isinstance(tok, sentencepiece.SentencePieceProcessor):
            return [tok.id_to_piece(i) for i in range(tok.vocab_size())]
        if hasattr(tok, "ind2lab"):
            return [tok.ind2lab[i] for i in range(len(tok.ind2lab))]
        raise ValueError("The tokenizer must be sentencepiece or CTCTextEncoder")

    @classmethod
    def from_hparams(cls, source, hparams_file="hyperparams.yaml", overrides=None, savedir=None, run_opts=None, **kwargs):
        from ..utils.hparams import load_pretrained_interface
        return load_pretrained_interface(cls, source, hparams_file, overrides or {}, run_opts or {})

    def engine(self):
        src = {"fbank": self.fbank, "normalize": self.normalize, "CNN.": self.cnn, "ctc_lin.": self.ctc_lin}
        return self.transformer.engine_slot(("ctc", id(self.ctc_lin))).get(self.device, ("fbank", "cnn", "encoder"), src)

    def _encode(self, wavs, wav_lens):
        eng = self.engine()
        wavs = wavs.float().to(self.device)
        enc = eng.encode_wav(wavs, wav_lens.to(self.device))
        return eng, enc

    @torch.no_grad()
    def encode_batch(self, wavs, wav_lens):
        """inference/ASR.py:297-323: -> log-posteriors [B, T, V]."""
        eng, enc = self._encode(wavs, wav_lens)
        lp, _ = eng.ctc_head(enc, want_log_probs=True, want_argmax=False)
        return lp

    @torch.no_grad()
    def transcribe_batch(self, wavs, wav_lens):
        """inference/ASR.py:325-373: -> (predicted_words, predicted_tokens); with a CTC beam searcher
        -> ([best text per utterance], the searcher's List[List[CTCHypothesis]])."""
        from ..decoders.ctc import greedy_from_argmax
        eng, enc = self._encode(wavs, wav_lens)
        if self.beam_search:
            lp, _ = eng.ctc_head(enc, want_log_probs=True, want_argmax=False)
            hyps = self.decoding_function(lp, wav_lens.to(self.device))
            return [h[0].text for h in hyps], hyps
        _, idx = eng.ctc_head(enc, want_log_probs=False, want_argmax=True)
        V = eng.cfg["vocab"]
        blank = self.blank_id + V if isinstance(self.blank_id, int) and self.blank_id < 0 else self.blank_id
        predictions = greedy_from_argmax(idx.cpu(), wav_lens, blank)
        if self.tokenizer is not None:
            words = [self.tokenizer.decode_ids(t) for t in predictions]
        else:
            words = [" ".join(map(str, t)) for t in predictions]
        return words, predictions

    def forward(self, wavs, wav_lens):
        """Runs the encoder (the reference's forward returns encode_batch)."""
        return self.encode_batch(wavs, wav_lens)


@dataclass
class ASRStreamingContext:
    """inference/ASR.py:947-975: the mutable state of one streaming session, passed to every chunk call."""

    config: Any
    """The DynChunkTrainConfig the context was made for."""
    fea_extractor_context: Any
    """StreamingFeatureWrapperContext, bound to the encoder context's device stream (which holds the audio context)."""
    encoder_context: Any
    """TransformerASRStreamingContext: per-layer device caches."""
    decoder_context: Any
    """The decoder's streaming context (TransducerGreedySearcherStreamingContext)."""
    tokenizer_context: Optional[List[Any]] = None
    """One detokeniser context per row, made by the first ``decode_chunk``."""


class StreamingASR(torch.nn.Module):
    """Drop-in for speechbrain.inference.ASR.StreamingASR (inference/ASR.py:978-1363): audio chunks to text for the
    streaming Conformer-Transducer.

    Per chunk, on the caller's stream: the feature wrapper's device front end over [audio context | chunk]
    (``sbk_asr_stream_frontend_chunk``), the encoder on its per-layer device caches (``enc.forward_streaming``), ``proj_enc``
    on the wgmma GEMM and the greedy transducer kernel carrying ``(out_PN, (h, c))``; the tokens then come to the host
    for the SentencePiece detokeniser.  ``hparams`` as the recipe's inference block builds them: ``fea_streaming_extractor``
    (a ``StreamingFeatureWrapper`` over Fbank, global InputNormalization and the ConvolutionFrontEnd),
    ``make_decoder_streaming_context``, ``decoding_function`` (``TransducerBeamSearcher.transducer_greedy_decode_streaming``
    bound to a greedy searcher), ``make_tokenizer_streaming_context``, ``tokenizer_decode_streaming`` and ``tokenizer``.

    The B rows of a batch advance together, and only the last chunk of a stream may be shorter than
    ``get_chunk_size_frames``: to flush a stream, append the recommended zero chunks to its audio before splitting it.
    ``transcribe_file`` / ``transcribe_file_streaming`` need audio file decoding, which is not built."""
    HPARAMS_NEEDED = ["fea_streaming_extractor", "make_decoder_streaming_context", "decoding_function",
                      "make_tokenizer_streaming_context", "tokenizer_decode_streaming"]
    MODULES_NEEDED = ["enc", "proj_enc"]

    def __init__(self, modules=None, hparams=None, run_opts=None, freeze_params=True):
        super().__init__()
        from ..lobes.features import StreamingFeatureWrapper
        from ..nnet.linear import Linear
        modules = dict(modules or {})
        for k in self.MODULES_NEEDED:
            if k not in modules:
                raise ValueError(f"Need modules['{k}']")
        self.mods = torch.nn.ModuleDict(modules)
        hp = dict(hparams) if isinstance(hparams, dict) else (dict(vars(hparams)) if hparams is not None else {})
        for k in self.HPARAMS_NEEDED:
            if k not in hp:
                raise ValueError(f"Need hparams['{k}']")
        self.hparams = types.SimpleNamespace(**hp)
        if not isinstance(self.mods["enc"], EncoderWrapper):
            raise NotImplementedError("speechbrain_b200.StreamingASR: modules['enc'] must be an EncoderWrapper(TransformerASR)")
        if not isinstance(self.mods["proj_enc"], Linear):
            raise NotImplementedError("speechbrain_b200.StreamingASR: modules['proj_enc'] must be a speechbrain_b200 Linear")
        fea = self.hparams.fea_streaming_extractor
        if not isinstance(fea, StreamingFeatureWrapper):
            raise NotImplementedError("speechbrain_b200.StreamingASR: fea_streaming_extractor must be a speechbrain_b200 "
                                      "StreamingFeatureWrapper")
        self.filter_props = fea.properties
        self.device = torch.device((run_opts or {}).get("device", "cuda:0"))
        object.__setattr__(self, "_slot", self.mods["enc"].transformer.engine_slot(("streaming", id(fea))))

    @classmethod
    def from_hparams(cls, source, hparams_file="hyperparams.yaml", overrides=None, savedir=None, run_opts=None, **kwargs):
        """Loads a LOCAL directory in the layout of the recipe's inference hparams (see EncoderDecoderASR.from_hparams)."""
        from ..utils.hparams import load_pretrained_interface
        return load_pretrained_interface(cls, source, hparams_file, overrides or {}, run_opts or {})

    def engine(self):
        """The engine holding this model's front end and encoder: the one the streams run on."""
        fea = self.hparams.fea_streaming_extractor
        return self._slot.get(self.device, ("fbank", "cnn", "encoder"),
                              {"fbank": fea.fbank, "normalize": fea.normalize, "CNN.": fea.cnn})

    def transcribe_file_streaming(self, path, dynchunktrain_config, use_torchaudio_streaming=True, **kwargs):
        raise NotImplementedError("speechbrain_b200.StreamingASR: audio file decoding is not built (this torchaudio has no "
                                  "torchaudio.io); load the audio yourself and call transcribe_chunk per chunk")

    def transcribe_file(self, path, dynchunktrain_config, use_torchaudio_streaming=True):
        raise NotImplementedError("speechbrain_b200.StreamingASR: audio file decoding is not built (this torchaudio has no "
                                  "torchaudio.io); load the audio yourself and call transcribe_chunk per chunk")

    def make_streaming_context(self, dynchunktrain_config):
        enc_ctx = self.mods["enc"].make_streaming_context(dynchunktrain_config)
        enc_ctx.encoder_context.slot = self._slot
        fea_ctx = self.hparams.fea_streaming_extractor.make_streaming_context()
        fea_ctx.stream_owner = enc_ctx.encoder_context
        return ASRStreamingContext(config=dynchunktrain_config, fea_extractor_context=fea_ctx, encoder_context=enc_ctx,
                                   decoder_context=self.hparams.make_decoder_streaming_context(), tokenizer_context=None)

    def get_chunk_size_frames(self, dynchunktrain_config) -> int:
        """Samples per chunk, (stride - 1) * chunk_size, as the reference computes it."""
        return (self.filter_props.stride - 1) * dynchunktrain_config.chunk_size

    @torch.no_grad()
    def encode_chunk(self, context, chunk, chunk_len=None):
        """chunk [B, n_samples <= get_chunk_size_frames] -> proj_enc(encoder output) [B, frames, joint]."""
        if chunk_len is None:
            chunk_len = torch.ones((chunk.size(0),))
        if chunk.dim() != 2 or chunk.shape[-1] > self.get_chunk_size_frames(context.config):
            raise ValueError(f"StreamingASR.encode_chunk: a chunk of shape {tuple(chunk.shape)}; expected [batch, <= "
                             f"{self.get_chunk_size_frames(context.config)}] samples")
        # chunk_len stays where it is: with global statistics in eval mode it changes no value (see the wrapper)
        chunk = chunk.float().to(self.device)
        context.encoder_context.encoder_context.ensure_stream(self.engine(), chunk.shape[0])
        x = self.hparams.fea_streaming_extractor(chunk, context=context.fea_extractor_context, lengths=chunk_len)
        x = self.mods["enc"].forward_streaming(x, context.encoder_context)
        return self.mods["proj_enc"](x)

    @torch.no_grad()
    def decode_chunk(self, context, x):
        """-> (text per row for this chunk, tokens per row)."""
        tokens = self.hparams.decoding_function(x, context.decoder_context)
        if context.tokenizer_context is None:
            context.tokenizer_context = [self.hparams.make_tokenizer_streaming_context() for _ in range(len(tokens))]
        words = [self.hparams.tokenizer_decode_streaming(self.hparams.tokenizer, cur_tokens, context.tokenizer_context[i])
                 for i, cur_tokens in enumerate(tokens)]
        return words, tokens

    def transcribe_chunk(self, context, chunk, chunk_len=None):
        """The text of one more chunk of every row (possibly empty strings)."""
        if chunk_len is None:
            chunk_len = torch.ones((chunk.size(0),))
        x = self.encode_chunk(context, chunk, chunk_len)
        words, _ = self.decode_chunk(context, x)
        return words
