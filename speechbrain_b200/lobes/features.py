"""Fbank -- drop-in for speechbrain.lobes.features.Fbank (lobes/features.py:22-173) on the sm_90a kernel.

Same constructor, ``forward(wav) -> [B, T_f, n_mels]`` and ``state_dict`` keys ({"compute_deltas.kernel"}).
Built natively: frozen triangular filters, no deltas, no context, mono [B, L] input -- i.e. what every ASR
recipe on the hot path uses (conformer_{small,large}.yaml).  Anything else raises (there is no CPU fallback).
"""
from dataclasses import dataclass
from typing import Any, Optional

import torch

from .._lib import require_cuda
from ..engine import FbankHandle, mel_filter_matrix, stft_window
from ..utils.filter_analysis import FilterProperties, upalign_value  # noqa: F401  (upalign_value: the reference's home)


class _DeltasBuffer(torch.nn.Module):
    """Only carries the ``kernel`` buffer so state_dict keys match (processing/features.py:857-869)."""

    def __init__(self, input_size, window_length=5):
        super().__init__()
        n = (window_length - 1) // 2
        self.register_buffer("kernel", torch.arange(-n, n + 1, dtype=torch.float32).repeat(input_size, 1, 1))


class Fbank(torch.nn.Module):
    def __init__(self, deltas=False, context=False, requires_grad=False, sample_rate=16000, f_min=0, f_max=None,
                 n_fft=400, n_mels=40, filter_shape="triangular", param_change_factor=1.0, param_rand_factor=0.0,
                 left_frames=5, right_frames=5, win_length=25, hop_length=10):
        super().__init__()
        if deltas or context:
            raise NotImplementedError("speechbrain_b200.Fbank: deltas/context are not on the H100 hot path")
        if requires_grad:
            raise NotImplementedError("speechbrain_b200.Fbank: learnable filters are not supported (inference only)")
        if filter_shape != "triangular":
            raise NotImplementedError(f"speechbrain_b200.Fbank: filter_shape={filter_shape!r} is not built")
        self.deltas, self.context, self.requires_grad = deltas, context, requires_grad
        if f_max is None:
            f_max = sample_rate // 2
        if f_min >= f_max:
            raise ValueError("Require f_min: %f < f_max: %f" % (f_min, f_max))
        self.sample_rate, self.n_fft, self.n_mels = sample_rate, n_fft, n_mels
        # ms -> samples exactly like STFT.__init__ (processing/features.py:132-137)
        self.win_length = int(round((sample_rate / 1000.0) * win_length))
        self.hop_length = int(round((sample_rate / 1000.0) * hop_length))
        if self.win_length > n_fft:
            raise ValueError("win_length (in samples) must be <= n_fft")  # torch.stft raises too
        self._window = stft_window(n_fft, self.win_length)
        self._mel = mel_filter_matrix(n_mels, n_fft, sample_rate, f_min, f_max)
        self.compute_deltas = _DeltasBuffer(input_size=n_mels)
        self._handle = None

    def _get_handle(self):
        if self._handle is None:
            self._handle = FbankHandle(self.n_fft, self.hop_length, self.n_mels, self._window, self._mel)
        return self._handle

    @torch.no_grad()
    def forward(self, wav):
        """wav [B, L] (any float dtype; computed in fp32 like the reference's fwd_default_precision decorator)."""
        if wav.dim() != 2:
            raise NotImplementedError("speechbrain_b200.Fbank: only mono [batch, time] input is built")
        require_cuda(wav, "Fbank")
        return self._get_handle().forward(wav)

    def get_filter_properties(self):
        """The centred STFT's window and hop in samples (lobes/features.py:171-173, processing/features.py:190-198)."""
        return FilterProperties(window_size=self.win_length, stride=self.hop_length)


@dataclass
class StreamingFeatureWrapperContext:
    """lobes/features.py:495-505.  ``left_context`` is None before the first chunk and then True: the carried samples
    themselves stay on the device, in ``stream`` (the ``EncoderStream`` of the streaming encoder context this context
    is bound to by ``StreamingASR.make_streaming_context``)."""

    left_context: Optional[bool] = None
    stream_owner: Any = None  # a ConformerEncoderStreamingContext: its ``stream`` holds the audio context


class StreamingFeatureWrapper(torch.nn.Module):
    """StreamingFeatureWrapper (lobes/features.py:508-670): runs a filter chunk by chunk, each chunk behind the last
    2 * pad samples of the previous window (zeros before the first), and trims pad / stride output frames off each side,
    with pad = upalign((window_size - 1) // 2, stride).

    Built for one module: ``LengthsCapableSequential(Fbank, InputNormalization(norm_type="global"), ConvolutionFrontEnd)``
    (the streaming Conformer-Transducer recipe's).  The window is assembled and the fused Fbank + CMVN and front-end
    kernels run over it on the device (``sbk_asr_stream_frontend_chunk``), so the STFT's centre padding, the top_db clamp
    and the CNN's reflect padding are those of the whole window, as in the reference.  With global statistics in eval
    mode ``lengths`` changes no value (the reference also normalises the padded samples), so it is accepted and unused."""

    def __init__(self, module, properties):
        super().__init__()
        self.module = module
        self.properties = properties
        if self.properties.causal:
            raise ValueError("Causal streaming feature wrapper is not yet supported")
        if self.properties.dilation != 1:
            raise ValueError("Dilation not yet supported in streaming feature wrapper")
        from ..lobes.models.convolution import ConvolutionFrontEnd
        from ..nnet.containers import LengthsCapableSequential
        from ..processing.features import InputNormalization
        parts = list(module.values()) if isinstance(module, LengthsCapableSequential) else []
        if (len(parts) != 3 or not isinstance(parts[0], Fbank) or not isinstance(parts[1], InputNormalization)
                or parts[1].norm_type != "global" or not isinstance(parts[2], ConvolutionFrontEnd)):
            raise NotImplementedError("speechbrain_b200.StreamingFeatureWrapper: the module must be LengthsCapableSequential("
                                      "Fbank, InputNormalization(norm_type='global'), ConvolutionFrontEnd)")
        self.fbank, self.normalize, self.cnn = parts
        # the device trims pad / (hop * 4) frames: properties that are not this module's would trim differently
        if self.properties.stride != 4 * self.fbank.hop_length:
            raise ValueError(f"StreamingFeatureWrapper: properties.stride={self.properties.stride}, but the module's stride "
                             f"is {4 * self.fbank.hop_length} (Fbank hop x the front end's two stride-2 blocks)")

    def get_required_padding(self) -> int:
        return upalign_value((self.properties.window_size - 1) // 2, self.properties.stride)

    def get_output_count_per_pad_frame(self) -> int:
        return self.get_required_padding() // self.properties.stride

    def get_recommended_final_chunk_count(self, frames_per_chunk: int) -> int:
        return upalign_value(self.get_required_padding(), frames_per_chunk) // frames_per_chunk

    @torch.no_grad()
    def forward(self, chunk, context, *extra_args, lengths=None, **extra_kwargs):
        """chunk [B, n_samples] on the device -> features [B, frames, input_size]: a view of the window's front-end output
        (the frames the reference keeps after trimming), enqueued on the current stream."""
        del extra_args, extra_kwargs, lengths
        require_cuda(chunk, "StreamingFeatureWrapper")
        owner = context.stream_owner
        if owner is None or owner.stream is None:
            raise RuntimeError("StreamingFeatureWrapper: the device front end keeps its audio context in a streaming "
                               "encoder's device stream; use a context from StreamingASR.make_streaming_context")
        if chunk.dim() != 2:
            raise ValueError(f"StreamingFeatureWrapper: expected a [batch, time] chunk, got {tuple(chunk.shape)}")
        out, trim, n = owner.stream.frontend_chunk(chunk, self.get_required_padding())
        context.left_context = owner.started = True
        return out[:, trim:trim + n]

    def get_filter_properties(self):
        return self.properties

    def make_streaming_context(self):
        return StreamingFeatureWrapperContext(None)
