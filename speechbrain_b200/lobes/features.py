"""Fbank -- drop-in for speechbrain.lobes.features.Fbank (lobes/features.py:22-173) on the sm_90a kernel.

Same constructor, ``forward(wav) -> [B, T_f, n_mels]`` and ``state_dict`` keys ({"compute_deltas.kernel"}).
Built natively: frozen triangular filters, no deltas, no context, mono [B, L] input -- i.e. what every ASR
recipe on the hot path uses (conformer_{small,large}.yaml).  Anything else raises (there is no CPU fallback).
"""
import torch

from .._lib import require_cuda
from ..engine import FbankHandle, mel_filter_matrix, stft_window


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
        """(window_size, stride) of the STFT, as processing/features.py:190-198 reports them."""
        if self.n_fft % 2 == 0:
            raise ValueError("Cannot determine the filter properties of an even-sized window STFT")
        return {"window_size": self.n_fft, "stride": self.hop_length}
