"""Linear -- drop-in for speechbrain.nnet.linear.Linear (nnet/linear.py:16-91): keys ``w.weight`` / ``w.bias``.
On CUDA the product runs on the wgmma GEMM (fp16 operands, fp32 accumulate)."""
import torch

from .._lib import check, lib, ptr, require_cuda, stream_ptr


class Linear(torch.nn.Module):
    def __init__(self, n_neurons, input_shape=None, input_size=None, bias=True, max_norm=None, combine_dims=False):
        super().__init__()
        if max_norm is not None:
            raise NotImplementedError("speechbrain_b200.Linear: max_norm is a training-time feature")
        if input_shape is None and input_size is None:
            raise ValueError("Expected one of input_shape or input_size")
        self.combine_dims = combine_dims
        if input_size is None:
            input_size = input_shape[-1]
            if len(input_shape) == 4 and combine_dims:
                input_size = input_shape[2] * input_shape[3]
        self.w = torch.nn.Linear(input_size, n_neurons, bias=bias)
        for p in self.parameters():
            p.requires_grad_(False)
        self._w16 = None
        self._fp = None

    @torch.no_grad()
    def forward(self, x):
        require_cuda(x, "Linear")
        if x.ndim == 4 and self.combine_dims:
            x = x.reshape(x.shape[0], x.shape[1], x.shape[2] * x.shape[3])
        K, N = self.w.in_features, self.w.out_features
        if K % 8 != 0:
            raise NotImplementedError("speechbrain_b200.Linear: input_size must be a multiple of 8 (TMA row pitch)")
        # fp16 operand snapshot, refreshed whenever the parameters change (load_state_dict / .to() / in-place ops)
        fp = tuple((t.data_ptr(), t._version) for t in self.w.parameters()) + (str(x.device),)
        if self._w16 is None or self._fp != fp:
            self._w16 = self.w.weight.detach().to(x.device, torch.float16).contiguous()
            self._b32 = self.w.bias.detach().to(x.device, torch.float32).contiguous() if self.w.bias is not None else None
            self._fp = fp
        a = x.reshape(-1, K).to(torch.float16).contiguous()
        out = torch.empty(a.shape[0], N, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            check(lib().sbk_gemm_f16_test(ptr(a), ptr(self._w16), ptr(self._b32), ptr(out), 1, 0, a.shape[0], N, K,
                                          stream_ptr(x.device)), "sbk_gemm_f16")
        return out.reshape(*x.shape[:-1], N)
