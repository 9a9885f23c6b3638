"""speechbrain.nnet.activations.Softmax and Swish mirrors (nnet/activations.py:20-87, 133-167): the recipes end their CTC
branch with ``Softmax(apply_log=True)``.  Inside EncoderASR the log-softmax is fused into the CTC head kernel; called on its
own this module runs torch's (log_)softmax on the tensor's device (plumbing, not part of the timed path).  ``Swish`` names the
Conformer and decoder FFN activation in the recipe YAMLs (``activation: !name:speechbrain.nnet.activations.Swish``); the
device kernels compute it in their GEMM epilogues."""
import torch


class Softmax(torch.nn.Module):
    def __init__(self, apply_log=False, dim=-1, reshape=True, dtype=torch.float32):
        super().__init__()
        self.apply_log, self.dim, self.dtype = apply_log, dim, dtype

    def forward(self, x):
        return torch.log_softmax(x, self.dim, dtype=self.dtype) if self.apply_log else torch.softmax(x, self.dim, dtype=self.dtype)


class Swish(torch.nn.Module):
    """silu(beta * x), as the reference computes it; the device kernels build beta = 1 (SiLU), the only value the recipes
    use (TransformerASR takes the class, so the default)."""

    def __init__(self, beta=1.0):
        super().__init__()
        self.beta = beta

    def forward(self, x):
        return torch.nn.functional.silu(self.beta * x)
