"""ConvolutionFrontEnd -- drop-in for speechbrain.lobes.models.convolution.ConvolutionFrontEnd
(lobes/models/convolution.py:116-320) for the two configurations the recipes use:
- the Conformer recipes': 2 blocks x 1 Conv2d(3x3, stride 2, reflect 'same' padding) + LayerNorm + LeakyReLU, no residuals,
  out_channels (64, 32), and the AISHELL-1 Transformer recipe's, the same blocks with out_channels (256, 256);
- the Transformer recipes': 3 blocks x 1 layer, out_channels (64, 64, 64), kernel_sizes (5, 5, 1), strides (2, 2, 1),
  residuals (False, False, True): the third block adds a 1x1 Conv2d + LayerNorm (reduce_conv) of its input.
Same constructor and state_dict keys; other configurations raise (no CPU fallback)."""
import torch

from ..._lib import require_cuda
from ...utils.filter_analysis import FilterProperties, stack_filter_properties
from ...utils.param_tree import build_param_tree, default_init
from ...utils.shapes import cnn3_frontend_shapes, cnn_frontend_shapes


class ConvolutionFrontEnd(torch.nn.Module):
    def __init__(self, input_shape, num_blocks=3, num_layers_per_block=5, out_channels=(128, 256, 512),
                 kernel_sizes=(3, 3, 3), strides=(1, 2, 2), dilations=(1, 1, 1), residuals=(True, True, True),
                 conv_module=None, activation=torch.nn.LeakyReLU, norm="LayerNorm", dropout=0.1, conv_bias=True,
                 padding="same", conv_init=None):
        super().__init__()
        common = (num_layers_per_block == 1 and conv_module is None and activation is torch.nn.LeakyReLU
                  and norm == "LayerNorm" and conv_bias and padding == "same")
        conformer = (common and num_blocks == 2 and tuple(kernel_sizes[:2]) == (3, 3) and tuple(strides[:2]) == (2, 2)
                     and not any(residuals[:2]) and tuple(dilations[:2]) == (1, 1)
                     and tuple(out_channels[:2]) in ((64, 32), (256, 256)))
        transformer = (common and num_blocks == 3 and tuple(kernel_sizes[:3]) == (5, 5, 1)
                       and tuple(strides[:3]) == (2, 2, 1) and tuple(bool(r) for r in residuals[:3]) == (False, False, True)
                       and tuple(dilations[:3]) == (1, 1, 1) and tuple(out_channels[:3]) == (64, 64, 64))
        if not (conformer or transformer):
            raise NotImplementedError(
                "speechbrain_b200.ConvolutionFrontEnd: only the Conformer recipes' front-end (num_blocks=2, "
                "num_layers_per_block=1, out_channels=(64, 32), 3x3, stride 2, no residuals), the same with "
                "out_channels=(256, 256) (AISHELL-1's Transformer) and the LibriSpeech Transformer recipes' "
                "(num_blocks=3, num_layers_per_block=1, out_channels=(64, 64, 64), kernel_sizes=(5, 5, 1), strides=(2, 2, 1), "
                "residuals=(False, False, True)) are built")
        self.n_mels = int(input_shape[-1])
        self.num_blocks = num_blocks
        # one Conv2d per block: its (kernel, stride) along time (ConvBlock.filter_properties, convolution.py:283-289)
        self._block_filters = [FilterProperties(window_size=k, stride=s)
                               for k, s in zip(kernel_sizes[:num_blocks], strides[:num_blocks])]
        self.out_channels = tuple(out_channels[:2])
        shapes = cnn3_frontend_shapes(self.n_mels) if transformer else cnn_frontend_shapes(self.n_mels, self.out_channels)
        build_param_tree(self, shapes, default_init)
        object.__setattr__(self, "_slot", None)

    def get_filter_properties(self):
        """The blocks' filters stacked (convolution.py:200-203, 319-320)."""
        return stack_filter_properties(self._block_filters)

    def _engine_cfg(self):
        f2 = ((self.n_mels - 1) // 2 + 1 - 1) // 2 + 1
        return dict(n_fft=400, hop=160, win=400, n_mels=self.n_mels, cnn_channels=self.out_channels,
                    input_size=f2 * self.out_channels[1], d_model=64, nhead=1, num_encoder_layers=0,
                    num_decoder_layers=0, d_ffn=64, vocab=8, attention_type="RoPEMHA", cnn_blocks=self.num_blocks)

    def _get_engine(self, device):
        """Stand-alone use (module-by-module pipelines): a CNN-only engine, rebuilt when the parameters change."""
        if self._slot is None:
            from ...engine_cache import EngineSlot
            object.__setattr__(self, "_slot", EngineSlot(self._engine_cfg))
        return self._slot.get(device, ("cnn",), {"CNN.": self})

    @torch.no_grad()
    def forward(self, x):
        """x [B, T, F] -> [B, T', F', C] (channels-last, like the reference)."""
        require_cuda(x, "ConvolutionFrontEnd")
        if x.dim() != 3:
            raise NotImplementedError("ConvolutionFrontEnd: expected [batch, time, features]")
        out = self._get_engine(x.device).cnn(x)
        B, T2, _ = out.shape
        return out.reshape(B, T2, -1, self.out_channels[1])
