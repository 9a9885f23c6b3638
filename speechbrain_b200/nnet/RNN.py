"""LSTM -- drop-in for speechbrain.nnet.RNN.LSTM (nnet/RNN.py:180-302): keys ``rnn.weight_ih_l0`` / ``rnn.weight_hh_l0`` /
``rnn.bias_ih_l0`` / ``rnn.bias_hh_l0`` (a batch-first ``torch.nn.LSTM`` under ``rnn``).

Only the transducer prediction network runs it, inside the greedy search kernel (decoders/transducer.py), and only as one
unidirectional layer with biases.  GRU, RNN and LiGRU have no mirror."""
import torch


class MissingInputSizeError(ValueError, NotImplementedError):
    """Raised when neither ``input_shape`` nor ``input_size`` is given.  The reference raises ``ValueError`` here, so
    code written against it keeps catching it; it is also a ``NotImplementedError`` because a recurrent layer built
    without its input size is not something this package can run, which is what configuration loaders catch for
    unsupported objects."""


class LSTM(torch.nn.Module):
    def __init__(self, hidden_size, input_shape=None, input_size=None, num_layers=1, bias=True, dropout=0.0, re_init=True,
                 bidirectional=False):
        super().__init__()
        if input_shape is None and input_size is None:
            raise MissingInputSizeError("Expected one of input_shape or input_size.")
        self.reshape = False
        if input_size is None:
            if len(input_shape) > 3:
                self.reshape = True
            input_size = int(torch.prod(torch.tensor(input_shape[2:])).item())
        self.rnn = torch.nn.LSTM(input_size=input_size, hidden_size=hidden_size, num_layers=num_layers, dropout=dropout,
                                 bidirectional=bidirectional, bias=bias, batch_first=True)
        for p in self.parameters():
            p.requires_grad_(False)

    def forward(self, x, hx=None, lengths=None):
        raise NotImplementedError("speechbrain_b200.LSTM: runs only as the transducer prediction network, inside "
                                  "TransducerBeamSearcher's search kernel")
