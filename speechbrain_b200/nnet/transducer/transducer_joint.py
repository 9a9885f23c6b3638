"""Transducer_joint -- drop-in for speechbrain.nnet.transducer.transducer_joint.Transducer_joint
(nnet/transducer/transducer_joint.py:13-103) as the transducer recipes build it: ``joint="sum"``, no joint network,
``nonlinearity=torch.nn.GELU``.  The joint runs inside the transducer search kernel (decoders/transducer.py) as
GELU(tn + out_PN) with the exact erf form; other joints raise NotImplementedError at construction."""
import torch


class Transducer_joint(torch.nn.Module):
    def __init__(self, joint_network=None, joint="sum", nonlinearity=torch.nn.LeakyReLU):
        super().__init__()
        if joint != "sum":
            raise NotImplementedError(f"speechbrain_b200.Transducer_joint: joint={joint!r} is not built (only 'sum')")
        if joint_network is not None:
            raise NotImplementedError("speechbrain_b200.Transducer_joint: a joint_network is not built")
        self.joint_network = joint_network
        self.joint = joint
        self.nonlinearity = nonlinearity()
        if type(self.nonlinearity) is not torch.nn.GELU or self.nonlinearity.approximate != "none":
            raise NotImplementedError("speechbrain_b200.Transducer_joint: only nonlinearity=torch.nn.GELU (erf form) is built")

    def forward(self, input_TN, input_PN):
        raise NotImplementedError("speechbrain_b200.Transducer_joint: the joint runs inside TransducerBeamSearcher's "
                                  "search kernel")
