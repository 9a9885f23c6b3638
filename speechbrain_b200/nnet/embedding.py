"""Embedding -- drop-in for speechbrain.nnet.embedding.Embedding (nnet/embedding.py:14-121): key ``Embedding.weight``.

It holds the parameters only.  Its one use on the device is the transducer prediction network, where the lookup is
folded into the input table ``U[v] = W_ih E[v] + b_ih + b_hh`` the search kernel reads (decoders/transducer.py)."""
import torch


class Embedding(torch.nn.Module):
    def __init__(self, num_embeddings, embedding_dim=128, consider_as_one_hot=False, blank_id=0):
        super().__init__()
        self.num_embeddings = num_embeddings
        self.consider_as_one_hot = consider_as_one_hot
        self.embedding_dim = num_embeddings - 1 if consider_as_one_hot else embedding_dim
        self.blank_id = blank_id
        if consider_as_one_hot:
            # the reference's fixed shifted identity: token v > blank -> e_{v-1}, v < blank -> e_v, blank -> 0
            self.Embedding = torch.nn.Embedding(num_embeddings, self.embedding_dim, padding_idx=blank_id)
            one_hot = torch.eye(self.embedding_dim)
            with torch.no_grad():
                if blank_id + 1 != num_embeddings:
                    self.Embedding.weight[blank_id + 1:] = one_hot[blank_id:]
                if blank_id != 0:
                    self.Embedding.weight[:blank_id] = one_hot[:blank_id]
        else:
            self.Embedding = torch.nn.Embedding(num_embeddings, self.embedding_dim)
        for p in self.parameters():
            p.requires_grad_(False)

    def forward(self, x):
        raise NotImplementedError("speechbrain_b200.Embedding: the lookup runs inside the transducer search kernel "
                                  "(TransducerBeamSearcher); there is no standalone forward")
