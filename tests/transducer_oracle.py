"""fp32 CPU restatement of TransducerBeamSearcher.transducer_greedy_decode (speechbrain/decoders/transducer.py:156-291)
for the Conformer-Transducer recipes' prediction network (one-hot Embedding -> 1-layer LSTM -> Linear(bias=False)), joint
GELU(tn + out_PN) and classifier Linear(bias=False) + log-softmax.

Rows of the reference's batched loop are independent, so the oracle walks each row on its own.  ``forced`` walks a row
along a given decision path (the device's tokens and the frames they were emitted at) instead of its own arg-max, and
every decision reports the chosen log-prob, the arg-max and the top-two log-probs, so a test can judge a differing
decision by the reference margin.  Also: the seeded recipe-shaped weights and tn_output the fixture and the GPU tests use."""
import math

import torch

# (joint_dim, dec_dim, V) of conformer_transducer.yaml: LibriSpeech, CommonVoice / GigaSpeech, VoxPopuli
RECIPE_SIZES = {"librispeech": (640, 512, 1000), "commonvoice": (512, 512, 1024), "voxpopuli": (512, 512, 512)}


def one_hot_embedding(V, blank):
    """nnet/embedding.py:84-101 with consider_as_one_hot=True: [V, V-1], blank row zero."""
    w = torch.zeros(V, V - 1)
    eye = torch.eye(V - 1)
    if blank + 1 != V:
        w[blank + 1:] = eye[blank:]
    if blank != 0:
        w[:blank] = eye[:blank]
    return w


def seeded_weights(seed, J, H, V, blank, blank_gain=2.0, out_gain=3.0, pd_gain=8.0):
    """Recipe-keyed state (module prefixes emb / dec / proj_dec / transducer_lin).  Xavier-like seeded matrices; the
    classifier is scaled by ``out_gain`` and its blank row gets ``blank_gain`` / sqrt(J) added to every entry, so blank wins
    unless tn_output points at a token (see seeded_tn): the search then emits 0, 1 or several tokens per frame, as a
    trained model does, instead of all-blank or all-emit.  The prediction-network projection is scaled by ``pd_gain`` so
    the emitted tokens move the joint."""
    g = torch.Generator().manual_seed(seed)

    def xavier(o, i):
        return math.sqrt(2.0 / (o + i)) * torch.randn(o, i, generator=g)
    out = xavier(V, J) * out_gain
    out[blank] += blank_gain / math.sqrt(J)
    return {
        "emb.Embedding.weight": one_hot_embedding(V, blank),
        "dec.rnn.weight_ih_l0": xavier(4 * H, V - 1) * 4.0,
        "dec.rnn.weight_hh_l0": xavier(4 * H, H),
        "dec.rnn.bias_ih_l0": 0.05 * torch.randn(4 * H, generator=g),
        "dec.rnn.bias_hh_l0": 0.05 * torch.randn(4 * H, generator=g),
        "proj_dec.w.weight": xavier(J, H) * pd_gain,
        "transducer_lin.w.weight": out,
    }


def seeded_tn(seed, B, T, W, p_token=0.35, strength=0.25, noise=0.5):
    """tn_output [B, T, J]: noise, and on a fraction ``p_token`` of the frames a push along a random token's classifier
    row, so those frames emit it (often more than once, until the prediction network's state moves the joint)."""
    out = W["transducer_lin.w.weight"]
    V, J = out.shape
    g = torch.Generator().manual_seed(seed)
    tn = noise * torch.randn(B, T, J, generator=g)
    hit = torch.rand(B, T, generator=g) < p_token
    tok = torch.randint(0, V, (B, T), generator=g)
    dirs = out[tok] / out[tok].norm(dim=-1, keepdim=True) * math.sqrt(J)
    return tn + strength * hit.unsqueeze(-1).float() * dirs


class Oracle:
    def __init__(self, W):
        self.E = W["emb.Embedding.weight"].float()
        self.w_ih = W["dec.rnn.weight_ih_l0"].float()
        self.w_hh = W["dec.rnn.weight_hh_l0"].float()
        self.b_ih, self.b_hh = W["dec.rnn.bias_ih_l0"].float(), W["dec.rnn.bias_hh_l0"].float()
        self.w_pd = W["proj_dec.w.weight"].float()
        self.w_out = W["transducer_lin.w.weight"].float()
        self.H = self.w_hh.shape[1]

    def pn(self, tok, h, c):
        """One prediction-network step: (out_PN, h, c) after token ``tok``."""
        gates = self.w_ih @ self.E[tok] + self.b_ih + self.w_hh @ h + self.b_hh
        i, f, gg, o = gates.split(self.H)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        return self.w_pd @ h, h, c

    def logp(self, tn_t, p):
        x = torch.nn.functional.gelu(tn_t + p)
        return torch.log_softmax(self.w_out @ x, dim=-1)

    @torch.no_grad()
    def row(self, tn, blank, max_sym, state=None, forced=None):
        """Greedy walk of one row.  tn [T, J]; state (p, h, c) or None for PN(blank) from zeros; forced = (tokens,
        frames) of a decision path to follow.  Returns dict(tokens, frames, score, decisions=[(frame, chosen, chosen_logp,
        argmax, top1, top2)], state=(p, h, c))."""
        if state is None:
            z = torch.zeros(self.H)
            p, h, c = self.pn(blank, z, z.clone())
        else:
            p, h, c = (s.float().clone() for s in state)
        toks, frs, decs = [], [], []
        score = torch.zeros((), dtype=torch.float32)
        fk = 0
        for t in range(tn.shape[0]):
            count = 0
            while count <= max_sym:
                lp = self.logp(tn[t].float(), p)
                top = lp.topk(2)
                am = int(lp.argmax())
                if forced is not None:
                    ft, ff = forced
                    tok = int(ft[fk]) if fk < len(ft) and int(ff[fk]) == t else blank
                else:
                    tok = am
                decs.append((t, tok, float(lp[tok]), am, float(top.values[0]), float(top.values[1])))
                if tok == blank:
                    break
                toks.append(tok)
                frs.append(t)
                fk += 1
                score = score + lp[tok]
                p, h, c = self.pn(tok, h, c)
                count += 1
        return dict(tokens=toks, frames=frs, score=float(score), decisions=decs, state=(p, h, c))

    def batch(self, tn, blank, max_sym, state=None):
        """All rows; returns (hyps, exp(score).mean(), rows)."""
        rows = [self.row(tn[b], blank, max_sym, None if state is None else tuple(s[b] for s in state))
                for b in range(tn.shape[0])]
        scores = torch.tensor([r["score"] for r in rows], dtype=torch.float32)
        return [r["tokens"] for r in rows], scores.exp().mean(), rows
