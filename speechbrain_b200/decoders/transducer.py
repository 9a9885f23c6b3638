"""TransducerBeamSearcher -- drop-in for speechbrain.decoders.transducer.TransducerBeamSearcher (decoders/transducer.py:25-
476): the greedy search (``beam_size=1``) and the beam search without a language model (``beam_size > 1``) of the
Conformer-Transducer recipes, on the device.

The prediction network must be the recipes' ``[Embedding, LSTM, Linear(bias=False)]`` (one unidirectional LSTM layer with
biases), the joint ``Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU)`` and the classifier
``[Linear(bias=False)]``.  The whole search of a call -- every frame, every emitted symbol, the LSTM steps, the joint and
the log-softmax -- runs in one persistent kernel (csrc/transducer.cu, C ABI ``sbk_transducer_greedy``).

Semantics kept from the reference:

* the start state is PN(blank) from a zero LSTM state (or ``hidden_state``);
* per frame a row emits at most ``max_symbols_per_step + 1`` symbols (the reference's ``count <= max`` loop), the arg-max
  takes the first index on ties, and the score of a row is the sum of its emitted tokens' log-probabilities;
* EVERY frame of ``tn_output`` is decoded: there is no lengths argument, so the padded frames of a batch are decoded too and
  a short utterance can pick up tokens from them, exactly as in the reference.

Rows are independent (a row that produced blank keeps producing blank for the rest of the frame), so the device walks
each row on its own; the results do not depend on the other rows of the batch.

The beam search (``transducer_beam_search_decode``, decoders/transducer.py:320-476, C ABI ``sbk_transducer_beam``) keeps
the reference's order of pops, its key score / len(prediction), its state_beam and expand_beam tests and its fp32 score
sums; each utterance is searched on its own, as in the reference.  Exact ties between top-K log-probabilities go to the
lower token id.  A frame stops after ``4 * beam_size`` pops at the most (the reference would loop for ever on a frame whose
top-K never holds blank); the call then raises naming the utterance and the frame.  RNNLM shallow fusion (``lm_weight >
0``), ``nbest > beam_size`` and beams above 32 are not built."""
import ctypes
from dataclasses import dataclass
from typing import Any, Optional

import torch

from .. import _lib as _L
from .._lib import check, lib, ptr, require_cuda, sbk_tensor, stream_ptr
from ..engine_cache import fingerprint
from ..nnet.embedding import Embedding
from ..nnet.linear import Linear
from ..nnet.RNN import LSTM
from ..nnet.transducer.transducer_joint import Transducer_joint

MAX_HIDDEN = 1024  # LSTM hidden and joint sizes: multiples of 64 up to this
MAX_VOCAB = 4096
MAX_BATCH = 1024
MAX_BEAM = 32  # SBK_TRANSDUCER_BEAM_MAX


def pop_cap(beam_size):
    """SBK_TRANSDUCER_BEAM_POP_CAP: the most pops of one frame of the beam search"""
    return 4 * beam_size


class sbk_transducer_config(ctypes.Structure):
    _fields_ = [("vocab", ctypes.c_int), ("emb_dim", ctypes.c_int), ("hidden", ctypes.c_int), ("joint", ctypes.c_int)]


@dataclass
class TransducerGreedySearcherStreamingContext(torch.nn.Module):
    """decoders/transducer.py:15-22: the ``(out_PN, (h, c))`` state carried across
    ``transducer_greedy_decode_streaming`` calls."""

    hidden: Optional[Any] = None


class _DeviceSearch:
    """The repacked weights of one prediction network + classifier on one device (``sbk_transducer``)."""

    def __init__(self, emb, lstm, proj_dec, lin, device):
        V, E = emb.Embedding.weight.shape
        H, J = lstm.rnn.hidden_size, proj_dec.w.out_features
        sd = {"emb.weight": emb.Embedding.weight, "lstm.weight_ih": lstm.rnn.weight_ih_l0,
              "lstm.weight_hh": lstm.rnn.weight_hh_l0, "lstm.bias_ih": lstm.rnn.bias_ih_l0,
              "lstm.bias_hh": lstm.rnn.bias_hh_l0, "proj_dec.weight": proj_dec.w.weight, "out.weight": lin.w.weight}
        host = {k: v.detach().float().cpu().contiguous() for k, v in sd.items()}
        arr = (sbk_tensor * len(host))(*[sbk_tensor(k.encode(), v.data_ptr(), v.numel()) for k, v in host.items()])
        cfg = sbk_transducer_config(V, E, H, J)
        self.V, self.H, self.J, self.device = V, H, J, device
        self.handle = ctypes.c_void_p()
        with torch.cuda.device(device):
            check(lib().sbk_transducer_create(ctypes.byref(cfg), arr, len(host), ctypes.byref(self.handle)),
                  "sbk_transducer_create")

    def __del__(self):
        if getattr(self, "handle", None) and _L._lib is not None:
            _L._lib.sbk_transducer_destroy(self.handle)
            self.handle = None

    def info(self):
        ctas, smem = ctypes.c_int(), ctypes.c_int()
        check(lib().sbk_transducer_info(self.handle, ctypes.byref(ctas), ctypes.byref(smem)), "sbk_transducer_info")
        return ctas.value, smem.value

    def greedy(self, tn, blank, max_symbols_per_step, state=None, want_frames=False, want_stats=False):
        """tn [B, T, J] fp32 on the device -> dict of device tensors (tokens, n_tokens, logp_sum, h, c, out_pn[, frames,
        stats]); enqueued on the current stream."""
        B, T, _ = tn.shape
        dev = tn.device
        f32 = dict(device=dev, dtype=torch.float32)
        if state is None:
            h, c, p = torch.empty(B, self.H, **f32), torch.empty(B, self.H, **f32), torch.empty(B, self.J, **f32)
        else:
            h, c, p = (s.detach().to(**f32).contiguous().clone() for s in state)
        stride = T * (max_symbols_per_step + 1)
        out = dict(tokens=torch.empty(B, stride, device=dev, dtype=torch.int32),
                   n_tokens=torch.empty(B, device=dev, dtype=torch.int32), logp_sum=torch.empty(B, **f32), h=h, c=c,
                   out_pn=p)
        frames = torch.empty(B, stride, device=dev, dtype=torch.int32) if want_frames else None
        stats = torch.zeros(2, device=dev, dtype=torch.int32) if want_stats else None
        with torch.cuda.device(dev):
            check(lib().sbk_transducer_greedy(self.handle, ptr(tn), B, T, blank, max_symbols_per_step, int(state is None),
                                              ptr(h), ptr(c), ptr(p), ptr(out["tokens"]), ptr(frames),
                                              ptr(out["n_tokens"]), ptr(out["logp_sum"]), ptr(stats), stream_ptr(dev)),
                  "sbk_transducer_greedy")
        if want_frames:
            out["frames"] = frames
        if want_stats:
            out["stats"] = stats
        return out

    def beam(self, tn, blank, beam_size, nbest, state_beam, expand_beam, want_trace=False, want_stats=False):
        """tn [B, T, J] fp32 on the device -> dict of device tensors (tokens [B, nbest, T * pop_cap], lens [B, nbest],
        scores [B, nbest][, trace [B, T * pop_cap, 6 + 2 beam_size], stats [4]]); enqueued on the current stream."""
        B, T, _ = tn.shape
        dev = tn.device
        cap = pop_cap(beam_size)
        i32 = dict(device=dev, dtype=torch.int32)
        out = dict(tokens=torch.empty(B, nbest, T * cap, **i32), lens=torch.empty(B, nbest, **i32),
                   scores=torch.empty(B, nbest, device=dev, dtype=torch.float32))
        if want_trace:
            out["trace"] = torch.empty(B, T * cap, 6 + 2 * beam_size, **i32)
        if want_stats:
            out["stats"] = torch.zeros(4, **i32)
        with torch.cuda.device(dev):
            check(lib().sbk_transducer_beam(self.handle, ptr(tn), B, T, blank, beam_size, nbest, ctypes.c_float(state_beam),
                                            ctypes.c_float(expand_beam), ptr(out["tokens"]), ptr(out["lens"]),
                                            ptr(out["scores"]), ptr(out.get("trace")), ptr(out.get("stats")),
                                            stream_ptr(dev)),
                  "sbk_transducer_beam")
        return out


class TransducerBeamSearcher(torch.nn.Module):
    """decoders/transducer.py:25-154 with the reference's constructor: ``beam_size=1`` selects the greedy search,
    ``beam_size > 1`` the beam search without a language model."""

    def __init__(self, decode_network_lst, tjoint, classifier_network, blank_id, beam_size=4, nbest=5, lm_module=None,
                 lm_weight=0.0, state_beam=2.3, expand_beam=2.3):
        super().__init__()
        self.decode_network_lst = decode_network_lst
        self.tjoint = tjoint
        self.classifier_network = classifier_network
        self.blank_id = blank_id
        self.beam_size = beam_size
        self.nbest = nbest
        self.lm = lm_module
        self.lm_weight = lm_weight
        if lm_module is None and lm_weight > 0:
            raise ValueError("Language model is not provided.")
        self.state_beam = state_beam
        self.expand_beam = expand_beam
        if beam_size > 1:
            if lm_module is not None and lm_weight > 0:
                raise NotImplementedError("speechbrain_b200.TransducerBeamSearcher: RNNLM shallow fusion (lm_weight > 0) "
                                          "is not built")
            if nbest > beam_size:
                raise NotImplementedError(f"speechbrain_b200.TransducerBeamSearcher: nbest {nbest} above beam_size "
                                          f"{beam_size} is not built")
            if beam_size > MAX_BEAM:
                raise NotImplementedError(f"speechbrain_b200.TransducerBeamSearcher: beam_size {beam_size} above "
                                          f"{MAX_BEAM}")
        self._check_layout()
        self.searcher = self.transducer_beam_search_decode if beam_size > 1 else self.transducer_greedy_decode
        self._search = None
        self._fp = None
        self.builds = 0

    def _check_layout(self):
        dec, cls = list(self.decode_network_lst), list(self.classifier_network)
        if (len(dec) != 3 or not isinstance(dec[0], Embedding) or type(dec[1]) is not LSTM
                or not isinstance(dec[2], Linear)):
            raise NotImplementedError("speechbrain_b200.TransducerBeamSearcher: decode_network_lst must be [Embedding, LSTM, "
                                      f"Linear] (got {[type(m).__name__ for m in dec]})")
        if len(cls) != 1 or not isinstance(cls[0], Linear):
            raise NotImplementedError("speechbrain_b200.TransducerBeamSearcher: classifier_network must be [Linear] "
                                      f"(got {[type(m).__name__ for m in cls]})")
        if not isinstance(self.tjoint, Transducer_joint):
            raise NotImplementedError("speechbrain_b200.TransducerBeamSearcher: tjoint must be a Transducer_joint")
        emb, lstm, proj, lin = dec[0], dec[1], dec[2], cls[0]
        rnn = lstm.rnn
        if rnn.num_layers != 1 or rnn.bidirectional or not rnn.bias or rnn.proj_size:
            raise NotImplementedError("speechbrain_b200.TransducerBeamSearcher: the LSTM must have one unidirectional layer "
                                      "with biases")
        if proj.w.bias is not None or lin.w.bias is not None:
            raise NotImplementedError("speechbrain_b200.TransducerBeamSearcher: the prediction-network projection and the "
                                      "output Linear must have bias=False")
        V, E = emb.Embedding.weight.shape
        H, J = rnn.hidden_size, proj.w.out_features
        if rnn.input_size != E or proj.w.in_features != H or lin.w.in_features != J or lin.w.out_features != V:
            raise ValueError(f"TransducerBeamSearcher: inconsistent sizes (Embedding {V}x{E}, LSTM {rnn.input_size}->{H}, "
                             f"proj {proj.w.in_features}->{J}, classifier {lin.w.in_features}->{lin.w.out_features})")
        for name, n in (("LSTM hidden size", H), ("joint size", J)):
            if n % 64 or not 64 <= n <= MAX_HIDDEN:
                raise NotImplementedError(f"speechbrain_b200.TransducerBeamSearcher: {name} {n} is not a multiple of 64 in "
                                          f"[64, {MAX_HIDDEN}]")
        if V > MAX_VOCAB:
            raise NotImplementedError(f"speechbrain_b200.TransducerBeamSearcher: vocabulary {V} above {MAX_VOCAB}")
        if not 0 <= self.blank_id < V:
            raise ValueError(f"TransducerBeamSearcher: blank_id {self.blank_id} outside [0, {V})")
        if self.beam_size > V:
            raise NotImplementedError(f"speechbrain_b200.TransducerBeamSearcher: beam_size {self.beam_size} above the "
                                      f"vocabulary size {V}")

    def _sources(self):
        dec = list(self.decode_network_lst)
        return {"emb": dec[0], "lstm": dec[1], "proj_dec": dec[2], "out": list(self.classifier_network)[0]}

    def device_search(self, device):
        """The repacked device weights, rebuilt when a source tensor changes (``load_state_dict``, ``.to()``)."""
        src = self._sources()
        fp = (fingerprint(src), str(device))
        if self._search is None or self._fp != fp:
            self._search = None
            self._search = _DeviceSearch(src["emb"], src["lstm"], src["proj_dec"], src["out"], torch.device(device))
            self._fp = fp
            self.builds += 1
        return self._search

    def forward(self, tn_output):
        return self.searcher(tn_output)

    @torch.no_grad()
    def transducer_greedy_decode(self, tn_output, hidden_state=None, return_hidden=False, max_symbols_per_step=5):
        """decoders/transducer.py:156-291.  tn_output [B, T, J] (the projected encoder states) on a CUDA device;
        ``hidden_state`` = ``(out_PN [B, 1, J], (h [1, B, H], c [1, B, H]))`` as returned with ``return_hidden``.
        Returns (hyps list[list[int]], exp(score).mean() over the batch, None, None[, (out_PN, (h, c))]); the state
        tensors are new tensors (the reference updates the passed-in ones in place)."""
        B, r = self._enqueue_search(tn_output, hidden_state, max_symbols_per_step)
        n = r["n_tokens"].cpu().tolist()
        toks = r["tokens"].cpu()
        hyps = [toks[b, :n[b]].tolist() for b in range(B)]
        score = r["logp_sum"].cpu().exp().mean()
        ret = (hyps, score, None, None)
        if return_hidden:
            ret += ((r["out_pn"].unsqueeze(1), (r["h"].unsqueeze(0), r["c"].unsqueeze(0))),)
        return ret

    def _check_input(self, tn_output):
        """Checks tn_output: (the device weights, B, T)."""
        require_cuda(tn_output, "TransducerBeamSearcher")
        if tn_output.ndim != 3:
            raise ValueError(f"TransducerBeamSearcher: tn_output must be [B, T, J], got {tuple(tn_output.shape)}")
        B, T, J = tn_output.shape
        s = self.device_search(tn_output.device)
        if J != s.J:
            raise ValueError(f"TransducerBeamSearcher: tn_output width {J}, the joint expects {s.J}")
        if not 1 <= B <= MAX_BATCH:
            raise NotImplementedError(f"speechbrain_b200.TransducerBeamSearcher: batch size {B} outside [1, {MAX_BATCH}]")
        return s, B, T

    def _enqueue_search(self, tn_output, hidden_state, max_symbols_per_step):
        """Checks the arguments and enqueues the device search: (B, the dict of device tensors of _DeviceSearch.greedy)."""
        s, B, T = self._check_input(tn_output)
        if max_symbols_per_step < 0:
            raise ValueError("max_symbols_per_step must be >= 0")
        state = None
        if hidden_state is not None:
            out_pn, (h, c) = hidden_state
            state = (h.reshape(B, s.H), c.reshape(B, s.H), out_pn.reshape(B, s.J))
        if T == 0:
            raise ValueError("TransducerBeamSearcher: tn_output has no frames")
        tn = tn_output.detach().to(torch.float32).contiguous()
        return B, s.greedy(tn, self.blank_id, int(max_symbols_per_step), state)

    def transducer_greedy_decode_streaming(self, x: torch.Tensor, context: TransducerGreedySearcherStreamingContext):
        """decoders/transducer.py:293-318: decode a chunk, carrying ``(out_PN, hidden)`` in ``context`` on the device.  The
        reference discards the score here, so it is not fetched: the token counts and ids come to the host in one copy,
        the call's only host synchronisation."""
        B, r = self._enqueue_search(x, context.hidden, 5)
        packed = torch.cat([r["n_tokens"].unsqueeze(1), r["tokens"]], dim=1).cpu()
        context.hidden = (r["out_pn"].unsqueeze(1), (r["h"].unsqueeze(0), r["c"].unsqueeze(0)))
        return [packed[b, 1:1 + int(packed[b, 0])].tolist() for b in range(B)]

    @torch.no_grad()
    def transducer_beam_search_decode(self, tn_output):
        """decoders/transducer.py:320-476 without a language model.  tn_output [B, T, J] on a CUDA device; every frame is
        decoded.  Returns (best hyps list[list[int]], exp(best normalised scores).mean(), nbest hyps per utterance, their
        normalised scores as 0-dim tensors), the reference's return value."""
        r, B = self._enqueue_beam(tn_output)
        lens = r["lens"].cpu()
        capped = [b for b in range(B) if int(lens[b, 0]) <= -2]
        if capped:
            b = capped[0]
            raise RuntimeError(f"TransducerBeamSearcher: utterance {b} reached the limit of {pop_cap(self.beam_size)} pops "
                               f"in frame {-2 - int(lens[b, 0])} (blank never entered the top {self.beam_size})")
        n = max(1, int(lens.max()))
        toks, scores = r["tokens"][:, :, :n].cpu(), r["scores"].cpu()
        nbest_batch = [[toks[b, k, :int(lens[b, k])].tolist() for k in range(self.nbest) if int(lens[b, k]) >= 0]
                       for b in range(B)]
        nbest_batch_score = [[scores[b, k].clone() for k in range(self.nbest) if int(lens[b, k]) >= 0] for b in range(B)]
        best = torch.Tensor([float(s[0]) for s in nbest_batch_score]).exp().mean()
        return [h[0] for h in nbest_batch], best, nbest_batch, nbest_batch_score

    def _enqueue_beam(self, tn_output, want_trace=False, want_stats=False):
        """Checks tn_output and enqueues the device beam search: (the dict of _DeviceSearch.beam, B)."""
        s, B, T = self._check_input(tn_output)
        if T == 0:
            raise ValueError("TransducerBeamSearcher: tn_output has no frames")
        tn = tn_output.detach().to(torch.float32).contiguous()
        return s.beam(tn, self.blank_id, int(self.beam_size), int(self.nbest), float(self.state_beam),
                      float(self.expand_beam), want_trace, want_stats), B
