"""CTC greedy decoding -- mirror of speechbrain.decoders.ctc.{filter_ctc_output, ctc_greedy_decode} (decoders/ctc.py:298-378)
for CUDA tensors: the per-frame arg-max runs in ``rows_logsoftmax_argmax_kernel`` (csrc/ctc_scorer.cu), the merge / blank
filter of at most T integers per utterance stays on the host like in the reference.  CTCBeamSearcher (decoders/ctc.py:510-1485,
no language model): the frame loop runs in ``ctc_beam_kernel`` (csrc/ctc_beam.cu), the replay of the surviving token chains
and finalize_decoding on the host.  CTCPrefixBeamSearcher (decoders/ctc.py:1488-1905, no language model): likewise with
``ctc_prefix_beam_kernel`` (csrc/ctc_prefix_beam.cu)."""
import dataclasses
import heapq
import logging
import math
import warnings
from itertools import groupby
from typing import Optional

import numpy as np
import torch

logger = logging.getLogger(__name__)


def filter_ctc_output(string_pred, blank_id=-1):
    """decoders/ctc.py:298-332: merge repetitions, then drop the blank."""
    if not isinstance(string_pred, list):
        raise ValueError("filter_ctc_out can only filter python lists")
    string_out = [i[0] for i in groupby(string_pred)]
    return list(filter(lambda elem: elem != blank_id, string_out))


def frame_argmax(probabilities):
    """[B, T, V] fp32 CUDA -> [B, T] int64 arg-max per frame (first index on ties, like torch.max)."""
    import ctypes  # noqa: F401

    from .._lib import check, lib, ptr, require_cuda, stream_ptr
    require_cuda(probabilities, "ctc_greedy_decode")
    x = probabilities.float().contiguous()
    B, T, V = x.shape
    idx = torch.empty(B, T, device=x.device, dtype=torch.int32)
    with torch.cuda.device(x.device):
        check(lib().sbk_rows_argmax_f32(ptr(x), B * T, V, ptr(idx), stream_ptr(x.device)), "sbk_rows_argmax_f32")
    return idx.long()


def ctc_greedy_decode(probabilities, seq_lens, blank_id=-1):
    """decoders/ctc.py:335-378: probabilities [B, T, V] (or log-probabilities), seq_lens relative -> list of token lists."""
    if isinstance(blank_id, int) and blank_id < 0:
        blank_id = probabilities.shape[-1] + blank_id
    batch_max_len = probabilities.shape[1]
    pred = frame_argmax(probabilities).cpu()
    return greedy_from_argmax(pred, seq_lens, blank_id, batch_max_len)


def greedy_from_argmax(pred, seq_lens, blank_id, batch_max_len=None):
    batch_max_len = batch_max_len or pred.shape[1]
    out = []
    for seq, seq_len in zip(pred.tolist(), seq_lens.cpu()):
        actual_size = int(torch.round(seq_len * batch_max_len))
        out.append(filter_ctc_output(seq[:actual_size], blank_id=blank_id))
    return out


# --------------------------------------------------------------------------------------------------- CTC beam search
@dataclasses.dataclass
class CTCHypothesis:
    """decoders/ctc.py:510-537."""
    text: str
    last_lm_state: None
    score: float
    lm_score: float
    text_frames: Optional[list] = None


_HASH_P = (1 << 61) - 1
_HASH_BASE = 0x1F3D5B79A2C4E6F1  # SBK_CTC_HASH_BASE (include/sbk.h)
_PLAIN, _BLANK, _WORD, _SPACE = 0, 1, 2, 3  # SBK_CTC_TOK_*
MAX_BEAM, MAX_VOCAB = 256, 8192


def _merge_words(a, b):
    """CTCBaseSearcher.merge_tokens (decoders/ctc.py:757-780)."""
    if not b:
        return a
    if not a:
        return b
    return a + " " + b


def _hash(s):
    """Polynomial hash of a string modulo 2^61 - 1 (characters as code point + 1) and base^len(s)."""
    h = 0
    for ch in s:
        h = (h * _HASH_BASE + ord(ch) + 1) % _HASH_P
    return h, pow(_HASH_BASE, len(s), _HASH_P)


class CTCBaseSearcher(torch.nn.Module):
    """The constructor of speechbrain.decoders.ctc.CTCBaseSearcher (decoders/ctc.py:540-716) without a language model, and
    the input checks of decode_beams shared by the device searchers: ``kenlm_model_path`` raises NotImplementedError,
    ``beam_size`` is limited to 256 and the log-probabilities' last dimension to 8192."""

    def __init__(self, blank_index, vocab_list, space_token=" ", kenlm_model_path=None, unigrams=None, alpha=0.5, beta=1.5,
                 unk_score_offset=-10.0, score_boundary=True, beam_size=100, beam_prune_logp=-10.0,
                 token_prune_min_logp=-5.0, prune_history=True, blank_skip_threshold=1.0, topk=1, spm_token="▁"):
        super().__init__()
        name = type(self).__name__
        if kenlm_model_path is not None:
            raise NotImplementedError(f"speechbrain_b200.{name}: KenLM scoring is not built")
        if not 1 <= int(beam_size) <= MAX_BEAM:
            raise ValueError(f"{name}: beam_size={beam_size} outside [1, {MAX_BEAM}]")
        self.blank_index = blank_index
        self.vocab_list = vocab_list
        self.space_token = space_token
        self.kenlm_model_path = kenlm_model_path
        self.unigrams = unigrams
        self.alpha, self.beta, self.unk_score_offset, self.score_boundary = alpha, beta, unk_score_offset, score_boundary
        self.beam_size = int(beam_size)
        self.beam_prune_logp = beam_prune_logp
        self.token_prune_min_logp = token_prune_min_logp
        self.prune_history = prune_history
        self.blank_skip_threshold = math.log(blank_skip_threshold)
        self.topk = topk
        self.spm_token = spm_token
        self.lm = None
        self.is_spm = any(str(s).startswith(spm_token) for s in vocab_list)
        if not self.is_spm:
            try:
                self.space_index = vocab_list.index(space_token)
            except ValueError:
                logger.warning(f"space_token `{space_token}` not found in the vocabulary.Using value -1 as `space_index`."
                               "Note: If your transcription is not expected to contain spaces, you can ignore this warning.")
                self.space_index = -1
        self._dev_tables = {}

    def _kinds(self):
        """Per token: kind (SBK_CTC_TOK_*) and string id (the first index holding the same string)."""
        kinds, sids, first = [], [], {}
        for i, s in enumerate(self.vocab_list):
            if i == self.blank_index:
                k = _BLANK
            elif self.is_spm and s[:1] == self.spm_token:
                k = _WORD
            elif not self.is_spm and i == self.space_index:
                k = _SPACE
            else:
                k = _PLAIN
            kinds.append(k)
            sids.append(first.setdefault(s, i))
        return kinds, sids

    def _tables(self, device):
        if device not in self._dev_tables:
            self._dev_tables[device] = (self._info.to(device).contiguous(), self._hash.to(device).contiguous())
        return self._dev_tables[device]

    def _check_input(self, log_probs, wav_lens, lm_start_state):
        """decode_beams' checks and lengths (decoders/ctc.py:936-986) -> absolute frame counts per utterance."""
        from .._lib import require_cuda
        name = type(self).__name__
        if lm_start_state is not None:
            raise NotImplementedError(f"speechbrain_b200.{name}: lm_start_state needs a language model (not built)")
        require_cuda(log_probs, name)
        if log_probs.dtype != torch.float32:
            raise ValueError(f"{name}: expected float32 log-probabilities, got {log_probs.dtype}")
        if log_probs.dim() != 3:
            raise ValueError(f"{name}: expected [batch, time, vocab] log-probabilities, got {tuple(log_probs.shape)}")
        if log_probs.size(2) != len(self.vocab_list):
            warnings.warn(f"Vocab size mismatch: log_probs vocab dim is {log_probs.size(2)} while vocab_list is "
                          f"{len(self.vocab_list)}. During decoding, going to truncate the log_probs vocab dim to match vocab_list.")
        B, T = log_probs.shape[0], log_probs.shape[1]
        if wav_lens is not None:
            raw = (T * wav_lens).cpu().numpy().astype(int).tolist()
        else:
            raw = [T] * B
        return [len(range(T)[:n]) for n in raw]  # used as a slice bound, like log_probs[:wav_len]

    def _check_shape(self, log_probs):
        B, T, V = log_probs.shape
        blank = self.blank_index
        name = type(self).__name__
        if not (isinstance(blank, int) and 0 <= blank < V):
            raise ValueError(f"{name}: blank_index {blank} outside [0, {V})")
        if V > MAX_VOCAB:
            raise ValueError(f"{name}: vocabulary dimension {V} above the supported {MAX_VOCAB}")
        return B, T, V, min(V, len(self.vocab_list))

    @torch.no_grad()
    def search(self, log_probs, lens):
        """The device search alone: log_probs [B, T, V] fp32 CUDA, lens list of absolute frame counts -> per-frame beam
        counts [B, T], parents and tokens [B, T, beam_size], final scores [B, beam_size], final counts [B] (device)."""
        import ctypes

        from .._lib import check, lib, ptr, stream_ptr
        B, T, V, nv = self._check_shape(log_probs)
        dev = log_probs.device
        x = log_probs.contiguous()
        lens_d = torch.tensor(lens, dtype=torch.int32).to(dev)
        info, hsh = self._tables(dev)
        prm = self._params(self.blank_index)
        K = self.beam_size
        ws_fn, search_fn = self._ABI
        with torch.cuda.device(dev):
            st = stream_ptr(dev)
            nbytes = ctypes.c_size_t(0)
            check(getattr(lib(), ws_fn)(ptr(x), ptr(lens_d), B, T, V, nv, ctypes.byref(prm), ctypes.byref(nbytes), st), ws_fn)
            ws = torch.empty(max(1, nbytes.value), dtype=torch.uint8, device=dev)
            fb = torch.empty(B, T, dtype=torch.int32, device=dev)
            par = torch.empty(B, T, K, dtype=torch.int32, device=dev)
            tok = torch.empty(B, T, K, dtype=torch.int32, device=dev)
            score = torch.empty(B, K, dtype=self._SCORE_DTYPE, device=dev)
            nfin = torch.empty(B, dtype=torch.int32, device=dev)
            check(getattr(lib(), search_fn)(ptr(x), ptr(lens_d), B, T, V, nv, ptr(info), ptr(hsh), ctypes.byref(prm), ptr(ws),
                                            ctypes.c_size_t(ws.numel()), ptr(fb), ptr(par), ptr(tok), ptr(score), ptr(nfin),
                                            st), search_fn)
        return fb, par, tok, score, nfin

    def decode_beams(self, log_probs, wav_lens=None, lm_start_state=None):
        """decoders/ctc.py:936-986: log_probs [B, T, V] fp32 CUDA log-probabilities, wav_lens relative (or None) ->
        B lists of at most topk CTCHypothesis."""
        lens = self._check_input(log_probs, wav_lens, lm_start_state)
        fb, par, tok, score, nfin = (t.cpu().numpy() for t in self.search(log_probs, lens))
        return [self._finalize(self._replay(lens[b], fb[b], par[b], tok[b], score[b], int(nfin[b])))
                for b in range(log_probs.shape[0])]

    def forward(self, log_probs, wav_lens=None, lm_start_state=None):
        return self.decode_beams(log_probs, wav_lens, lm_start_state)

    def __call__(self, log_probs, wav_lens=None, lm_start_state=None):
        return self.decode_beams(log_probs, wav_lens, lm_start_state)


class CTCBeamSearcher(CTCBaseSearcher):
    """Mirror of speechbrain.decoders.ctc.CTCBeamSearcher (decoders/ctc.py:540-1485) without a language model, for CUDA
    log-probabilities [B, T, V] fp32.  The frame loop (token pruning, extension, merging of beams with equal
    (text, partial word, last token), beam pruning, stable top-beam_size sort and history pruning) runs in
    ``ctc_beam_kernel`` (csrc/ctc_beam.cu), one CTA per utterance, on string hashes; the host then replays the string
    rules on the surviving token chains and runs finalize_decoding (commit, merge by text, prune, sort) exactly, in
    NumPy float32.  Constructor keywords and defaults are the reference's (CTCBaseSearcher)."""

    _ABI = ("sbk_ctc_beam_workspace_bytes", "sbk_ctc_beam_search")
    _SCORE_DTYPE = torch.float32

    def __init__(self, blank_index, vocab_list, space_token=" ", kenlm_model_path=None, unigrams=None, alpha=0.5, beta=1.5,
                 unk_score_offset=-10.0, score_boundary=True, beam_size=100, beam_prune_logp=-10.0,
                 token_prune_min_logp=-5.0, prune_history=True, blank_skip_threshold=1.0, topk=1, spm_token="▁"):
        super().__init__(blank_index, vocab_list, space_token, kenlm_model_path, unigrams, alpha, beta, unk_score_offset,
                         score_boundary, beam_size, beam_prune_logp, token_prune_min_logp, prune_history,
                         blank_skip_threshold, topk, spm_token)
        # per-token tables: kind, string id, appended string (its hash, base^length, length)
        kinds, sids = self._kinds()
        app = [s[1:] if k == _WORD else (s if k == _PLAIN else "") for s, k in zip(vocab_list, kinds)]
        if prune_history and any(a and a.split() != [a] for a in app):
            # the device keys the history by the last committed word, which needs whitespace-free token strings
            raise NotImplementedError("CTCBeamSearcher: prune_history with tokens that contain whitespace is not built")
        self._kind = np.array(kinds, dtype=np.int64)
        self._sid = np.array(sids + [-1], dtype=np.int64)  # [-1]: "no token yet"
        self._app = app
        self._info = torch.tensor([(k, sid, len(a)) for k, sid, a in zip(kinds, sids, app)], dtype=torch.int32).reshape(-1, 3)
        self._hash = torch.tensor(np.array([_hash(a) for a in app], dtype=np.uint64).view(np.int64)).reshape(-1, 2)

    def _params(self, blank):
        from .._lib import sbk_ctc_beam_params
        return sbk_ctc_beam_params(blank=blank, beam_size=self.beam_size, prune_history=int(bool(self.prune_history)),
                                   token_prune_min_logp=float(np.float32(self.token_prune_min_logp)),
                                   beam_prune_logp=float(np.float32(self.beam_prune_logp)),
                                   blank_skip_logp=float(np.float32(self.blank_skip_threshold)))


    def _replay(self, n, fb, par, tok, score, nfin):
        """The final beams of one utterance from the search history: text, partial word, word frames, partial frames."""
        if nfin < 0:
            raise ValueError("max() arg is an empty sequence (a frame had no candidate token inside vocab_list)")
        proc = np.flatnonzero(fb[:n] >= 0)
        if len(proc) == 0:
            return [("", "", (), (-1, -1), 0.0)]
        P, K = len(proc), nfin
        chain = np.empty((P, K), dtype=np.int64)
        idx = np.arange(K)
        for j in range(P - 1, -1, -1):
            chain[j] = tok[proc[j], idx]
            idx = par[proc[j], idx]
        sid = self._sid[chain]
        prev = np.concatenate([np.full((1, K), -1, dtype=np.int64), sid[:-1]], 0)
        nonblank = chain != self.blank_index
        rep = (nonblank & (sid == prev)).T.tolist()
        kind, app, frames_of = self._kind, self._app, proc.tolist()
        chain_t = chain.T.tolist()
        out = []
        for k in range(K):
            text, part, words, pf = "", "", [], (-1, -1)
            ck, rk = chain_t[k], rep[k]
            for j in np.flatnonzero(nonblank[:, k]).tolist():
                f, t = frames_of[j], ck[j]
                if rk[j]:
                    pf = (pf[0], f + 1)
                    continue
                kd = kind[t]
                if kd == _WORD or kd == _SPACE:
                    if part:
                        words.append(pf)
                        text = _merge_words(text, part)
                    part, pf = (app[t], (f, f + 1)) if kd == _WORD else ("", (-1, -1))
                else:
                    part += app[t]
                    pf = (f, f + 1) if pf[0] < 0 else (pf[0], f + 1)
            out.append((text, part, tuple(words), pf, score[k]))
        return out

    def _finalize(self, beams):
        """finalize_decoding(force_next_word=True, is_end=True) + decode_log_probs' CTCHypothesis list (:868-934, :1127-1152)."""
        fin = {}
        for text, part, words, pf, sc in beams:
            nw = words + (pf,) if part else words
            key = _merge_words(text, part)
            fin[key] = (np.logaddexp(fin[key][0], sc), nw) if key in fin else (sc, nw)
        items = [(s, text, nw) for text, (s, nw) in fin.items()]
        top = max(it[0] for it in items)
        items = [it for it in items if it[0] >= top + self.beam_prune_logp]
        items = heapq.nlargest(self.beam_size, items, key=lambda it: it[0])
        return [CTCHypothesis(text=" ".join(text.split()), last_lm_state=None, text_frames=list(zip(text.split(), nw)),
                              score=s, lm_score=s) for s, text, nw in items][: self.topk]


class CTCPrefixBeamSearcher(CTCBaseSearcher):
    """Mirror of speechbrain.decoders.ctc.CTCPrefixBeamSearcher (decoders/ctc.py:1488-1905) without a language model, for
    CUDA log-probabilities [B, T, V] fp32.  The frame loop (candidate tokens in CPython's set order, prefix extension with
    blank / non-blank probabilities, step, beam pruning, stable top-beam_size sort and history pruning) runs in
    ``ctc_prefix_beam_kernel`` (csrc/ctc_prefix_beam.cu), one CTA per utterance, on string hashes, with the reference's
    float32 / float64 sums; the host then replays the texts of the surviving beams with exact strings and runs
    finalize_decoding (merge by text, prune, sort) in NumPy float64.  Scores are float64, as in the reference.
    Constructor keywords and defaults are the reference's (CTCBaseSearcher)."""

    _ABI = ("sbk_ctc_prefix_beam_workspace_bytes", "sbk_ctc_prefix_beam_search")
    _SCORE_DTYPE = torch.float64

    def __init__(self, blank_index, vocab_list, space_token=" ", kenlm_model_path=None, unigrams=None, alpha=0.5, beta=1.5,
                 unk_score_offset=-10.0, score_boundary=True, beam_size=100, beam_prune_logp=-10.0,
                 token_prune_min_logp=-5.0, prune_history=True, blank_skip_threshold=1.0, topk=1, spm_token="▁"):
        super().__init__(blank_index, vocab_list, space_token, kenlm_model_path, unigrams, alpha, beta, unk_score_offset,
                         score_boundary, beam_size, beam_prune_logp, token_prune_min_logp, prune_history,
                         blank_skip_threshold, topk, spm_token)
        kinds, sids = self._kinds()
        info, hashes = [], []
        for s, k, sid in zip(vocab_list, kinds, sids):
            app = " " + s[1:] if k == _WORD else s   # what a new beam appends to its text
            ws = [i for i, ch in enumerate(app) if ch.isspace()]
            lead, tail = (app[:ws[0]], app[ws[-1] + 1:]) if ws else (app, "")
            inner = [w for w in app[ws[0] + 1:ws[-1]].split()][-1:] if len(ws) > 1 else []
            inner = inner[0] if inner else ""
            part = s[1:] if k == _WORD else ""
            info.append((k, sid, len(s), len(app), len(part), int(bool(ws)), len(lead), len(tail), len(inner)))
            hashes.append(_hash(s) + _hash(app) + (_hash(part)[0],) + _hash(lead) + (_hash(tail)[0], _hash(inner)[0]))
        self._kind = kinds
        self._info = torch.tensor(info, dtype=torch.int32).reshape(-1, 9)
        self._hash = torch.tensor(np.array(hashes, dtype=np.uint64).view(np.int64)).reshape(-1, 9)

    def _params(self, blank):
        from .._lib import sbk_ctc_prefix_beam_params
        return sbk_ctc_prefix_beam_params(blank=blank, beam_size=self.beam_size, prune_history=int(bool(self.prune_history)),
                                          token_prune_min_logp=float(np.float32(self.token_prune_min_logp)),
                                          blank_skip_logp=float(np.float32(self.blank_skip_threshold)),
                                          beam_prune_logp=float(self.beam_prune_logp))

    def _replay(self, n, fb, par, tok, score, nfin):
        """The final beams of one utterance from the search history: text, partial word, word frames, partial frames,
        score.  Each surviving beam was carried over (token -1) or created from its parent by a token
        (_get_new_beam's four cases)."""
        proc = np.flatnonzero(fb[:n] >= 0)
        if len(proc) == 0:
            return [("", "", (), (-1, -1), 0.0)]
        P, K = len(proc), nfin
        chain = np.empty((P, K), dtype=np.int64)
        idx = np.arange(K)
        for j in range(P - 1, -1, -1):
            chain[j] = tok[proc[j], idx]
            idx = par[proc[j], idx]
        vocab, kind, frames_of = self.vocab_list, self._kind, proc.tolist()
        out = []
        for k in range(K):
            text, part, words, pf, last = "", "", (), (-1, -1), None
            ck = chain[:, k].tolist()
            for j in np.flatnonzero(chain[:, k] >= 0).tolist():
                f, t = frames_of[j], ck[j]
                s, kd = vocab[t], kind[t]
                if kd == _SPACE or kd == _WORD:
                    words = words + (pf,) if part else words
                    text, part, pf = (text + s, "", (-1, -1)) if kd == _SPACE else (text + " " + s[1:], s[1:], (f, f + 1))
                elif t == last:
                    text, pf = text + s, (pf[0], f + 1)
                else:
                    text, part, pf = text + s, part + s, ((f, f + 1) if pf[0] < 0 else (pf[0], f + 1))
                last = t
            out.append((text, part, words, pf, score[k]))
        return out

    def _finalize(self, beams):
        """finalize_decoding(force_next_word=True, is_end=True) + decode_log_probs' CTCHypothesis list (:868-934,
        :1127-1152): the key merge(text, partial word) repeats the partial word, which the text already ends in; a merged
        entry takes the later beam's text and frames."""
        fin = {}
        for text, part, words, pf, sc in beams:
            nw = words + (pf,) if part else words
            key = _merge_words(text, part)
            fin[key] = (np.logaddexp(fin[key][0], sc), text, nw) if key in fin else (sc, text, nw)
        items = list(fin.values())
        top = max(it[0] for it in items)
        items = [it for it in items if it[0] >= top + self.beam_prune_logp]
        items = heapq.nlargest(self.beam_size, items, key=lambda it: it[0])
        return [CTCHypothesis(text=" ".join(text.split()), last_lm_state=None, text_frames=list(zip(text.split(), nw)),
                              score=s, lm_score=s) for s, text, nw in items][: self.topk]
