"""CPU oracle of CTCPrefixBeamSearcher without a language model (speechbrain.decoders.ctc, v1.1.0), restated in NumPy.

A beam is (text, partial word, last token string, last token index, word frames, partial frames) with the prefix-search
probabilities p_b / p_nb (after the last step), n_p_b / n_p_nb (being accumulated) and score.  Per frame f < length:
  * skip the frame when lp[blank] > float32(log(blank_skip_threshold));
  * candidate tokens: the CPython set ``{t : lp[t] > token_prune_min_logp} | {argmax} & set(range(len(vocab)))``, visited
    in that set's iteration order (``candidate_order``, an emulation of CPython 3.12's set tables for int keys);
  * token-major, over the beams at the frame's start in order: the blank adds score + p to n_p_b; any other token first
    adds p_nb + p to the beam's own n_p_nb when the token's STRING equals the last token's, then looks up
    ``text + token`` among all beams (those created earlier in the frame included, first match in list order), creates
    it on a miss (space token, sentencepiece word start stored as ``text + " " + token[1:]``, repeated INDEX, plain) and
    adds p_b + p (same index, p_b > -inf) or score + p (other index) to that beam's n_p_nb;
  * step: p_b, p_nb = n_p_b, n_p_nb; score = logaddexp(p_b, p_nb); keep score >= max + beam_prune_logp, the beam_size
    best (stable), and with prune_history the first beam per (last word of the text, partial word, last token).
Arithmetic follows the reference's types under NumPy 2: p_b, p_nb and n_p_* are Python floats, score is a float64 after
the first step (a Python 0.0 before it), p is a float32, and a Python float next to a float32 is cast to float32.  So
``score + p`` folds in float64 except on the first processed frame, and ``p_nb + p`` / ``p_b + p`` fold in float32.
At the end every beam's key is merge(text, partial word) (the text already holds the partial word, so it appears twice),
equal keys merge (the later beam's fields, logaddexp of the scores), then the prune and sort run once more; the top
``topk`` are returned with whitespace normalised and ``text_frames = zip(text.split(), word frames)``."""
import math

import numpy as np

NEG = -math.inf


# ------------------------------------------------------------------------------ CPython 3.12 set tables, int keys
class PySetEmu:
    """The slot table of a CPython 3.12 set of non-negative ints (hash(v) == v < 2^61 - 1), without deletions:
    set_add_entry, set_insert_clean, set_table_resize and set_merge of Objects/setobject.c."""

    def __init__(self):
        self.table = [None] * 8
        self.used = 0

    @property
    def mask(self):
        return len(self.table) - 1

    @staticmethod
    def _probe(table, v, stop):
        """First slot on v's probe sequence where stop(entry) holds (9 linear probes, then perturbation)."""
        mask = len(table) - 1
        perturb, i = v, v & mask
        while True:
            for j in range(10 if i + 9 <= mask else 1):
                if stop(table[i + j]):
                    return i + j
            perturb >>= 5
            i = (i * 5 + 1 + perturb) & mask

    def _resize(self, minused):
        size = 8
        while size <= minused:
            size <<= 1
        old, self.table = self.table, [None] * size
        for v in old:
            if v is not None:
                self.table[self._probe(self.table, v, lambda e: e is None)] = v

    def add(self, v):
        i = self._probe(self.table, v, lambda e: e is None or e == v)
        if self.table[i] is None:
            self.table[i] = v
            self.used += 1
            if self.used * 5 >= self.mask * 3:
                self._resize(self.used * 2 if self.used > 50000 else self.used * 4)

    def merge(self, other):
        """set_merge(self, other): set(other_set), a | b and update()."""
        if other.used == 0:
            return
        if (self.used + other.used) * 5 >= self.mask * 3:
            self._resize((self.used + other.used) * 2)
        if self.used == 0 and self.mask == other.mask:
            self.table = list(other.table)
            self.used = other.used
        elif self.used == 0:
            for v in other:
                self.table[self._probe(self.table, v, lambda e: e is None)] = v
            self.used = other.used
        else:
            for v in other:
                self.add(v)

    def __iter__(self):
        return (v for v in self.table if v is not None)

    def __len__(self):
        return self.used


def candidate_order(above, argmax, n_vocab):
    """list(set(above) | {argmax} & set(range(n_vocab))) for ascending ``above``, as CPython 3.12 iterates it."""
    a = PySetEmu()
    for v in above:
        a.add(int(v))
    u = PySetEmu()
    u.merge(a)
    m = PySetEmu()
    m.add(int(argmax))
    u.merge(m)
    r = PySetEmu()
    if n_vocab > len(u):   # set_intersection walks the smaller operand (the right one on equal sizes)
        for v in u:
            if v < n_vocab:
                r.add(v)
    else:                  # set(range(n)) holds v in slot v: it iterates in ascending order
        members = set(u)
        for v in range(n_vocab):
            if v in members:
                r.add(v)
    return list(r)


# ------------------------------------------------------------------------------------------------- the search
def lae32(a, b):
    """np.logaddexp of a Python float and a float32 (both cast to float32), back to a Python float."""
    return float(np.logaddexp(np.float32(a), np.float32(b)))


def lae64(a, b):
    return float(np.logaddexp(np.float64(a), np.float64(b)))


def merge_words(a, b):
    if not b:
        return a
    if not a:
        return b
    return a + " " + b


def frame_lengths(T, wav_lens, B):
    """decode_beams' lengths: None -> T each; else (T * wav_lens) truncated, then the number of frames a slice [:n] keeps."""
    if wav_lens is None:
        raw = [T] * B
    else:
        raw = (T * wav_lens).cpu().numpy().astype(int).tolist()
    return [len(range(T)[:n]) for n in raw]


class _Beam:
    __slots__ = ("text", "part", "last", "lidx", "frames", "pf", "p_b", "p_nb", "n_p_b", "n_p_nb", "score", "first")

    def __init__(self, text, part, last, lidx, frames, pf, p_b=NEG, score=NEG, first=False):
        self.text, self.part, self.last, self.lidx, self.frames, self.pf = text, part, last, lidx, frames, pf
        self.p_b, self.p_nb, self.n_p_b, self.n_p_nb, self.score = p_b, NEG, NEG, NEG, score
        self.first = first   # score is still the Python 0.0 of the start beam: score + p is a float32


def decode_one(lp, n, vocab, blank, space_token=" ", beam_size=100, beam_prune_logp=-10.0, token_prune_min_logp=-5.0,
               prune_history=True, blank_skip_threshold=1.0, topk=1, spm_token="▁", stats=None):
    """lp: [T, V] float32 numpy; n: frames to decode.  -> list of (text, text_frames, score)."""
    lp = np.asarray(lp, dtype=np.float32)
    nvocab = len(vocab)
    is_spm = any(str(s).startswith(spm_token) for s in vocab)
    space = -1
    if not is_spm:
        space = vocab.index(space_token) if space_token in vocab else -1
    skip = np.float32(math.log(blank_skip_threshold))
    tok_thr = np.float32(token_prune_min_logp)
    beams = [_Beam("", "", None, None, (), (-1, -1), p_b=0.0, score=0.0, first=True)]
    live, created = [], []
    for f in range(n):
        col = lp[f]
        if col[blank] > skip:
            continue
        order = candidate_order(np.flatnonzero(col > tok_thr).tolist(), int(np.argmax(col)), nvocab)
        cur = list(beams)
        by_text = {}
        for i, b in enumerate(beams):
            by_text.setdefault(b.text, i)
        for t in order:
            p = col[t]
            tok = vocab[t]
            for b in cur:
                sc = np.float32(b.score) + p if b.first else b.score + np.float64(p)
                fold = lae32 if b.first else lae64
                if t == blank:
                    b.n_p_b = fold(b.n_p_b, sc)
                    continue
                if tok == b.last:
                    b.n_p_nb = lae32(b.n_p_nb, np.float32(b.p_nb) + p)
                j = by_text.get(b.text + tok)
                if j is None:
                    if not is_spm and t == space:
                        nb = _Beam(b.text + tok, "", tok, t, b.frames + (b.pf,) if b.part else b.frames, (-1, -1))
                    elif is_spm and tok[:1] == spm_token:
                        nb = _Beam(b.text + " " + tok[1:], tok[1:], tok, t, b.frames + (b.pf,) if b.part else b.frames,
                                   (f, f + 1))
                    elif t == b.lidx:
                        nb = _Beam(b.text + tok, b.part, tok, t, b.frames, (b.pf[0], f + 1))
                    else:
                        nb = _Beam(b.text + tok, b.part + tok, tok, t, b.frames,
                                   (f, f + 1) if b.pf[0] < 0 else (b.pf[0], f + 1))
                    j = len(beams)
                    beams.append(nb)
                    by_text.setdefault(nb.text, j)
                nb = beams[j]
                if t == b.lidx:
                    if b.p_b > NEG:
                        nb.n_p_nb = lae32(nb.n_p_nb, np.float32(b.p_b) + p)
                else:
                    nb.n_p_nb = fold(nb.n_p_nb, sc)
        created.append(len(beams) - len(cur))
        for b in beams:
            b.p_b, b.p_nb, b.n_p_b, b.n_p_nb = b.n_p_b, b.n_p_nb, NEG, NEG
            b.score = lae64(b.p_b, b.p_nb)
            b.first = False
        top = max(b.score for b in beams)
        beams = [b for b in beams if b.score >= top + beam_prune_logp]
        beams = sorted(beams, key=lambda b: b.score, reverse=True)[:beam_size]
        if prune_history:
            seen, kept = set(), []
            for b in beams:
                h = (tuple(b.text.split()[-1:]), b.part, b.last)
                if h not in seen:
                    seen.add(h)
                    kept.append(b)
            beams = kept
        live.append(len(beams))
    if stats is not None:
        stats["live"] = live
        stats["created"] = created
    return finalize([(b.text, b.part, b.frames, b.pf, b.score) for b in beams], beam_size, beam_prune_logp, topk)


def finalize(beams, beam_size, beam_prune_logp, topk):
    """finalize_decoding(force_next_word=True, is_end=True) + the CTCHypothesis list: beams are (text, partial word,
    word frames, partial frames, score)."""
    fin = {}
    for text, part, frames, pf, sc in beams:
        nf = frames + (pf,) if part else frames
        key = merge_words(text, part)
        fin[key] = (text, nf, np.logaddexp(fin[key][2], sc)) if key in fin else (text, nf, sc)
    items = list(fin.values())
    top = max(it[2] for it in items)
    items = [it for it in items if it[2] >= top + beam_prune_logp]
    items = sorted(items, key=lambda it: it[2], reverse=True)[:beam_size]
    return [(" ".join(text.split()), list(zip(text.split(), nf)), sc) for text, nf, sc in items][:topk]


def decode(log_probs, wav_lens, vocab, blank_index, stats_list=None, **kw):
    """decode_beams: log_probs [B, T, V] tensor (any device), wav_lens relative or None."""
    B, T = log_probs.shape[0], log_probs.shape[1]
    lens = frame_lengths(T, wav_lens, B)
    lp = log_probs.detach().float().cpu().numpy()
    out = []
    for b in range(B):
        st = {} if stats_list is not None else None
        out.append(decode_one(lp[b], lens[b], vocab, blank_index, stats=st, **kw))
        if stats_list is not None:
            stats_list.append(st)
    return out
