"""CPU oracle of CTCBeamSearcher without a language model (speechbrain.decoders.ctc, v1.1.0), restated in NumPy float32.

A beam is (text, partial word, last token, word frames, partial frames, score), keyed by the strings
(text, partial word, last token).  Per frame f < length:
  * skip the frame when lp[blank] > float32(log(blank_skip_threshold));
  * candidate tokens: lp[t] > float32(token_prune_min_logp), plus the arg-max (first index on ties), restricted to
    t < len(vocab_list), walked in ASCENDING order (beams in rank order inside a token);
  * blank or the last token's string repeated: only the last token (and, for a repeat, the partial word's end frame)
    changes; a sentencepiece word start commits the partial word (merge: "a" + " " + "b", empty sides dropped) and starts
    token[1:]; outside sentencepiece mode the space token commits it; any other token is appended;
  * equal keys merge: np.logaddexp of the scores in candidate order, the first candidate's position, the last one's frames;
  * keep score >= max + beam_prune_logp (float32), then the beam_size best, ties in position order;
  * with prune_history, the first beam per (last word of the text, partial word, last token).
At the end every beam commits its partial word, the beams merge by text, and the prune and sort run once more; the top
``topk`` are returned with whitespace normalised and ``text_frames = zip(text.split(), word frames)``.

Lengths are ``(T * wav_lens)`` in the tensor's dtype truncated by ``astype(int)`` and used as a Python slice bound.
All scores stay float32 (NumPy 2 keeps ``python float + np.float32`` in float32); a beam that saw no frame scores 0.0.
``stats`` (optional dict) receives per-frame live-beam counts and merge counts."""
import math

import numpy as np


def frame_lengths(T, wav_lens, B):
    """decode_beams' lengths: None -> T each; else (T * wav_lens) truncated, then the number of frames a slice [:n] keeps."""
    if wav_lens is None:
        raw = [T] * B
    else:
        raw = (T * wav_lens).cpu().numpy().astype(int).tolist()
    return [len(range(T)[:n]) for n in raw]


def merge_words(a, b):
    if not b:
        return a
    if not a:
        return b
    return a + " " + b


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
    bp = np.float32(beam_prune_logp)
    # (text, partial, last, frames, pf, score)
    beams = [("", "", None, (), (-1, -1), 0.0)]
    live, merges = [], []
    for f in range(n):
        col = lp[f]
        if col[blank] > skip:
            continue
        toks = set(np.flatnonzero(col > tok_thr).tolist())
        toks.add(int(np.argmax(col)))
        toks = sorted(t for t in toks if t < nvocab)
        cand = {}
        ncand = 0
        for t in toks:
            p = col[t]
            tok = vocab[t]
            for text, part, last, frames, pf, sc in beams:
                s = sc + p
                if t == blank or last == tok:
                    key = (text, part, tok)
                    ent = (frames, pf if t == blank else (pf[0], f + 1))
                elif is_spm and tok[:1] == spm_token:
                    key = (merge_words(text, part), tok[1:], tok)
                    ent = (frames + (pf,) if part else frames, (f, f + 1))
                elif not is_spm and t == space:
                    key = (merge_words(text, part), "", tok)
                    ent = (frames + (pf,) if part else frames, (-1, -1))
                else:
                    key = (text, part + tok, tok)
                    ent = (frames, (f, f + 1) if pf[0] < 0 else (pf[0], f + 1))
                ncand += 1
                if key in cand:
                    cand[key] = (np.logaddexp(cand[key][0], s), ent)
                else:
                    cand[key] = (s, ent)
        items = [(s, key, ent) for key, (s, ent) in cand.items()]
        top = max(it[0] for it in items)
        items = [it for it in items if it[0] >= top + bp]
        items = sorted(items, key=lambda it: it[0], reverse=True)[:beam_size]
        if prune_history:
            seen, kept = set(), []
            for it in items:
                h = (tuple(it[1][0].split()[-1:]), it[1][1], it[1][2])
                if h not in seen:
                    seen.add(h)
                    kept.append(it)
            items = kept
        beams = [(key[0], key[1], key[2], ent[0], ent[1], s) for s, key, ent in items]
        live.append(len(beams))
        merges.append(ncand - len(cand))
    if stats is not None:
        stats["live"] = live
        stats["merges"] = merges
    return finalize(beams, beam_size, bp, topk)


def finalize(beams, beam_size, bp, topk):
    """finalize_decoding(force_next_word=True, is_end=True) + the CTCHypothesis list of decode_log_probs."""
    fin = {}
    for text, part, last, frames, pf, sc in beams:
        nf = frames + (pf,) if part else frames
        key = merge_words(text, part)
        if key in fin:
            fin[key] = (np.logaddexp(fin[key][0], sc), nf)
        else:
            fin[key] = (sc, nf)
    items = [(s, text, nf) for text, (s, nf) in fin.items()]
    top = max(it[0] for it in items)
    items = [it for it in items if it[0] >= top + np.float32(bp)]
    items = sorted(items, key=lambda it: it[0], reverse=True)[:beam_size]
    return [(" ".join(text.split()), list(zip(text.split(), nf)), s) for s, text, nf in items][:topk]


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


def as_tuples(hyps):
    """Reference CTCHypothesis lists (or this module's tuples) -> [[(text, text_frames, score)]]."""
    out = []
    for hs in hyps:
        out.append([(h.text, [tuple(x) for x in h.text_frames], h.score) if hasattr(h, "text") else
                    (h[0], [tuple(x) for x in h[1]], h[2]) for h in hs])
    return out



# ------------------------------------------------------------------------------------------- seeded test inputs
# The LibriSpeech character CTC vocabulary layout: blank 0, space 1, then 29 symbols (31 outputs).
CHAR_VOCAB = ["<blank>", " "] + list("ETAOINSHRDLUCMFWYPVBGKQJXZ") + ["'", "-", "."]


def spm_vocab(V=5000, seed=0):
    """Sentencepiece-style pieces: blank "<unk>" at 0, a bare "▁", pieces whose concatenations coincide ("▁a" + "b" and
    "▁ab", "a" + "b" and "ab"), one duplicated piece (two ids, one string), then seeded random pieces up to V."""
    import random
    rng = random.Random(seed)
    vocab = ["<unk>", "▁", "▁a", "b", "▁ab", "a", "ab", "▁b", "▁abb", "bb", "b"]
    seen = set(vocab)
    while len(vocab) < V:
        p = ("▁" if rng.random() < 0.5 else "") + "".join(rng.choice("abcdefghijklmnopqrst") for _ in range(rng.randint(1, 4)))
        if p not in seen:
            seen.add(p)
            vocab.append(p)
    return vocab


def synthetic_log_probs(seed, B, T, V, blank=0, active=None, peak=9.0, p_blank=0.45):
    """Peaked CTC log-posteriors [B, T, V] float32: per frame one dominant token (the blank with probability p_blank),
    a second strong alternative on 60 % of the frames and a third on 25 %, over low noise; tokens are drawn from
    ``active`` (default: all), so that beams fill and merge."""
    import torch
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, V, generator=g) * 0.7
    act = torch.arange(V) if active is None else torch.as_tensor(active)

    def pick():
        return act[torch.randint(len(act), (B, T), generator=g)]
    dom = torch.where(torch.rand(B, T, generator=g) < p_blank, torch.full((B, T), blank), pick())
    x.scatter_add_(2, dom[..., None], torch.full((B, T, 1), peak))
    for prob, lo, hi in ((0.6, 0.0, 2.0), (0.25, 0.5, 3.0)):
        alt = torch.where(torch.rand(B, T, generator=g) < 0.3, torch.full((B, T), blank), pick())
        on = torch.rand(B, T, generator=g) < prob
        gap = lo + (hi - lo) * torch.rand(B, T, generator=g)
        x.scatter_add_(2, alt[..., None], torch.where(on, peak - gap, torch.zeros(B, T))[..., None])
    return torch.log_softmax(x, dim=-1).float()


def tied_log_probs(B, T, V=31, tied=(2, 3, 4, 5, 6, 7)):
    """Exact float32 score ties: every frame gives the ``tied`` tokens log-probability -1.0 and every other token -30, so
    many different texts end with bit-identical scores and only the position order decides which beams survive."""
    import torch
    x = torch.full((B, T, V), -30.0)
    x[..., list(tied)] = -1.0
    return x
