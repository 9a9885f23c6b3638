"""fp32 CPU restatement of TransducerBeamSearcher.transducer_beam_search_decode (speechbrain/decoders/transducer.py:320-
476) without a language model, on the prediction network, joint and classifier of tests/transducer_oracle.Oracle.

``search`` walks one utterance as the reference does: per frame, pop the first hypothesis of the list with the largest
key score / len(prediction), stop when the beam holds beam_size hypotheses or when the beam's best raw score is state_beam
above the popped one's, extend by the top beam_size tokens (blank -> beam, a token within expand_beam of the best
non-blank -> the list).  Scores are fp32 sums in the reference's order.  It records the smallest margin of every kind of
comparison it made, so a test knows how far a decision was from flipping.

``replay`` walks one utterance along a device trace instead (the popped hypothesis, the top-K tokens, the kept children
and the frame ends the device chose) and reports, at every decision, the oracle's own choice and its margin."""
import math

import torch

import transducer_oracle as TO

KINDS = ("key", "topk", "expand", "state", "sort")


def _key(h):
    return h["score"] / len(h["pred"])


def _argmax_key(hyps):
    """index of the first live hypothesis with the largest key (Python max), and the gap to the runner-up key"""
    best, bk, second = None, None, -math.inf
    for i, h in enumerate(hyps):
        if h is None:
            continue
        k = float(_key(h))
        if best is None or k > bk:
            if best is not None:
                second = max(second, bk)
            best, bk = i, k
        else:
            second = max(second, k)
    return best, bk, bk - second


def _flip_margin(proc, beam, sb, outcome, m):
    """How far the state_beam test was from giving ``outcome``: m (its own margin), or, when the test gives outcome for a
    hypothesis of the list and one of the beam whose keys are within g of the largest, the smallest such g"""
    def gaps(hyps):
        keys = [(float(_key(h)), h) for h in hyps if h is not None]
        top = max(k for k, _ in keys)
        return [(top - k, h) for k, h in keys]
    for ga, a in gaps(proc):
        for gb, b in gaps(beam):
            if bool(b["score"] >= sb + a["score"]) == outcome:
                m = min(m, max(ga, gb))
    return m


class BeamOracle:
    def __init__(self, W):
        self.o = TO.Oracle(W)
        self.H = self.o.H

    def _pn(self, h):
        """(out_PN, h, c) of the hypothesis' next PN step, cached on it (a blank child shares its parent's)"""
        if h["pn"] is None:
            st = h["state"]
            if st is None:
                z = torch.zeros(self.H)
                st = (z, z.clone())
            h["pn"] = self.o.pn(h["pred"][-1], st[0], st[1])
        return h["pn"]

    @torch.no_grad()
    def search(self, tn, blank, K, nbest, state_beam, expand_beam, replay=None):
        """tn [T, J] of one utterance.  Returns dict(hyps, scores (normalised), pops, max_pops_per_frame, margins {kind:
        smallest}, trace (one dict per pop: frame, hyp, tokens, kept, score -- the popped hypothesis' raw score), and with
        replay: issues [(kind, record index, margin)] and raw (per record, the popped hypothesis' oracle raw score and
        the number of log-probabilities it sums: its tokens and one blank per earlier frame)).  replay: the utterance's
        pops in the same form (a device trace, see read_trace)."""
        margins = {k: math.inf for k in KINDS}
        issues, raw, trace = [], [], []
        beam = [dict(pred=[blank], score=torch.zeros(()), state=None, pn=None)]
        pops, max_pf, ri = 0, 0, 0
        sb, eb = torch.tensor(state_beam, dtype=torch.float32), torch.tensor(expand_beam, dtype=torch.float32)

        def note(kind, m, rec=None, differs=False):
            margins[kind] = min(margins[kind], abs(m))
            if differs:
                issues.append((kind, rec, abs(m)))

        for t in range(tn.shape[0]):
            proc, beam, pf = beam[:], [], 0
            while len(beam) < K:
                ia, ka, gap = _argmax_key(proc)
                rec = replay[ri] if replay is not None and ri < len(replay) else None
                if len(beam) > 0:
                    b = max(beam, key=_key)
                    a_score = proc[ia]["score"]
                    stop = bool(b["score"] >= sb + a_score)
                    m = float(b["score"] - (sb + a_score))
                    if replay is not None:
                        dev_stop = rec is None or rec["frame"] != t
                        if stop != dev_stop:   # the test may compare other hypotheses after a near-tie of keys
                            m = _flip_margin(proc, beam, sb, dev_stop, abs(m))
                        note("state", m, ri, stop != dev_stop)
                        stop = dev_stop
                    else:
                        note("state", m)
                    if stop:
                        break
                if replay is not None:
                    assert rec is not None and rec["frame"] == t, (ri, t)
                    if rec["hyp"] != ia:
                        note("key", ka - float(_key(proc[rec["hyp"]])), ri, True)
                    elif math.isfinite(gap):
                        note("key", gap)
                    ia = rec["hyp"]
                elif math.isfinite(gap):
                    note("key", gap)
                a = proc[ia]
                proc[ia] = None
                pops, pf = pops + 1, pf + 1
                p, h, c = self._pn(a)
                lp = self.o.logp(tn[t].float(), p)
                top = lp.topk(min(K + 1, lp.numel()))
                vals, pos = top.values[:K], top.indices[:K].tolist()
                if lp.numel() > K:
                    note("topk", float(top.values[K - 1] - top.values[K]))
                if replay is not None:
                    raw.append((float(a["score"]), len(a["pred"]) - 1 + t))
                    if set(rec["tokens"]) != set(pos):
                        note("topk", float(top.values[K - 1] - top.values[K]) if lp.numel() > K else 0.0, ri, True)
                    pos = list(rec["tokens"])
                    vals = lp[pos]
                best = vals[0] if pos[0] != blank else vals[1]
                kept = 0
                for j in range(K):
                    child = dict(pred=a["pred"][:], score=a["score"] + vals[j], state=a["state"], pn=a["pn"])
                    if pos[j] == blank:
                        beam.append(child)
                        kept |= 1 << j
                        continue
                    keep = bool(vals[j] >= best - eb)
                    m = float(vals[j] - (best - eb))
                    if replay is not None:
                        dev_keep = bool(rec["kept"] >> j & 1)
                        note("expand", m, ri, keep != dev_keep)
                        keep = dev_keep
                    else:
                        note("expand", m)
                    if keep:
                        kept |= 1 << j
                        child["pred"].append(pos[j])
                        child["state"], child["pn"] = (h, c), None
                        proc.append(child)
                trace.append(dict(frame=t, hyp=ia, tokens=list(pos), kept=kept, score=float(a["score"])))
                ri += 1
            max_pf = max(max_pf, pf)
        keys = [float(_key(h)) for h in beam]
        order = sorted(range(len(beam)), key=lambda i: keys[i], reverse=True)
        for r in range(min(nbest, len(order) - 1)):
            note("sort", keys[order[r]] - keys[order[r + 1]])
        best = [beam[i] for i in order[:nbest]]
        out = dict(hyps=[h["pred"][1:] for h in best], scores=[float(h["score"] / len(h["pred"])) for h in best],
                   pops=pops, max_pops_per_frame=max_pf, margins=margins, trace=trace)
        if replay is not None:
            assert ri == len(replay), (ri, len(replay))
            out.update(issues=issues, raw=raw)
        return out

    @staticmethod
    def read_trace(trace, b, K):
        """utterance b's records of a device trace [B, records, 6 + 2K] int32 (sbk_transducer_beam) as search's dicts"""
        rows = trace[b]
        rows = rows[rows[:, 0] >= 0]
        lp = rows[:, 6 + K:].contiguous().view(torch.float32)
        sc = rows[:, 5].contiguous().view(torch.float32)
        return [dict(frame=int(r[1]), hyp=int(r[2]), ended=int(r[3]), kept=int(r[4]) & 0xffffffff, score=float(sc[i]),
                     tokens=r[6:6 + K].tolist(), logp=lp[i].tolist()) for i, r in enumerate(rows)]

    def batch(self, tn, blank, K, nbest, state_beam=2.3, expand_beam=2.3):
        """every utterance of tn [B, T, J]: (best hyps, exp(best scores).mean(), nbest hyps, nbest scores, per-utterance
        results), the reference's return value followed by the walks"""
        rows = [self.search(tn[b], blank, K, nbest, state_beam, expand_beam) for b in range(tn.shape[0])]
        best = torch.tensor([r["scores"][0] for r in rows], dtype=torch.float32)
        return ([r["hyps"][0] for r in rows], best.exp().mean(), [r["hyps"] for r in rows], [r["scores"] for r in rows],
                rows)
