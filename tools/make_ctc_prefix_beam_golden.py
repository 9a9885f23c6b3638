"""Generate tests/golden/ctc_prefix_beam.pt by RUNNING THE REFERENCE CTCPrefixBeamSearcher (speechbrain.decoders.ctc, no LM).

How to run it: oracle/goldens.py.  Every case's log-posteriors are regenerated from a seed (tests/ctc_beam_oracle.synthetic_log_probs; the fixture keeps the
seed and a checksum) or, for the Branchformer CTC cases, read from tests/golden/branchformer.pt.  For every case the
script asserts that the NumPy oracle (tests/ctc_prefix_beam_oracle.py) equals the reference exactly: texts, text_frames
and float64 score bits.  It stores the reference hypotheses, the oracle's per-frame live and created beam counts, and the
reference's CPU time per case."""
import time

import numpy as np
import torch

from oracle import goldens as G  # also puts tests/, where the oracles live, on sys.path

import ctc_beam_oracle as CO  # noqa: E402
import ctc_prefix_beam_oracle as PO  # noqa: E402

RECIPE = dict(blank_index=0, beam_size=100, beam_prune_logp=-12.0, token_prune_min_logp=-1.2, prune_history=False)
DEFAULTS = dict(blank_index=0, topk=5)
BLANK_LAST_VOCAB = CO.CHAR_VOCAB[1:] + ["<blank>"]


def vocab_of(name):
    return {"char": CO.CHAR_VOCAB, "spm": CO.spm_vocab(5000, 0), "blank_last": BLANK_LAST_VOCAB}[name]


def case_list():
    spm_active = list(range(11)) + [17, 40, 99, 512, 1024, 2048, 3001, 4099, 4999]
    lens8 = [1.0, 0.9, 0.75, 0.6, 0.5, 0.33, 0.2, 0.1]   # 0.9 * 251 = 225.9: truncation 225, rounding 226
    return [
        dict(name="recipe", vocab="char", params=RECIPE, gen=dict(seed=301, B=8, T=251, V=31), lens=lens8),
        dict(name="defaults", vocab="char", params=DEFAULTS, gen=dict(seed=302, B=8, T=251, V=31), lens=lens8),
        dict(name="spm", vocab="spm", params=dict(blank_index=0, token_prune_min_logp=-5.0, topk=5),
             gen=dict(seed=303, B=4, T=160, V=5000, peak=12.0, active=spm_active), lens=[1.0, 0.8, 0.55, 0.3]),
        dict(name="spm_dup", vocab="spm", params=dict(blank_index=0, prune_history=False, beam_size=50, topk=10,
                                                       token_prune_min_logp=-3.0), dup=True, lens=[1.0]),
        dict(name="skip", vocab="char", params=dict(RECIPE, blank_skip_threshold=0.9, topk=3),
             gen=dict(seed=305, B=4, T=251, V=31, p_blank=0.6), lens=[1.0, 0.8, 0.0, 0.5]),
        dict(name="beam1", vocab="char", params=dict(blank_index=0, beam_size=1, topk=3),
             gen=dict(seed=306, B=4, T=251, V=31), lens=[1.0, 0.9, 0.6, 0.3]),
        dict(name="t1", vocab="char", params=dict(RECIPE, topk=3), gen=dict(seed=307, B=3, T=1, V=31), lens=[1.0, 0.0, 0.99]),
        dict(name="ties", vocab="char", params=dict(RECIPE, beam_size=10, topk=10), tied=dict(B=2, T=4), lens=[1.0, 0.75]),
        dict(name="blank_last", vocab="blank_last", params=dict(DEFAULTS, blank_index=30),
             gen=dict(seed=308, B=4, T=200, V=31, blank=30), lens=[1.0, 0.9, 0.5, 0.2]),
        dict(name="wide", vocab="char", params=dict(RECIPE, topk=3), gen=dict(seed=309, B=3, T=120, V=40),
             lens=[1.0, 0.8, 0.6]),
        dict(name="branchformer_recipe", vocab="char", params=RECIPE, stored=True),
        dict(name="branchformer_defaults", vocab="char", params=DEFAULTS, stored=True),
    ]


def duplicate_text_log_probs():
    """[1, 8, 5000] log-probs on the sentencepiece vocabulary (2 "▁a", 3 "b", 4 "▁ab", 6 "ab") that make beams with
    equal texts coexist (" a" + "b" and "" + "▁ab" both give " ab") and then look that text up again: which of the
    equal-text beams a lookup finds (the first in list order) decides the frames of the result."""
    frames = [{2: -0.7, 0: -0.9, 4: -1.5}, {3: -0.8, 4: -0.9, 0: -1.2}, {3: -0.8, 0: -0.9, 6: -1.3}, {0: -0.5, 3: -1.0}]
    lp = torch.full((1, 2 * len(frames), 5000), -40.0)
    for f, d in enumerate(frames + frames):
        for k, v in d.items():
            lp[0, f, k] = v
    return lp


def case_inputs(case):
    """(log_probs [B, T, V] float32, wav_lens float32) of a fixture case."""
    if case.get("stored"):
        bf = G.load("branchformer.pt")["ctc"]
        return bf["log_probs"].float(), bf["wav_lens"].float()
    if "tied" in case:
        lp = CO.tied_log_probs(**case["tied"])
    elif case.get("dup"):
        lp = duplicate_text_log_probs()
    else:
        g = dict(case["gen"])
        lp = CO.synthetic_log_probs(g.pop("seed"), g.pop("B"), g.pop("T"), g.pop("V"), **g)
    return lp.float(), torch.tensor(case["lens"], dtype=torch.float32)


def as_tuples(hyps):
    return [[(h.text, [(w, (int(a), int(b))) for w, (a, b) in h.text_frames], float(h.score)) for h in hs] for hs in hyps]


def oracle(lp, lens, vocab, params, stats=None):
    kw = {k: v for k, v in params.items() if k != "blank_index"}
    out = PO.decode(lp, lens, vocab, params["blank_index"], stats_list=stats, **kw)
    return [[(t, [(w, (int(a), int(b))) for w, (a, b) in fr], float(sc)) for t, fr, sc in hs] for hs in out]


def main():
    import warnings

    from speechbrain.decoders.ctc import CTCPrefixBeamSearcher
    out = {"cases": []}
    for case in case_list():
        lp, lens = case_inputs(case)
        vocab = vocab_of(case["vocab"])
        searcher = CTCPrefixBeamSearcher(vocab_list=vocab, **case["params"])
        t0 = time.perf_counter()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            ref = as_tuples(searcher(lp, lens))
        t_ref = time.perf_counter() - t0
        stats = []
        ora = oracle(lp, lens, vocab, case["params"], stats)
        assert ref == ora, case["name"]
        live = [s.get("live", []) for s in stats]
        created = [s.get("created", []) for s in stats]
        print(f"[{case['name']}] B={lp.shape[0]} T={lp.shape[1]} V={lp.shape[2]}: reference {t_ref:.2f} s on the CPU; "
              f"max live beams {max((max(v) for v in live if v), default=0)}, "
              f"mean {np.mean([x for v in live for x in v] or [0]):.1f}; created {sum(sum(c) for c in created)}; "
              f"best {[h[0][0][:40] if h else None for h in ref]}")
        entry = dict(name=case["name"], vocab=case["vocab"], params=case["params"], hyps=ref, live=live, created=created,
                     ref_cpu_seconds=t_ref, checksum=float(lp.double().abs().sum()))
        for k in ("gen", "tied", "dup", "lens", "stored"):
            if k in case:
                entry[k] = case[k]
        out["cases"].append(entry)
    G.save(out, "ctc_prefix_beam.pt")


if __name__ == "__main__":
    main()
