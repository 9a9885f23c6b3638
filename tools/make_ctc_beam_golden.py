"""Generate tests/golden/ctc_beam.pt by RUNNING THE REFERENCE CTCBeamSearcher (speechbrain.decoders.ctc, no LM).

How to run it: oracle/goldens.py.  Every case's log-posteriors are regenerated from a seed (tests/ctc_beam_oracle.synthetic_log_probs; the fixture keeps the
seed and a checksum) or, for the Branchformer CTC cases, read from tests/golden/branchformer.pt.  For every case the
script asserts that the NumPy oracle (tests/ctc_beam_oracle.py) equals the reference: texts and text_frames identical,
scores bit-equal, except where two hypotheses' scores tie exactly (reported).  It stores the reference hypotheses, the
oracle's per-frame live-beam and merge counts (evidence that the beam fills and merges happen) and the reference's CPU
time per case."""
import time

import numpy as np
import torch

from oracle import goldens as G  # also puts tests/, where the oracles live, on sys.path

import ctc_beam_oracle as CO  # noqa: E402

RECIPE = dict(blank_index=0, beam_size=100, beam_prune_logp=-12.0, token_prune_min_logp=-1.2, prune_history=False)
DEFAULTS = dict(blank_index=0, topk=5)


def case_list():
    spm = CO.spm_vocab(5000, 0)
    spm_active = list(range(11)) + [17, 40, 99, 512, 1024, 2048, 3001, 4999]
    bf = G.load("branchformer.pt")["ctc"]
    lens8 = [1.0, 0.9, 0.75, 0.6, 0.5, 0.33, 0.2, 0.1]   # 0.9 * 251 = 225.9: truncation 225, rounding 226
    return [
        dict(name="recipe", vocab=CO.CHAR_VOCAB, params=RECIPE, gen=dict(seed=101, B=8, T=251, V=31), lens=lens8),
        dict(name="defaults", vocab=CO.CHAR_VOCAB, params=DEFAULTS, gen=dict(seed=102, B=8, T=251, V=31), lens=lens8),
        dict(name="spm", vocab=spm, params=dict(blank_index=0, token_prune_min_logp=-5.0, topk=5),
             gen=dict(seed=103, B=4, T=251, V=5000, peak=12.0, active=spm_active), lens=[1.0, 0.8, 0.55, 0.3]),
        dict(name="skip", vocab=CO.CHAR_VOCAB, params=dict(RECIPE, blank_skip_threshold=0.9, topk=3),
             gen=dict(seed=104, B=4, T=251, V=31, p_blank=0.6), lens=[1.0, 0.8, 0.0, 0.5]),
        dict(name="beam1", vocab=CO.CHAR_VOCAB, params=dict(blank_index=0, beam_size=1, topk=3),
             gen=dict(seed=105, B=4, T=251, V=31), lens=[1.0, 0.9, 0.6, 0.3]),
        dict(name="t1", vocab=CO.CHAR_VOCAB, params=dict(RECIPE, topk=3), gen=dict(seed=106, B=3, T=1, V=31),
             lens=[1.0, 0.0, 0.99]),
        dict(name="ties", vocab=CO.CHAR_VOCAB, params=dict(RECIPE, beam_size=10, topk=10), tied=dict(B=2, T=4), lens=[1.0, 0.75]),
        dict(name="branchformer_recipe", vocab=CO.CHAR_VOCAB, params=RECIPE, stored=bf["log_probs"], lens=bf["wav_lens"].tolist()),
        dict(name="branchformer_defaults", vocab=CO.CHAR_VOCAB, params=DEFAULTS, stored=bf["log_probs"],
             lens=bf["wav_lens"].tolist()),
    ]


def case_inputs(case):
    """(log_probs [B, T, V] float32, wav_lens float32) of a fixture case."""
    if "stored" in case:
        lp = case["stored"]
    elif "tied" in case:
        lp = CO.tied_log_probs(**case["tied"])
    else:
        g = dict(case["gen"])
        lp = CO.synthetic_log_probs(g.pop("seed"), g.pop("B"), g.pop("T"), g.pop("V"), **g)
    return lp.float(), torch.tensor(case["lens"], dtype=torch.float32)


def compare(name, ref, ora):
    """texts / frames identical and scores bit-equal, except inside exact score ties; returns the tie report."""
    ties = []
    for b, (hr, ho) in enumerate(zip(ref, ora)):
        assert len(hr) == len(ho), (name, b, len(hr), len(ho))
        for r, (x, y) in enumerate(zip(hr, ho)):
            assert np.float32(x[2]) == np.float32(y[2]), (name, b, r, x[2], y[2])
            if (x[0], x[1]) != (y[0], y[1]):
                tied = [i for i, h in enumerate(hr) if np.float32(h[2]) == np.float32(x[2])]
                assert len(tied) > 1 and any((hr[i][0], hr[i][1]) == (y[0], y[1]) for i in tied), (name, b, r, x, y)
                ties.append((b, r))
    return ties


def main():
    from speechbrain.decoders.ctc import CTCBeamSearcher
    out = {"cases": []}
    for case in case_list():
        lp, lens = case_inputs(case)
        searcher = CTCBeamSearcher(vocab_list=case["vocab"], **case["params"])
        t0 = time.perf_counter()
        ref = CO.as_tuples(searcher(lp, lens))
        t_ref = time.perf_counter() - t0
        stats = []
        kw = {k: v for k, v in case["params"].items() if k != "blank_index"}
        ora = CO.as_tuples(CO.decode(lp, lens, case["vocab"], case["params"]["blank_index"], stats_list=stats, **kw))
        ties = compare(case["name"], ref, ora)
        live = [s.get("live", []) for s in stats]
        merges = [s.get("merges", []) for s in stats]
        print(f"[{case['name']}] B={lp.shape[0]} T={lp.shape[1]} V={lp.shape[2]}: reference {t_ref:.2f} s on the CPU; "
              f"max live beams {max((max(v) for v in live if v), default=0)}, mean {np.mean([x for v in live for x in v] or [0]):.1f}; "
              f"merges {sum(sum(m) for m in merges)}; exact-tie rank swaps {ties}; best {[h[0][0][:40] for h in ref]}")
        hyps = [[(t, [(w, (int(a), int(b))) for w, (a, b) in fr], float(sc)) for t, fr, sc in hs] for hs in ref]  # plain types
        entry = dict(name=case["name"], params=case["params"], lens=[float(x) for x in case["lens"]], hyps=hyps, live=live, merges=merges, ties=ties,
                     ref_cpu_seconds=t_ref, checksum=float(lp.double().abs().sum()))
        entry["vocab"] = "char" if case["vocab"] is CO.CHAR_VOCAB else "spm"
        if "gen" in case:
            entry["gen"] = case["gen"]
        elif "tied" in case:
            entry["tied"] = case["tied"]
        else:
            entry["stored"] = "branchformer.pt:ctc.log_probs"
        out["cases"].append(entry)
    G.save(out, "ctc_beam.pt")


if __name__ == "__main__":
    main()
