"""Generate tests/golden/switchboard.pt by RUNNING THE REFERENCE's Switchboard transformer.yaml recipe on seeded weights (how
to run it: oracle/goldens.py).

* lm: the recipe's lm_model, TransformerLM(vocab 2000, d_model 264, d_embedding 128, 12 heads, 12 layers, d_ffn 1024, ReLU,
  post-norm; seeded_init seed 1), TransformerLM.forward on 6 ragged sequences padded with 0 that also hold id 0 inside
  their valid lengths: per position the logsumexp and the top-8 logits / ids, and the full rows of sampled positions;
* asr: SWITCHBOARD_TRANSFORMER (speechbrain_b200.utils.seeded_init, seed 0), 4 x 10 s ragged waveforms [1.0, 0.9, 0.6, 0.3]
  -> Fbank -> CMVN -> 3-block CNN -> encoder states at d_model 256 (T = 251), then 48 greedy steps;
* beam60: on those encoder states, the recipe's test search: beam 60, temperature 1.0, no EOS threshold, length
  normalisation, ScorerBuilder(full_scorers=[TransformerLMScorer(temperature 1.0), CTCScorer], weights transformerlm 0.3,
  ctc 0.3, scorer_beam_scale 0.3) over 16 steps;
* both modules' state_dict key -> shape lists.

The tests recompute the LM with tests/switchboard_oracle.py and the encoder with tests/transformer_oracle.py, which this
script asserts equal the reference (rel-L2 < 1e-5).  Weights and waveforms are regenerated from their seeds.
"""
import torch

from oracle import goldens as G
from speechbrain_b200.utils.seeded_init import SWITCHBOARD_LM, SWITCHBOARD_TRANSFORMER

HEAD = (0, 1, 2, 3)
LM_SEED = 1
LENGTHS = [80, 1, 37, 64, 65, 12]
INTERIOR_PAD = [(0, 5), (0, 40), (0, 70), (3, 20), (4, 64)]  # (sequence, position) holding id 0 inside the valid length


def reference_lm():
    from speechbrain.lobes.models.transformer.TransformerLM import TransformerLM

    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    lm = TransformerLM(**SWITCHBOARD_LM, dropout=0.0, activation=torch.nn.ReLU)
    sd = seeded_state_dict(lm, seed=LM_SEED)
    lm.load_state_dict(sd)
    lm.eval()
    return lm, sd


def lm_case(lm, sd):
    import switchboard_oracle as SO
    g = torch.Generator().manual_seed(2025)
    n, s = len(LENGTHS), max(LENGTHS)
    tokens = torch.zeros(n, s, dtype=torch.long)
    for i, L in enumerate(LENGTHS):
        tokens[i, 0] = 1
        if L > 1:
            tokens[i, 1:L] = torch.randint(3, 2000, (L - 1,), generator=g)
    for i, p in INTERIOR_PAD:
        tokens[i, p] = 0
    with torch.no_grad():
        ref = lm(tokens)
        ours = SO.lm_forward(tokens, sd)
    err = max(G.rel(ours[i], ref[i]) for i in range(n))
    print(f"[switchboard lm] logits {tuple(ref.shape)} oracle rel err (worst sequence) {err:.2e}")
    assert err < 1e-5 and torch.isfinite(ref).all()
    top_v, top_i = ref.topk(8, dim=-1)
    pos = sorted({(i, L - 1) for i, L in enumerate(LENGTHS)} | {(0, 0), (0, 40), (0, 41), (3, 21), (1, 40), (5, 79)})
    idx = torch.tensor(pos, dtype=torch.long)
    return dict(tokens=tokens.to(torch.int32), lengths=torch.tensor(LENGTHS, dtype=torch.int32),
                logsumexp=ref.logsumexp(-1).clone(), top_values=top_v.clone(), top_ids=top_i.to(torch.int32),
                sample_idx=idx.to(torch.int32), sample_logits=ref[idx[:, 0], idx[:, 1]].clone(), seed=LM_SEED)


@torch.no_grad()
def beam60_case(ref, lm, enc, wav_lens, steps=16):
    from speechbrain.decoders.scorer import CTCScorer, ScorerBuilder, TransformerLMScorer
    from speechbrain.decoders.seq2seq import S2STransformerBeamSearcher
    T = enc.shape[1]
    kwargs = dict(beam_size=60, temperature=1.0, using_eos_threshold=False, eos_threshold=1.5, length_normalization=True,
                  min_decode_ratio=0.0)
    scorer = ScorerBuilder(full_scorers=[TransformerLMScorer(language_model=lm, temperature=1.0),
                                         CTCScorer(eos_index=2, blank_index=0, ctc_fc=ref.mods["ctc_lin"])],
                           weights=dict(transformerlm=0.3, ctc=0.3), scorer_beam_scale=0.3)
    bs = S2STransformerBeamSearcher(modules=[ref.mods["Transformer"], ref.mods["seq_lin"]], bos_index=1, eos_index=2,
                                    max_decode_ratio=(steps + 0.5) / T, scorer=scorer, **kwargs)
    hyps, _, scores, lp = bs(enc, wav_lens)
    print(f"[switchboard beam60 lm+ctc] hyps lengths {[len(h) for h in hyps]} scores {scores.tolist()}")
    return dict(kwargs=kwargs, max_decode_ratio=(steps + 0.5) / T, lm_weight=0.3, lm_temperature=1.0, ctc_weight=0.3,
                hyps=hyps, scores=scores.clone(), log_probs=lp.clone())


def main():
    import transformer_oracle as TO

    cfg = SWITCHBOARD_TRANSFORMER
    lm, sd_lm = reference_lm()
    ref = G.build_reference(cfg, cnn_blocks=3, encoder_module="transformer", positional_encoding="fixed_abs_sine")
    out = dict(weight_seed=0, keys=dict(cnn=ref.keys("CNN"), transformer=ref.keys(),
                                        lm=[(k, tuple(v.shape)) for k, v in lm.state_dict().items()]))
    out["lm"] = lm_case(lm, sd_lm)
    B = 4
    wav, wav_lens, res = G.wav_case(2470, B, 160000, [1.0, 0.9, 0.6, 0.3])
    cnn = ref.cnn(wav, wav_lens)
    with torch.no_grad():
        enc = ref.mods["Transformer"].encode(cnn, wav_lens)
        oenc = TO.encode(TO.wav_to_cnn(wav, wav_lens, ref.sd, cfg), wav_lens, ref.sd, cfg)
    T = enc.shape[1]
    print(f"[switchboard] enc T={T} oracle rel {G.rel(oenc, enc):.2e}")
    assert enc.shape == (B, 251, 256) and G.rel(oenc, enc) < 1e-5
    abs_len = torch.round(wav_lens * T).int()
    res.update(abs_len=abs_len, enc=G.frame_summary(enc, abs_len, HEAD))
    res.update(G.greedy_record(*G.greedy_case(ref, enc, wav_lens, 48, "switchboard"), chosen_lp=False))
    out["asr"] = res
    out["beam60"] = beam60_case(ref, lm, enc, wav_lens)
    G.save(out, "switchboard.pt")


if __name__ == "__main__":
    main()
