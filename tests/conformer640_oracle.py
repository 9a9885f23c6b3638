"""The fp32 CPU oracle of the d_model 640 Conformer recipes (utils/seeded_init.CONFORMER_640 / CONFORMER_640_PEOPLES) on the
inputs of tests/golden/conformer640.pt (generator: tools/make_conformer640_golden.py, which asserts this module equals the
reference on every output).  oracle/asr_oracle.py builds the decoder FFN with GELU or ReLU; the People's Speech decoder's
Swish FFN is its decode() with SiLU in place of GELU (swish_decoder)."""
import contextlib
from unittest import mock

import torch
import torch.nn.functional as F

from mirrors import seeded as state  # noqa: F401  (the seed-0 weights the oracle runs on)
from oracle import asr_oracle as O
from oracle.goldens import wav_case
from parity import lm_scorer_state, oracle_lm

WAV_SEED, LENS, STEPS, BOS, EOS = 7, [1.0, 0.9, 0.6, 0.3], 48, 1, 2
PREFIX = "Transformer."


def waveforms(seed=WAV_SEED, L=160000, lens=LENS):
    return wav_case(seed, len(lens), L, lens)[:2]


def swish_decoder(cfg):
    """a context in which O.decode (and so O.greedy_search / O.beam_search) runs the config's decoder FFN"""
    if cfg["decoder_activation"] != "swish":
        return contextlib.nullcontext()
    orig = O.decode

    def decode(tgt, enc_out, enc_len, sd, c, prefix=""):
        with mock.patch.object(O.F, "gelu", F.silu):
            return orig(tgt, enc_out, enc_len, sd, dict(c, decoder_activation="gelu"), prefix)
    return mock.patch.object(O, "decode", decode)


@torch.no_grad()
def encode(cfg, sd, wav, lens):
    feats = O.full_pipeline_features(wav, lens, sd, dict(cfg, win_length=cfg["win"] * 1000 // cfg["sample_rate"]))
    return O.encode(feats, lens, sd, cfg, PREFIX)


@torch.no_grad()
def greedy(cfg, sd, enc, lens, ratio=None):
    """(hyps, log_probs [B, L, V], logits [B, L, V]) of STEPS greedy steps (ratio: max_decode_ratio instead)"""
    ratio = (STEPS + 0.5) / enc.shape[1] if ratio is None else ratio
    with swish_decoder(cfg):
        out = O.greedy_search(enc, lens, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], BOS, EOS, 0.0, ratio, PREFIX,
                              return_logits=True)
    return out[0], out[3][:, 0], out[4]


def teacher_tokens(cfg, n=4):
    g = torch.Generator().manual_seed(3)
    tgt = torch.randint(3, cfg["vocab"], (n, STEPS), generator=g)
    tgt[:, 0] = BOS
    return tgt


@torch.no_grad()
def decode(cfg, sd, tgt, enc, abs_len):
    with swish_decoder(cfg):
        return O.decode(tgt, enc, abs_len, sd, cfg, PREFIX)[0]


def lm_scorer(cfg):
    return lm_scorer_state(cfg["vocab"])


@torch.no_grad()
def beam(cfg, sd, enc, lens, case, **extra):
    """O.beam_search with the recipe's test search of a fixture beam case (dict(beam, lm_weight, ctc_weight, steps))"""
    lm = oracle_lm(case["lm_weight"], 1.15, cfg["vocab"]) if case["lm_weight"] else None
    ctc = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=case["ctc_weight"], blank_index=0)
    kw = dict(beam_size=case["beam"], max_decode_ratio=(case["steps"] + 0.5) / enc.shape[1])
    kw.update(extra)
    with swish_decoder(cfg):
        return O.beam_search(enc, lens, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], BOS, EOS, temperature=1.15,
                             using_eos_threshold=False, length_normalization=True, prefix=PREFIX, lm=lm, ctc=ctc, **kw)
