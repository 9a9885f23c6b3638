"""The fp32 CPU oracle of the Loquacious Conformers (utils/seeded_init.LOQUACIOUS_*: conformer_activation=torch.nn.GELU) on
the inputs of tests/golden/loquacious.pt (generator: tools/make_loquacious_golden.py, which asserts this module equals the
reference on every output).  oracle/asr_oracle.py builds the Conformer with Swish; gelu_conformer() runs its two
Conformer sub-modules that apply conformer_activation (conformer_ffn: both FFN modules; conv_module: after the convolution
module's LayerNorm) with the exact erf GELU, and nothing else.  The decoders are GELU, as asr_oracle builds them."""
import contextlib
import functools
from unittest import mock

import torch
import torch.nn.functional as F

from mirrors import seeded as state  # noqa: F401  (the seed-0 weights the oracle runs on)
from oracle import asr_oracle as O
from oracle.goldens import wav_case

WAV_SEED, LENS, STEPS = 7, [1.0, 0.9, 0.6, 0.3], 48
BLANK, BOS, EOS = 3, 1, 2  # the recipes' blank_index, bos_index, eos_index (pad_index 0)
PREFIX = "Transformer."
# the recipe's test search: S2STransformerBeamSearcher(beam_size=80, temperature=1.15, using_eos_threshold=True) with
# ScorerBuilder(full_scorers=[CTCScorer(blank 3)], weights ctc 0.3, scorer_beam_scale 0.3); the scale only sizes partial
# scorers' candidate lists, and the recipe has none
BEAM = dict(beam=80, ctc_weight=0.3, temperature=1.15, steps=10)
# the reduced-depth cases: every size with 2 encoder layers and 1 decoder layer
REDUCED = dict(num_encoder_layers=2, num_decoder_layers=1)
DYNCHUNK = (16, 2)  # DynChunkTrainConfig(chunk_size=16, left_context_size=2) of the masked-mode case


def sizes():
    from speechbrain_b200.utils import seeded_init as S
    return {c["name"]: c for c in (S.LOQUACIOUS_SMALL, S.LOQUACIOUS_BASE, S.LOQUACIOUS_LARGE, S.LOQUACIOUS_XLARGE)}


def reduced(cfg, **kw):
    return dict(cfg, **REDUCED, **kw)


class _GeluFunctional:
    """torch.nn.functional with silu -> gelu, seen only by the two wrapped oracle functions"""

    def __getattr__(self, name):
        return F.gelu if name == "silu" else getattr(F, name)


def _with_gelu(fn):
    @functools.wraps(fn)
    def run(*args, **kwargs):
        with mock.patch.object(O, "F", _GeluFunctional()):
            return fn(*args, **kwargs)
    return run


@contextlib.contextmanager
def gelu_conformer():
    """a context in which O.encode runs the Conformer with conformer_activation=torch.nn.GELU: O.conformer_ffn and
    O.conv_module (the only two places the Conformer layer applies its activation) see GELU for silu; every other oracle
    function, and torch.nn.functional itself, are untouched"""
    with mock.patch.object(O, "conformer_ffn", _with_gelu(O.conformer_ffn)), \
            mock.patch.object(O, "conv_module", _with_gelu(O.conv_module)):
        yield


def waveforms(seed=WAV_SEED, L=160000, lens=LENS):
    return wav_case(seed, len(lens), L, lens)[:2]


@torch.no_grad()
def encode(cfg, sd, wav, lens, dynchunk=None):
    feats = O.full_pipeline_features(wav, lens, sd, dict(cfg, win_length=cfg["win"] * 1000 // cfg["sample_rate"]))
    with gelu_conformer():
        return O.encode(feats, lens, sd, cfg, PREFIX, dynchunk=dynchunk)


@torch.no_grad()
def greedy(cfg, sd, enc, lens, steps=STEPS):
    """(hyps, log_probs [B, L, V], logits [B, L, V]) of `steps` greedy steps"""
    out = O.greedy_search(enc, lens, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], BOS, EOS, 0.0,
                          (steps + 0.5) / enc.shape[1], PREFIX, return_logits=True)
    return out[0], out[3][:, 0], out[4]


@torch.no_grad()
def beam(cfg, sd, enc, lens, case=BEAM, **extra):
    """O.beam_search with the recipe's test search for case["steps"] steps"""
    ctc = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=case["ctc_weight"], blank_index=BLANK)
    kw = dict(beam_size=case["beam"], max_decode_ratio=(case["steps"] + 0.5) / enc.shape[1])
    kw.update(extra)
    return O.beam_search(enc, lens, sd, cfg, sd["seq_lin.w.weight"], sd["seq_lin.w.bias"], BOS, EOS,
                         temperature=case["temperature"], using_eos_threshold=True, length_normalization=True,
                         prefix=PREFIX, ctc=ctc, **kw)
