"""The device-side modules of the parity tests, built once: speechbrain_b200's Fbank, global CMVN, CNN front end,
TransformerASR, seq_lin and ctc_lin of a recipe config (utils/seeded_init) holding a seeded flat state, and the assemblies
the tests wire from them.  It is the counterpart of oracle.goldens.build_reference, which builds the reference's modules
from the same config and state.

Test modules and tools import it the way they import parity.py (tests/ on sys.path)."""
import functools

import torch

from parity import lm_scorer

BOS, EOS = 1, 2
LM_TEMPERATURE = 1.15


@functools.lru_cache(maxsize=4)
def _seeded(items, seed):
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    return seeded_asr_state(dict(items), seed)


def seeded(cfg, seed=0, transform=None):
    """seeded_asr_state(cfg, seed), cached on the whole config (a name is not a key: the reduced Loquacious configs keep
    their full model's), as a new dict on every call so that callers may replace entries; transform(sd) rescales it"""
    sd = dict(_seeded(tuple(sorted(cfg.items())), seed))
    return sd if transform is None else transform(sd)


def _positional_table(key):
    owner, name = ("." + key).split(".")[-2:]
    return owner.startswith("positional_encoding") and name in ("pe", "inv_freq")


def load(module, sd, prefix):
    """module loaded with the entries of sd under prefix; no entry may be unexpected, and only the positional-encoding
    tables (buffers the module computes itself) may be missing.  Returns the module."""
    res = module.load_state_dict({k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}, strict=False)
    missing = [k for k in res.missing_keys if not _positional_table(k)]
    assert not res.unexpected_keys and not missing, (prefix, res.unexpected_keys, missing)
    return module


def raise_bias(sd, head, raised):
    """a copy of sd whose head ("seq_lin" / "ctc_lin") bias is raised by {index: amount}"""
    bias = sd[head + ".w.bias"].clone()
    for i, amount in raised.items():
        bias[i] += amount
    return dict(sd, **{head + ".w.bias": bias})


def transformer_kwargs(cfg):
    """the TransformerASR keywords of a recipe config: sizes, attention, encoder module and the three activations"""
    from speechbrain_b200.nnet.activations import Swish
    act = {"gelu": torch.nn.GELU, "relu": torch.nn.ReLU, "swish": Swish}
    return dict(input_size=cfg["input_size"], tgt_vocab=cfg["vocab"], d_model=cfg["d_model"], nhead=cfg["nhead"],
                num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=cfg["num_decoder_layers"],
                d_ffn=cfg["d_ffn"], kernel_size=cfg.get("kernel_size", 31), attention_type=cfg["attention_type"],
                encoder_module=cfg.get("encoder_module", "conformer"), activation=act[cfg["decoder_activation"]],
                conformer_activation=act[cfg.get("conformer_activation", "swish")],
                branchformer_activation=act[cfg.get("branchformer_activation", "gelu")],
                csgu_linear_units=cfg.get("csgu_linear_units", 3072), max_length=cfg.get("max_length", 2500),
                normalize_before=True, causal=False)


class Mirror:
    """speechbrain_b200's modules of a recipe config holding the flat state sd: fb, norm, cnn, tr, ctc_lin and, when the
    config has decoder layers, seq_lin"""

    def __init__(self, cfg, sd, **transformer_kw):
        from speechbrain_b200.lobes.features import Fbank
        from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
        from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
        from speechbrain_b200.processing.features import InputNormalization
        self.cfg, self.sd = cfg, sd
        self.fb = Fbank(sample_rate=cfg["sample_rate"], n_fft=cfg["n_fft"], n_mels=cfg["n_mels"],
                        win_length=cfg["win"] * 1000 // cfg["sample_rate"])
        self.norm = InputNormalization(norm_type="global")
        self.norm.glob_mean, self.norm.glob_std, self.norm.count = sd["normalize.glob_mean"], sd["normalize.glob_std"], 1
        self.norm.eval()
        # the seeded state's CNN keys follow the config's cnn_blocks (utils/shapes.asr_model_shapes)
        if cfg.get("cnn_blocks", 2) == 3:
            cnn = ConvolutionFrontEnd(input_shape=(8, 10, cfg["n_mels"]), num_blocks=3, num_layers_per_block=1,
                                      out_channels=(cfg["cnn_channels"][0],) * 3, kernel_sizes=(5, 5, 1), strides=(2, 2, 1),
                                      residuals=(False, False, True))
        else:
            cnn = ConvolutionFrontEnd(input_shape=(8, 10, cfg["n_mels"]), num_blocks=2, num_layers_per_block=1,
                                      out_channels=cfg["cnn_channels"], kernel_sizes=(3, 3), strides=(2, 2),
                                      residuals=(False, False))
        self.cnn = load(cnn, sd, "CNN.")
        self.tr = load(TransformerASR(**dict(transformer_kwargs(cfg), **transformer_kw)), sd, "Transformer.")
        self.ctc_lin = self.head("ctc_lin")
        if cfg["num_decoder_layers"] > 0:
            self.seq_lin = self.head("seq_lin")

    def head(self, name, raised=None):
        """a new Linear holding sd's head name ("seq_lin" / "ctc_lin"), its bias raised by {index: amount}"""
        from speechbrain_b200.nnet.linear import Linear
        sd = raise_bias(self.sd, name, raised) if raised else self.sd
        return load(Linear(input_size=self.cfg["d_model"], n_neurons=self.cfg["vocab"]), sd, name + ".")

    def front_end(self, ctc_lin=None):
        """LengthsCapableSequential(Fbank, CMVN, CNN), the encoder of the recipes' EncoderDecoderASR layout; with a CTC
        head, EncoderASR's: EncoderWrapper(tr), ctc_lin and a log-softmax follow"""
        from speechbrain_b200.lobes.models.transformer.TransformerASR import EncoderWrapper
        from speechbrain_b200.nnet.activations import Softmax
        from speechbrain_b200.nnet.containers import LengthsCapableSequential
        if ctc_lin is None:
            return LengthsCapableSequential(compute_features=self.fb, normalize=self.norm, cnn=self.cnn)
        return LengthsCapableSequential(compute_features=self.fb, normalize=self.norm, cnn=self.cnn,
                                        transformer_encoder=EncoderWrapper(self.tr), ctc_lin=ctc_lin,
                                        log_softmax=Softmax(apply_log=True))

    def searcher(self, kwargs, max_decode_ratio, eos_bias=0.0, scorers=None, topk=None, blank=0, lm=None,
                 lm_temperature=LM_TEMPERATURE, coverage_threshold=0.5, scorer_beam_scale=2):
        """S2STransformerBeamSearcher over tr and a seq_lin with its EOS bias raised by eos_bias, built with kwargs and,
        when topk, return_topk=True.  scorers: an ordered {name: weight} of full scorers, built in that order, as
        oracle.goldens.run_beam takes them: "transformerlm" (lm, default parity.lm_scorer), "ctc" (ctc_lin with blank),
        "length" and "coverage" (coverage_threshold)."""
        from speechbrain_b200.decoders.scorer import (CoverageScorer, CTCScorer, LengthScorer, ScorerBuilder,
                                                      TransformerLMScorer)
        from speechbrain_b200.decoders.seq2seq import S2STransformerBeamSearcher
        full, vocab = [], self.cfg["vocab"]
        for name in scorers or {}:
            if name == "transformerlm":
                full.append(TransformerLMScorer(language_model=lm if lm is not None else lm_scorer(vocab),
                                                temperature=lm_temperature))
            elif name == "ctc":
                full.append(CTCScorer(eos_index=EOS, blank_index=blank, ctc_fc=self.ctc_lin))
            elif name == "length":
                full.append(LengthScorer(vocab))
            else:
                full.append(CoverageScorer(vocab, threshold=coverage_threshold))
        scorer = ScorerBuilder(full_scorers=full, weights=dict(scorers), scorer_beam_scale=scorer_beam_scale) if scorers else None
        return S2STransformerBeamSearcher(modules=[self.tr, self.head("seq_lin", {EOS: eos_bias})], bos_index=BOS,
                                          eos_index=EOS, max_decode_ratio=max_decode_ratio, scorer=scorer,
                                          **(dict(return_topk=True, topk=topk) if topk else {}), **kwargs)


def build_mirror(cfg, sd, **transformer_kw):
    """Mirror of cfg holding sd; transformer_kw override the TransformerASR keywords read from cfg"""
    return Mirror(cfg, sd, **transformer_kw)
