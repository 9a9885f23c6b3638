"""Scorer interfaces of the beam search -- mirrors of speechbrain.decoders.scorer for what is built on the H100 path:
``TransformerLMScorer`` (scorer.py:455-560) and ``CTCScorer`` (scorer.py:81-249, CTCPrefixScore decoders/ctc.py:46-295)
as *full* scorers of a ``ScorerBuilder`` (scorer.py:1075-1341), i.e. the recipe's ``scorer_test_search`` /
``scorer_valid_search`` (conformer_large.yaml:209-228), plus ``CoverageScorer`` (:788-955) and ``LengthScorer`` (:956-1072).
KenLM / RNNLM scorers and partial scorers raise.  The scoring itself runs inside the engine's beam search (csrc/engine.cu run_beam, csrc/ctc_scorer.cu).

``TransformerLMRescorer`` (scorer.py:1642-1882) + ``RescorerBuilder`` (scorer.py:2068-2189): n-best rescoring of text
hypotheses; tokenisation and the re-ranking stay on the host like in the reference, the LM forward runs teacher-forced on
the engine's KV-cached LM step (csrc/engine.cu run_lm_rescore)."""
import torch


class TransformerLMScorer:
    def __init__(self, language_model, temperature=1.0):
        self.lm = language_model
        self.temperature = temperature


class CTCScorer:
    def __init__(self, ctc_fc, blank_index, eos_index, ctc_window_size=0):
        if ctc_window_size != 0:
            raise NotImplementedError("speechbrain_b200.CTCScorer: ctc_window_size != 0 is not built")
        self.ctc_fc = ctc_fc
        self.blank_index = blank_index
        self.eos_index = eos_index
        self.ctc_window_size = ctc_window_size


class LengthScorer:
    """Length reward (scorer.py:956-1072): +weight on every token at every step; not compatible with length normalisation."""

    def __init__(self, vocab_size):
        self.vocab_size = vocab_size


class CoverageScorer:
    """Coverage penalty (scorer.py:788-955): cumulative last-layer cross-attention above ``threshold`` per frame is penalised."""

    def __init__(self, vocab_size, threshold=0.5):
        self.vocab_size = vocab_size
        self.threshold = threshold


_NAMES = {TransformerLMScorer: "transformerlm", CTCScorer: "ctc", LengthScorer: "length", CoverageScorer: "coverage"}
_ALL = ("ctc", "rnnlm", "transformerlm", "kenlm", "coverage", "length")


class ScorerBuilder:
    def __init__(self, weights=dict(), full_scorers=list(), partial_scorers=list(), scorer_beam_scale=2):
        assert len(weights) == len(full_scorers) + len(partial_scorers), "Weights and scorers are not matched."
        if partial_scorers:
            raise NotImplementedError("speechbrain_b200.ScorerBuilder: partial scorers are not built")
        names = []
        for impl in full_scorers:
            if type(impl) not in _NAMES:
                raise NotImplementedError(f"speechbrain_b200.ScorerBuilder: {type(impl).__name__} is not built "
                                          "(TransformerLMScorer, CTCScorer, CoverageScorer and LengthScorer are)")
            names.append(_NAMES[type(impl)])
        if len(set(names)) != len(names):
            raise ValueError("ScorerBuilder: duplicate scorers")
        unknown = set(weights) - set(_ALL)
        if unknown:
            raise ValueError(f"Weights for unavailable scorers: {sorted(unknown)}")
        if set(weights) != set(names):
            raise ValueError(f"ScorerBuilder: weights {sorted(weights)} do not match scorers {sorted(names)}")
        if names == ["ctc", "transformerlm"]:
            pass  # order only changes the float summation order of the added scores
        self.weights = {**dict.fromkeys(_ALL, 0.0), **{k: float(v) for k, v in weights.items()}}
        self.full_scorers = dict(zip(names, full_scorers))
        self.partial_scorers = {}
        self.scorer_beam_scale = scorer_beam_scale


class TransformerLMRescorer:
    def __init__(self, language_model, tokenizer, device="cuda", temperature=1.0, bos_index=0, eos_index=0, pad_index=0):
        if pad_index != 0:
            raise NotImplementedError("speechbrain_b200.TransformerLMRescorer: pad_index must be 0 (TransformerLM pads with 0)")
        self.lm = language_model
        self.tokenizer = tokenizer
        self.device = device
        self.temperature = temperature
        self.bos_index, self.eos_index, self.pad_index = bos_index, eos_index, pad_index
        self._slot = None

    def normalize_text(self, text):
        """scorer.py:1754-1771: the LM was trained on upper-case LibriSpeech text."""
        return text.upper()

    def to_device(self, device=None):
        if device is not None:
            self.device = device

    def preprocess_func(self, topk_hyps):
        """scorer.py:1793-1833: normalise, tokenise with bos/eos, pad.  Returns (padded int64 [n, L] on CPU, lengths)."""
        enc = [torch.tensor([self.bos_index] + list(self.tokenizer.encode_as_ids(self.normalize_text(seq))) + [self.eos_index])
               for batch in topk_hyps for seq in batch]
        lengths = [e.shape[0] for e in enc]
        padded = torch.nn.utils.rnn.pad_sequence(enc, batch_first=True, padding_value=self.pad_index)
        return padded, lengths

    def _engine_cfg(self):
        return dict(n_fft=400, hop=160, n_mels=80, cnn_channels=(64, 32), input_size=640, d_model=512, nhead=8,
                    num_encoder_layers=0, num_decoder_layers=0, d_ffn=2048, vocab=self.lm.vocab, attention_type="RoPEMHA")

    def _get_engine(self):
        if self._slot is None:
            from ..engine_cache import EngineSlot
            self._slot = EngineSlot(self._engine_cfg)
        return self._slot.get(self.device, ("lm",), {"lm.": self.lm})

    @torch.no_grad()
    def rescore_hyps(self, topk_hyps):
        """Returns the [B * topk] LM log-probability of every hypothesis (CUDA tensor), scorer.py:1835-1882."""
        padded, lengths = self.preprocess_func(topk_hyps)
        eng = self._get_engine()
        return eng.lm_rescore(padded.to(eng.device), torch.tensor(lengths), self.temperature, self.pad_index)


class RescorerBuilder:
    def __init__(self, weights=dict(), rescorers=list()):
        assert len(weights) == len(rescorers), "Weights and rescorers are not matched."
        names = []
        for impl in rescorers:
            if not isinstance(impl, TransformerLMRescorer):
                raise NotImplementedError(f"speechbrain_b200.RescorerBuilder: {type(impl).__name__} is not built "
                                          "(TransformerLMRescorer is)")
            names.append("transformerlm")
        if set(weights) - {"rnnlm", "transformerlm", "huggingfacelm"}:
            raise ValueError("The keys of weights should be named in ['rnnlm', 'transformerlm', 'huggingfacelm']")
        self.weights = {**dict.fromkeys(("rnnlm", "transformerlm", "huggingfacelm"), 0.0), **weights}
        self.rescorers = dict(zip(names, rescorers))

    def rescore(self, topk_candidates, topk_scores):
        """scorer.py:2113-2162: add weight * LM score to every candidate's score and sort each utterance's candidates."""
        new_scores = [list(row) for row in topk_scores]
        for k, impl in self.rescorers.items():
            scores = impl.rescore_hyps(topk_candidates).tolist()
            it = iter(scores)
            for i in range(len(new_scores)):
                for j in range(len(new_scores[i])):
                    new_scores[i][j] += self.weights[k] * next(it)
        output_candidates, output_scores = [], []
        for cands, scs in zip(topk_candidates, new_scores):
            order = sorted(zip(cands, scs), key=lambda x: x[1], reverse=True)
            output_candidates.append([c for c, _ in order])
            output_scores.append([s_ for _, s_ in order])
        return output_candidates, output_scores

    def move_rescorers_to_device(self, device=None):
        for impl in self.rescorers.values():
            impl.to_device(device)
