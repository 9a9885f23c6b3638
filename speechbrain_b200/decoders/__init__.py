"""speechbrain.decoders namespace: the names the recipes' YAML files reach through the package (decoders/__init__.py)."""
from .scorer import (CoverageScorer, CTCScorer, LengthScorer, RescorerBuilder, ScorerBuilder, TransformerLMRescorer,  # noqa: F401
                     TransformerLMScorer)
from .seq2seq import S2STransformerBeamSearcher, S2STransformerGreedySearcher  # noqa: F401
from .ctc import (CTCBeamSearcher, CTCHypothesis, CTCPrefixBeamSearcher, ctc_greedy_decode,  # noqa: F401
                  filter_ctc_output)
