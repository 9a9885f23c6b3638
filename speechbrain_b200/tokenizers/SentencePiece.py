"""SentencePiece streaming detokeniser -- mirror of SentencePieceDecoderStreamingContext and
spm_decode_preserve_leading_space (speechbrain/tokenizers/SentencePiece.py:519-577), which ``StreamingASR`` uses to turn
each chunk's tokens into text.  Host-side string work on a ``sentencepiece.SentencePieceProcessor``."""
from dataclasses import dataclass
from typing import List


@dataclass
class SentencePieceDecoderStreamingContext:
    """Mutable streaming context for a single SentencePiece streaming session."""

    emitted_symbol_count: int = 0
    """The number of symbols that have been emitted for this transcription."""


def spm_decode_preserve_leading_space(tokenizer, hyps: List[int], context: SentencePieceDecoderStreamingContext) -> str:
    """Decodes one hypothesis' tokens, keeping the leading space that SentencePiece strips from a sentence start when the
    stream has already emitted symbols and the first piece starts with the word-boundary mark U+2581."""
    proto = tokenizer.decode([hyps], out_type="immutable_proto")[0]
    text = proto.text
    if len(proto.pieces) >= 1:
        should_preserve_space = context.emitted_symbol_count > 0
        if should_preserve_space and proto.pieces[0].piece.startswith("▁"):
            text = " " + text
        context.emitted_symbol_count += len(proto.pieces)
    return text
