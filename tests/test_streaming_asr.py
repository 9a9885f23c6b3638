"""StreamingASR host logic without a GPU: the filter properties and padding of every front end this project builds (numbers
from the reference's speechbrain.utils.filter_analysis), the SentencePiece streaming detokeniser, the loader's dotted
names, and the refusals that come before any device work."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from streaming_asr_util import sp_model  # noqa: E402


def _cnn(kind):
    from speechbrain_b200.lobes.models.convolution import ConvolutionFrontEnd
    if kind == "conformer":
        return ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1, out_channels=(64, 32),
                                   kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
    if kind == "aishell":
        return ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1, out_channels=(256, 256),
                                   kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
    return ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=3, num_layers_per_block=1, out_channels=(64, 64, 64),
                               kernel_sizes=(5, 5, 1), strides=(2, 2, 1), residuals=(False, False, True))


# (Fbank win_length ms, front end) -> (CNN window, CNN stride, stacked window, stacked stride), from the reference
REFERENCE = {(25, "conformer"): (7, 4, 1361, 640), (32, "conformer"): (7, 4, 1473, 640), (25, "aishell"): (7, 4, 1361, 640),
             (25, "transformer"): (13, 4, 2321, 640), (32, "transformer"): (13, 4, 2433, 640)}


@pytest.mark.parametrize("win,kind", sorted(REFERENCE))
def test_filter_properties_and_padding(win, kind):
    from speechbrain_b200.lobes.features import Fbank, StreamingFeatureWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.processing.features import InputNormalization
    from speechbrain_b200.utils.filter_analysis import FilterProperties, stack_filter_properties
    fb = Fbank(n_fft=512 if win == 32 else 400, n_mels=80, win_length=win)
    cnn = _cnn(kind)
    cw, cs, w, s = REFERENCE[(win, kind)]
    assert fb.get_filter_properties() == FilterProperties(16 * win, 160)
    assert cnn.get_filter_properties() == FilterProperties(cw, cs)
    props = stack_filter_properties([fb, cnn])
    assert props == FilterProperties(w, s)
    wrap = StreamingFeatureWrapper(LengthsCapableSequential(fb, InputNormalization(norm_type="global"), cnn), props)
    assert wrap.get_required_padding() == 1280 and wrap.get_output_count_per_pad_frame() == 2
    assert wrap.get_recommended_final_chunk_count(639 * 24) == 1 and wrap.get_recommended_final_chunk_count(1000) == 2
    assert wrap.get_filter_properties() is props


def test_filter_analysis_rules():
    from speechbrain_b200.utils.filter_analysis import FilterProperties, stack_filter_properties, upalign_value
    assert stack_filter_properties([]) == FilterProperties(1, 1)
    assert upalign_value(680, 640) == 1280 and upalign_value(1280, 640) == 1280 and upalign_value(0, 7) == 0
    causal = FilterProperties(3, 1, causal=True)
    assert causal.get_noncausal_equivalent() == FilterProperties(5, 1)
    assert stack_filter_properties([causal, FilterProperties(3, 2)]) == FilterProperties(7, 2)
    with pytest.raises(ValueError):
        stack_filter_properties([FilterProperties(3, 1), FilterProperties(4, 1)], allow_approximate=False)
    assert FilterProperties(5, 1, dilation=2).get_convolution_padding() == 4


def test_wrapper_refusals():
    from speechbrain_b200.lobes.features import Fbank, StreamingFeatureWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.processing.features import InputNormalization
    from speechbrain_b200.utils.filter_analysis import FilterProperties
    fb, cnn = Fbank(n_mels=80), _cnn("conformer")
    mod = LengthsCapableSequential(fb, InputNormalization(norm_type="global"), cnn)
    with pytest.raises(ValueError, match="Causal"):
        StreamingFeatureWrapper(mod, FilterProperties(3, 1, causal=True))
    with pytest.raises(ValueError, match="Dilation"):
        StreamingFeatureWrapper(mod, FilterProperties(3, 1, dilation=2))
    for other in (LengthsCapableSequential(fb, cnn), LengthsCapableSequential(fb, InputNormalization(norm_type="sentence"), cnn),
                  fb):
        with pytest.raises(NotImplementedError):
            StreamingFeatureWrapper(other, FilterProperties(1361, 640))
    with pytest.raises(ValueError, match="stride"):  # properties that are not the module's would trim differently
        StreamingFeatureWrapper(mod, FilterProperties(1361, 1280))
    wrap = StreamingFeatureWrapper(mod, FilterProperties(1361, 640))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        wrap(torch.zeros(1, 100), context=wrap.make_streaming_context())


def test_detokeniser_streams_like_a_whole_decode():
    """Each chunk's text, concatenated, is the decode of the whole token stream: the leading space SentencePiece drops at a
    sentence start is put back mid-stream (U+2581 first piece), and not at the stream's start or inside a word."""
    from speechbrain_b200.tokenizers.SentencePiece import (SentencePieceDecoderStreamingContext,
                                                           spm_decode_preserve_leading_space)
    sp = sp_model()
    assert sp.vocab_size() == 1000
    gen = torch.Generator().manual_seed(5)
    starts = [i for i in range(1, 1000) if sp.id_to_piece(i).startswith("▁")]
    assert 0 < len(starts) < 999
    checked_space = checked_word = 0
    for _ in range(50):
        toks = torch.randint(1, 1000, (40,), generator=gen).tolist()
        cuts = sorted(torch.randint(0, 41, (6,), generator=gen).tolist())
        ctx = SentencePieceDecoderStreamingContext()
        parts = [spm_decode_preserve_leading_space(sp, toks[a:b], ctx) for a, b in zip([0] + cuts, cuts + [40])]
        assert "".join(parts) == sp.decode(toks)
        assert ctx.emitted_symbol_count == len(sp.decode([toks], out_type="immutable_proto")[0].pieces)
        for (a, b), text in zip(zip([0] + cuts, cuts + [40]), parts):
            if a > 0 and b > a:
                checked_space += text.startswith(" ")
                checked_word += not text.startswith(" ")
    assert checked_space > 0 and checked_word > 0
    ctx = SentencePieceDecoderStreamingContext()
    assert spm_decode_preserve_leading_space(sp, [], ctx) == "" and ctx.emitted_symbol_count == 0
    first = spm_decode_preserve_leading_space(sp, [starts[0]], ctx)
    assert not first.startswith(" ") and spm_decode_preserve_leading_space(sp, [starts[1]], ctx).startswith(" ")


def test_loader_resolves_the_streaming_names():
    import functools

    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.lobes.features import StreamingFeatureWrapper
    from speechbrain_b200.tokenizers.SentencePiece import (SentencePieceDecoderStreamingContext,
                                                           spm_decode_preserve_leading_space)
    from speechbrain_b200.utils.filter_analysis import stack_filter_properties
    from speechbrain_b200.utils.hparams import load_hyperpyyaml, resolve_name
    assert resolve_name("speechbrain.utils.filter_analysis.stack_filter_properties") is stack_filter_properties
    assert resolve_name("speechbrain.lobes.features.StreamingFeatureWrapper") is StreamingFeatureWrapper
    assert resolve_name("speechbrain.tokenizers.SentencePiece.spm_decode_preserve_leading_space") is \
        spm_decode_preserve_leading_space
    assert resolve_name("speechbrain.tokenizers.SentencePiece.SentencePieceDecoderStreamingContext") is \
        SentencePieceDecoderStreamingContext
    hp = load_hyperpyyaml("""
searcher: !new:builtins.object
decoding_function: !name:speechbrain.decoders.transducer.TransducerBeamSearcher.transducer_greedy_decode_streaming
    - !ref <searcher>
fb: !new:speechbrain.lobes.features.Fbank
    n_mels: 80
props: !apply:speechbrain.utils.filter_analysis.stack_filter_properties
    - [!ref <fb>]
""")
    fn = hp["decoding_function"]
    assert isinstance(fn, functools.partial) and fn.func is TransducerBeamSearcher.transducer_greedy_decode_streaming
    assert fn.args == (hp["searcher"],)
    assert (hp["props"].window_size, hp["props"].stride) == (401, 160)


def test_file_transcription_is_refused():
    from speechbrain_b200.inference.ASR import StreamingASR
    asr = object.__new__(StreamingASR)
    for call in (lambda: asr.transcribe_file("x.wav", None), lambda: next(iter(asr.transcribe_file_streaming("x.wav", None)))):
        with pytest.raises(NotImplementedError, match="audio file"):
            call()
