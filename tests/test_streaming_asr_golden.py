"""The reference StreamingASR run of tests/golden/streaming_asr.pt (tools/make_streaming_asr_golden.py) without a GPU: the
CPU oracle (tests/streaming_asr_oracle.py) gives the reference's tokens and strings, the wrapper's filter properties and
padding are the reference's, and the detokeniser mirror turns the stored token streams into the reference's strings,
leading-space cases included."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import streaming_asr_oracle as SO  # noqa: E402
import streaming_asr_util as SU  # noqa: E402


def _fixture():
    fx = torch.load(os.path.join(SO.GOLDEN, "streaming_asr.pt"))
    assert fx["spm_checksum"] == sum(SO.sp_model().serialized_model_proto())
    return fx


def test_fixture_covers_the_cases():
    fx = _fixture()
    assert set(fx["cases"]) == set(SO.CASES)
    for name, (att, chunk, left) in SO.CASES.items():
        g = fx["cases"][name]
        assert (g["att"], g["chunk"], g["left"]) == (att, chunk, left)
        assert g["feat_norms"][-1].shape[1] < chunk and all(f.shape[1] == chunk for f in g["feat_norms"][:-1])
    assert sum(len(t) for g in fx["cases"].values() for c in g["tokens"] for t in c) > 0


@pytest.mark.parametrize("name", list(SO.CASES))
def test_filter_properties_and_padding_equal_the_reference(name):
    from speechbrain_b200.lobes.features import StreamingFeatureWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.utils.filter_analysis import stack_filter_properties
    g = _fixture()["cases"][name]
    cfg, sd, w_enc, W, wav = SU.model_inputs(g["att"])
    fb, norm, cnn = SU.modules(cfg, sd, w_enc, W)[:3]
    fea = StreamingFeatureWrapper(LengthsCapableSequential(fb, norm, cnn), stack_filter_properties([fb, cnn]))
    assert (fea.properties.window_size, fea.properties.stride, fea.get_required_padding()) == (g["window_size"], g["stride"],
                                                                                               g["pad"])
    assert (SO.STRIDE - 1) * g["chunk"] == g["chunk_samples"] and SO.PAD == g["pad"]
    assert len(SO.chunks(wav, g["chunk"])) == len(g["tokens"])


@pytest.mark.parametrize("name", list(SO.CASES))
def test_oracle_equals_the_reference(name):
    g = _fixture()["cases"][name]
    cfg, sd, w_enc, W, wav = SU.model_inputs(g["att"])
    out = SO.run(wav, sd, cfg, w_enc, W, g["chunk"], g["left"], SO.sp_model())
    assert [c[2] for c in out] == g["tokens"]
    assert [c[3] for c in out] == g["words"]
    for c, fn, tn in zip(out, g["feat_norms"], g["tn_norms"]):
        assert rel(c[0].norm(dim=-1), fn) < 1e-4 and rel(c[1].norm(dim=-1), tn) < 1e-4


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_detokeniser_mirror_gives_the_reference_strings():
    from speechbrain_b200.tokenizers.SentencePiece import (SentencePieceDecoderStreamingContext,
                                                           spm_decode_preserve_leading_space)
    sp = SO.sp_model()
    spaced = 0
    for g in _fixture()["cases"].values():
        B = len(g["tokens"][0])
        ctxs = [SentencePieceDecoderStreamingContext() for _ in range(B)]
        for toks, words in zip(g["tokens"], g["words"]):
            got = [spm_decode_preserve_leading_space(sp, toks[b], ctxs[b]) for b in range(B)]
            assert got == words
            spaced += sum(w.startswith(" ") for w in words)
    assert spaced > 0  # the mid-stream leading space was exercised
