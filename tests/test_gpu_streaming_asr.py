"""-m gpu: StreamingASR on the LibriSpeech Conformer-Transducer model of tests/golden/transducer.pt's "e2e" entry (12-layer
Conformer, proj_enc, 640 / 512 / 1000 prediction network; RoPEMHA, and RelPosMHAXL at (16, 2)) against the reference
StreamingASR run stored in tests/golden/streaming_asr.pt (tools/make_streaming_asr_golden.py): the first 6 s of the e2e
batch's first three rows, the recommended zero chunks appended to the audio, so only the last chunk is short.

* Front end, every chunk (the first and the short last included): the wrapper output's per-frame norms within 2e-3 rel-L2
  of the reference's (the offline front-end parity tests allow 2e-3 abs on the fp16-operand CNN output), and bit-identical
  to the device's offline front end (Fbank -> InputNormalization -> ConvolutionFrontEnd mirrors) on the same window.
* Encoder, every whole chunk after the first: proj_enc output per-frame norms within 1e-3 rel-L2 of the reference's, and
  the output within 1e-3 rel-L2 of the fp32 CPU oracle (tests/streaming_asr_oracle.py).
* Decoding: each row's decisions equal the reference's up to its first near-tie (reference margin < 5e-3); from there the
  oracle walked along the device's decisions accepts every one (check_rows).  A chunk's strings equal the reference's
  while the row's tokens so far are equal, and a row with no near-tie gives the reference's whole text.
* Reruns, reset and a stream inside a batch of 4 are bit-identical; from_hparams on a recipe-layout directory transcribes
  like direct construction; bad chunks are refused before any device work."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import streaming_asr_oracle as SO  # noqa: E402
import streaming_asr_util as SU  # noqa: E402
import test_gpu_transducer as GT  # noqa: E402
import transducer_oracle as TO  # noqa: E402
from parity import normalizer_ckpt, write_pretrained_dir  # noqa: E402

pytestmark = pytest.mark.gpu
MARGIN = 5e-3

_ASR = {}


def _asr(att="RoPEMHA"):
    """(StreamingASR, cfg, sd, w_enc, W, wav), built once per attention type."""
    if att not in _ASR:
        _ASR[att] = SU.build(att)
    return _ASR[att]


def _fixture():
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "streaming_asr.pt"))
    assert fx["spm_checksum"] == sum(SO.sp_model().serialized_model_proto())
    return fx


def _chunks(asr, wav, cfg):
    """The audio with the recommended zero chunks appended, split into chunks of get_chunk_size_frames samples."""
    n = asr.get_chunk_size_frames(cfg)
    k = asr.hparams.fea_streaming_extractor.get_recommended_final_chunk_count(n)
    full = torch.cat([wav, torch.zeros(wav.shape[0], k * n)], dim=1)
    return [full[:, t:t + n].contiguous() for t in range(0, full.shape[1], n)]


def _stream(asr, wav, cfg, ctx=None):
    """Per chunk: (wrapper output, proj_enc output, tokens per row, text per row); and the context."""
    ctx = ctx or asr.make_streaming_context(cfg)
    out = []
    for ch in _chunks(asr, wav, cfg):
        ch = ch.cuda()
        feats = []
        fea = asr.hparams.fea_streaming_extractor
        orig = fea.forward

        def rec(*a, **k):
            y = orig(*a, **k)
            feats.append(y.clone())
            return y
        fea.forward = rec
        try:
            x = asr.encode_chunk(ctx, ch)
        finally:
            del fea.forward
        words, toks = asr.decode_chunk(ctx, x)
        out.append((feats[0].cpu(), x.cpu(), toks, words))
    return out, ctx


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("name", list(SO.CASES))
def test_against_the_reference(name):
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    g = _fixture()["cases"][name]
    asr, mcfg, sd, w_enc, W, wav = _asr(g["att"])
    fea = asr.hparams.fea_streaming_extractor
    chunk, left = g["chunk"], g["left"]
    assert (fea.get_required_padding(), fea.properties.window_size, fea.properties.stride) == (g["pad"], g["window_size"],
                                                                                                 g["stride"])
    cfg = DynChunkTrainConfig(chunk, left)
    assert asr.get_chunk_size_frames(cfg) == g["chunk_samples"]
    res, _ = _stream(asr, wav, cfg)
    assert len(res) == len(g["tokens"])
    trim = fea.get_output_count_per_pad_frame()
    worst_fe = 0.0
    for k, win in enumerate(SO.windows(wav, chunk)):
        got = res[k][0]
        off = fea.cnn(fea.normalize(fea.fbank(win.cuda())))
        off = off.reshape(off.shape[0], off.shape[1], -1)[:, trim:off.shape[1] - trim].cpu()
        assert torch.equal(got, off), f"chunk {k}: differs from the offline front end, max {float((got - off).abs().max())}"
        worst_fe = max(worst_fe, rel(got.norm(dim=-1), g["feat_norms"][k]))
    n_last = res[-1][0].shape[1]
    assert n_last < chunk and all(r[0].shape[1] == chunk for r in res[:-1])
    # whole chunks after the first (at (24, 8) the 6 s stream ends before the cache holds 8 chunks)
    whole = range(1, len(res) - 1)
    worst_tn = max(rel(res[k][1].norm(dim=-1), g["tn_norms"][k]) for k in whole)
    o = SO.run(wav, sd, mcfg, w_enc, W, chunk, left, SO.sp_model())
    worst_or = max(rel(res[k][1], o[k][1]) for k in whole)
    print(f"[stream asr {name}] {len(res)} chunks, last {n_last} frames; front end norms vs reference {worst_fe:.2e}; "
          f"proj_enc norms vs reference {worst_tn:.2e}, vs oracle {worst_or:.2e}")
    assert worst_fe < 2e-3 and worst_tn < 1e-3 and worst_or < 1e-3
    # decisions: the chunked tokens equal one greedy call over the concatenated frames, whose frames give the decisions
    B = wav.shape[0]
    tn = torch.cat([r[1] for r in res], dim=1)
    T = tn.shape[1]
    toks = [sum((r[2][b] for r in res), []) for b in range(B)]
    r = GT.run_device(asr.hparams.decoding_function.args[0], tn.cuda(), SO.MAX_SYMBOLS)
    assert toks == [r["tokens"][b, :int(r["n_tokens"][b])].tolist() for b in range(B)]
    offsets = [sum(x[1].shape[1] for x in res[:k]) for k in range(len(res))]
    ref_words = g["words"]
    for b in range(B):
        ref = [(int(t) + offsets[k], int(tok)) for k in range(len(res)) for t, tok in g["decisions"][k][b].tolist()]
        margins = [m for k in range(len(res)) for m in g["margins"][k][b].tolist()]
        cut = next((i for i, mg in enumerate(margins) if mg < MARGIN), len(ref))
        got = GT.device_decisions(r, b, T, SO.MAX_SYMBOLS)
        assert got[:cut] == ref[:cut], f"row {b}: differs from the reference before its first near-tie (decision {cut})"
        for k in range(len(res)):  # strings equal while the tokens so far are equal
            if all(res[j][2][b] == g["tokens"][j][b] for j in range(k + 1)):
                assert res[k][3][b] == ref_words[k][b], (b, k)
        if cut == len(ref):
            assert "".join(x[3][b] for x in res) == "".join(w[b] for w in ref_words)
    GT.check_rows(TO.Oracle(W), tn, 0, SO.MAX_SYMBOLS, r, range(B))


def test_reruns_reset_and_batch_are_bit_identical():
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    asr = _asr()[0]
    cfg = DynChunkTrainConfig(16, 2)
    wav4 = torch.cat([_asr()[5], _asr()[5][:1].flip(1)], dim=0)
    a, ctx = _stream(asr, wav4, cfg)
    b, _ = _stream(asr, wav4, cfg)
    ctx.encoder_context.reset()
    ctx.decoder_context.hidden = None
    ctx.tokenizer_context = None
    c, _ = _stream(asr, wav4, cfg, ctx)
    assert sum(len(t) for x in a for t in x[2]) > 0  # the seeded model emits tokens at (16, 2) on this audio
    for x, y, z in zip(a, b, c):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) and x[2] == y[2] == z[2] and torch.equal(x[1], z[1])
    for i in (0, 3):
        alone, _ = _stream(asr, wav4[i:i + 1], cfg)
        for x, y in zip(a, alone):
            assert torch.equal(x[0][i:i + 1], y[0]) and torch.equal(x[1][i:i + 1], y[1]) and x[2][i] == y[2][0]


def test_rejections_before_device_work():
    from speechbrain_b200._lib import lib
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    asr = _asr()[0]
    cfg = DynChunkTrainConfig(8, 2)
    n = asr.get_chunk_size_frames(cfg)
    ctx = asr.make_streaming_context(cfg)
    wav = _asr()[5][:2]
    asr.transcribe_chunk(ctx, wav[:, :n].cuda())
    torch.cuda.synchronize()
    n0 = lib().sbk_launch_count()
    with pytest.raises(ValueError, match="expected"):
        asr.transcribe_chunk(ctx, wav[:, :n + 1].cuda())
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        asr.hparams.fea_streaming_extractor(wav[:, :n], context=ctx.fea_extractor_context)
    assert lib().sbk_launch_count() == n0
    asr.transcribe_chunk(ctx, wav[:, n:n + 1000].cuda())  # a short chunk ends the stream
    n0 = lib().sbk_launch_count()
    with pytest.raises(RuntimeError, match="last chunk"):
        asr.transcribe_chunk(ctx, wav[:, :n].cuda())
    assert lib().sbk_launch_count() == n0


HPARAMS = GT.HPARAMS.replace("tokenizer: null\n", "").replace("transducer_beam_search: True\n", "") + """
Greedysearcher: !ref <decoder>
tokenizer: !apply:streaming_asr_oracle.sp_model
make_tokenizer_streaming_context: !name:speechbrain.tokenizers.SentencePiece.SentencePieceDecoderStreamingContext
tokenizer_decode_streaming: !name:speechbrain.tokenizers.SentencePiece.spm_decode_preserve_leading_space
make_decoder_streaming_context: !name:speechbrain.decoders.transducer.TransducerGreedySearcherStreamingContext
decoding_function: !name:speechbrain.decoders.transducer.TransducerBeamSearcher.transducer_greedy_decode_streaming
    - !ref <Greedysearcher>
fea_streaming_extractor: !new:speechbrain.lobes.features.StreamingFeatureWrapper
    module: !new:speechbrain.nnet.containers.LengthsCapableSequential
        - !ref <compute_features>
        - !ref <normalizer>
        - !ref <CNN>
    properties: !apply:speechbrain.utils.filter_analysis.stack_filter_properties
        - [!ref <compute_features>, !ref <CNN>]
streaming_modules:
    enc: !ref <enc>
    proj_enc: !ref <proj_enc>
""".replace("modules:\n    encoder: !ref <encoder>\n    decoder: !ref <decoder>\n", "")


def test_from_hparams_local_directory_matches_direct_construction(tmp_path):
    from speechbrain_b200.inference.ASR import StreamingASR
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    asr, mcfg, sd, w_enc, W, _ = _asr()
    _, parts = GT._transducer_modules(mcfg, sd, w_enc, W)
    order = ["CNN", "Transformer", "proj_enc", "emb", "dec", "proj_dec", "transducer_lin"]
    ck = {f"{i}.{k}": v for i, n in enumerate(order) for k, v in parts[n].state_dict().items()}
    text = HPARAMS.replace("streaming_modules:", "modules:")
    tmp = write_pretrained_dir(tmp_path, text, dict(asr=ck, normalizer=normalizer_ckpt(sd)))
    loaded = StreamingASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    cfg = DynChunkTrainConfig(16, 2)
    wav = _asr()[5][:2]
    a, _ = _stream(loaded, wav, cfg)
    b, _ = _stream(asr, wav, cfg)
    assert [x[2] for x in a] == [x[2] for x in b] and [x[3] for x in a] == [x[3] for x in b]
    assert all(torch.equal(x[1], y[1]) for x, y in zip(a, b))
