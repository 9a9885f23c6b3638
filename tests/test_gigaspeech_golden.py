"""The reference run of tests/golden/gigaspeech.pt (tools/make_gigaspeech_golden.py) without a GPU: the CPU oracles
(gigaspeech_oracle.py, transducer_oracle.py, transducer_beam_oracle.py, streaming_asr_oracle.run) equal the fixture; the
mirror's state_dict keys and shapes equal the reference modules' in both directions; the recipe-layout inference YAMLs
(the offline EncoderDecoderASR transducer block and the commented StreamingASR block) load through from_hparams."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gigaspeech_oracle as GO  # noqa: E402
import streaming_asr_oracle as SO  # noqa: E402
import transducer_beam_oracle as BO  # noqa: E402
from parity import normalizer_ckpt, write_pretrained_dir  # noqa: E402

CASES = ["32_4", "16_8", "8_2"]


@pytest.fixture(scope="module")
def fx():
    g = torch.load(os.path.join(GO.GOLDEN, "gigaspeech.pt"))
    assert g["spm_checksum"] == sum(GO.sp_model().serialized_model_proto())
    return g


@pytest.fixture(scope="module")
def offline():
    sd, w_enc, W = GO.weights()
    wav, lens = GO.waveforms()
    enc = GO.encode(sd, wav, lens)
    return dict(sd=sd, w_enc=w_enc, W=W, wav=wav, lens=lens, enc=enc, tn=GO.tn_output(enc, w_enc))


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def test_oracle_equals_the_reference_offline(fx, offline):
    g = fx["offline"]
    assert g["wav_checksum"] == pytest.approx(float(offline["wav"].double().abs().sum()), rel=1e-9)
    assert rel(offline["enc"].norm(dim=-1), g["enc_norms"]) < 1e-5 and rel(offline["tn"].norm(dim=-1), g["tn_norms"]) < 1e-5
    dc = GO.encode(offline["sd"], offline["wav"], offline["lens"], dynchunk=tuple(g["dynchunk"]))
    assert rel(dc.norm(dim=-1), g["dynchunk_enc_norms"]) < 1e-5
    rows = GO.greedy(offline["W"], offline["tn"])
    assert [r["tokens"] for r in rows] == g["tokens"]
    for b, r in enumerate(rows):
        assert [(d[0], d[1]) for d in r["decisions"]] == [tuple(x) for x in g["decisions"][b].tolist()]
    assert all(g["emission_hist"][k] > 0 for k in (0, 1, 2))
    best, _, nb, nbs, _ = BO.BeamOracle(offline["W"]).batch(offline["tn"], GO.BLANK, GO.BEAM, 1, GO.STATE_BEAM, GO.EXPAND_BEAM)
    assert nb == g["beam"]["tokens"]
    assert all(abs(a[0] - b[0]) <= 1e-5 for a, b in zip(nbs, g["beam"]["scores"]))


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_the_reference_streaming(fx, offline, name):
    g = fx["streaming"][name]
    assert (g["pad"], g["stride"], g["chunk_samples"]) == (SO.PAD, SO.STRIDE, SO.chunk_samples(g["chunk"]))
    wav = offline["wav"][:3, :SO.L_AUDIO].contiguous()
    out = SO.run(wav, offline["sd"], GO.config(), offline["w_enc"], offline["W"], g["chunk"], g["left"], GO.sp_model())
    assert [c[2] for c in out] == g["tokens"] and [c[3] for c in out] == g["words"]
    for c, fn, tn in zip(out, g["feat_norms"], g["tn_norms"]):
        assert rel(c[0].norm(dim=-1), fn) < 1e-4 and rel(c[1].norm(dim=-1), tn) < 1e-4
    assert sum(len(t) for c in g["tokens"] for t in c) > 0


def test_state_dict_equals_the_reference(fx, offline):
    """every reference module's keys and shapes against the mirror's, in both directions"""
    m = GO.modules(offline["sd"], offline["w_enc"], offline["W"])
    for name, ref in fx["keys"].items():
        got = {k: list(v.shape) for k, v in m[name].state_dict().items()}
        if name == "Transformer":  # the positional buffers: the reference keeps inv_freq only for RelPosMHAXL
            assert {k for k in ref if k.startswith("positional_encoding")} <= set(got)
        assert got == ref, name
    assert fx["keys"]["Transformer"]["encoder.layers.0.mha_layer.pos_bias_u"] == [96, 8]


def _ckpts(offline):
    m = GO.modules(offline["sd"], offline["w_enc"], offline["W"])
    return m, dict(asr=GO.asr_ckpt(m), normalizer=normalizer_ckpt(offline["sd"]))


def test_offline_inference_yaml_loads(tmp_path, offline):
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    m, ck = _ckpts(offline)
    asr = EncoderDecoderASR.from_hparams(source=write_pretrained_dir(tmp_path, GO.HPARAMS, ck), run_opts={"device": "cuda:0"})
    dec = asr.mods["decoder"]
    assert isinstance(dec, TransducerBeamSearcher) and asr.transducer_beam_search
    assert (dec.beam_size, dec.nbest, dec.state_beam, dec.expand_beam) == (10, 1, 2.3, 2.3)
    tr = asr.mods["encoder"].transformer_encoder.transformer
    assert (tr.d_model, tr.nhead, tr.num_decoder_layers) == (768, 8, 0)
    key = "encoder.layers.3.mha_layer.pos_bias_v"
    assert torch.equal(tr.state_dict()[key], m["Transformer"].state_dict()[key])
    assert torch.equal(dec.classifier_network[0].w.weight, offline["W"]["transducer_lin.w.weight"])


def test_streaming_inference_yaml_loads(tmp_path, offline):
    from speechbrain_b200.inference.ASR import StreamingASR
    _, ck = _ckpts(offline)
    asr = StreamingASR.from_hparams(source=write_pretrained_dir(tmp_path, GO.STREAMING_HPARAMS, ck),
                                    run_opts={"device": "cuda:0"})
    fea = asr.hparams.fea_streaming_extractor
    assert (fea.get_required_padding(), fea.properties.stride) == (SO.PAD, SO.STRIDE)
    assert asr.hparams.tokenizer.get_piece_size() == GO.V
    assert torch.equal(asr.mods["proj_enc"].w.weight, offline["w_enc"])
