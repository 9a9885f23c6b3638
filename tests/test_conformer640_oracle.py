"""CPU tests of the d_model 640 Conformer (Libriheavy / People's Speech conformer_large: 8 heads of 80, RelPosMHAXL; GELU
or Swish decoder FFN): what the TransformerASR mirror accepts and rejects at head width 80, its state_dict against the
reference's, the CPU oracle against the reference outputs in tests/golden/conformer640.pt (generator:
tools/make_conformer640_golden.py), and the fp16-operand error estimate the device encoder bar of test_gpu_conformer640.py
rests on."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import conformer640_oracle as CO  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "conformer640.pt")


def _tr(**kw):
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    args = dict(tgt_vocab=5120, input_size=640, d_model=640, nhead=8, num_encoder_layers=2, num_decoder_layers=1, d_ffn=2048,
                encoder_module="conformer", attention_type="RelPosMHAXL", normalize_before=True, causal=False)
    args.update(kw)
    return TransformerASR(**args)


def test_head_width_80_accepted_for_relpos_conformer_only():
    from speechbrain_b200.nnet.activations import Swish
    assert _tr(activation=Swish, conformer_activation=Swish).decoder_activation == "swish"
    assert _tr(activation=torch.nn.SiLU).decoder_activation == "swish"
    assert _tr(activation=torch.nn.GELU).decoder_activation == "gelu"
    for kw in (dict(attention_type="RoPEMHA"), dict(encoder_module="branchformer"),
               dict(encoder_module="transformer", attention_type="regularMHA"), dict(d_model=768, nhead=8)):
        with pytest.raises(NotImplementedError):
            _tr(**kw)
    with pytest.raises(NotImplementedError):
        _tr(activation=torch.nn.Tanh)


def test_streaming_rejected_at_head_width_80():
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _tr()
    with pytest.raises(NotImplementedError):
        tr.make_streaming_context(DynChunkTrainConfig(chunk_size=16, left_context_size=2))


@pytest.fixture(scope="module")
def fx():
    return torch.load(GOLDEN)


def _cfg(recipe):
    from speechbrain_b200.utils.seeded_init import CONFORMER_640, CONFORMER_640_PEOPLES
    return CONFORMER_640 if recipe == "libriheavy" else CONFORMER_640_PEOPLES


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _check_summary(name, x, summ):
    idx = summ["sample_idx"].long()
    e = max(_rel(x.double().norm(dim=-1), summ["row_norm"]), _rel(x[idx[:, 0], idx[:, 1]], summ["sample_rows"]))
    print(f"{name}: oracle vs reference rel-L2 {e:.2e}")
    assert e < 1e-5, name


@pytest.mark.parametrize("recipe", ["libriheavy", "peoples"])
def test_state_dict_matches_the_reference(fx, recipe):
    """the mirror's TransformerASR state_dict keys and shapes equal the reference's, in both directions"""
    from speechbrain_b200.nnet.activations import Swish
    cfg = _cfg(recipe)
    tr = _tr(tgt_vocab=cfg["vocab"], num_encoder_layers=14, num_decoder_layers=6, conformer_activation=Swish,
             activation=Swish if cfg["decoder_activation"] == "swish" else torch.nn.GELU)
    ours = [(k, tuple(v.shape)) for k, v in tr.state_dict().items()]
    ref = [(k, tuple(s)) for k, s in fx[recipe]["keys"]]
    assert sorted(ours) == sorted(ref)


@pytest.mark.parametrize("recipe", ["libriheavy", "peoples"])
def test_oracle_matches_reference(fx, recipe):
    """conformer640_oracle (oracle/asr_oracle.py, Swish decoder FFN for People's Speech) equals the reference on every
    fixture entry: encoder states, greedy hypotheses / tokens / chosen log-probs, teacher-forced decode(), the beam search's
    best hypotheses and scores, and the 1.3 s utterance"""
    cfg, g = _cfg(recipe), fx[recipe]
    sd = CO.state(cfg)
    wav, lens = CO.waveforms()
    assert torch.equal(lens, g["wav_lens"])
    enc = CO.encode(cfg, sd, wav, lens)
    _check_summary(f"{recipe} encoder", enc, g["enc"])
    hyps, lp, logits = CO.greedy(cfg, sd, enc, lens)
    tok = logits.argmax(-1)
    assert hyps == g["greedy_hyps"] and torch.equal(tok.int(), g["greedy_tokens"])
    assert (lp.gather(-1, tok.unsqueeze(-1)).squeeze(-1) - g["greedy_chosen_lp"]).abs().max() < 1e-4
    dec = CO.decode(cfg, sd, CO.teacher_tokens(cfg), enc, g["abs_len"])
    _check_summary(f"{recipe} decode()", dec, g["decode"])
    gb = g["beam"]
    ohyps, _, oscores, _ = CO.beam(cfg, sd, enc[gb["utts"]], lens[gb["utts"]], gb)
    print(f"{recipe} beam {gb['beam']}: oracle {oscores.view(-1).tolist()} reference {gb['scores'].tolist()}")
    assert [list(h) for h in ohyps] == [list(h) for h in gb["hyps"]]
    assert (oscores.view(-1) - gb["scores"]).abs().max() < 1e-4
    if "short" in g:
        w1, l1 = CO.waveforms(seed=13, L=20800, lens=[1.0])
        e1 = CO.encode(cfg, sd, w1, l1)
        assert _rel(e1, g["short"]["enc"]) < 1e-5 and CO.greedy(cfg, sd, e1, l1, ratio=1.0)[0] == g["short"]["greedy_hyps"]


def test_fp16_operand_error_estimate():
    """The oracle with every GEMM operand rounded to fp16 on the 4 x 10 s input of test_gpu_conformer640.py: about 5.4e-4
    rel-L2 against the fp32 oracle, so the Conformer's 1e-3 encoder bar holds at d_model 640."""
    from oracle import asr_oracle as O
    from speechbrain_b200.utils.seeded_init import CONFORMER_640, seeded_asr_state
    cfg = CONFORMER_640
    sd = seeded_asr_state(cfg, 0)
    g = torch.Generator().manual_seed(7)
    lens = torch.tensor([1.0, 0.9, 0.6, 0.3])
    wav = torch.randn(4, 160000, generator=g)
    for b, f in enumerate(lens.tolist()):
        wav[b, int(round(f * 160000)):] = 0
    with torch.no_grad():
        feats = O.full_pipeline_features(wav, lens, sd, dict(cfg, win_length=32))
        ref = O.encode(feats, lens, sd, cfg, "Transformer.")
        q = O.encode(feats, lens, sd, cfg, "Transformer.", q=lambda t: t.half().float())
    r = float((q - ref).norm() / ref.norm())
    print(f"fp16-operand oracle vs fp32 oracle at d_model 640: encoder rel-L2 {r:.2e}")
    assert r <= 7e-4
