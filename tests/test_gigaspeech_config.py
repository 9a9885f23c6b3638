"""CPU tests of what is built for GigaSpeech's Conformer-Transducer: TransformerASR accepts head width 96 for the Conformer
with RelPosMHAXL and no decoder layers, streams it, and refuses every other use of 96; the seeded model that test_gpu_gigaspeech.py runs gives a search that says something
(0, 1 and >= 2 tokens on some frames)."""
import collections
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gigaspeech_oracle as GO  # noqa: E402


def _tr(**kw):
    from mirrors import transformer_kwargs
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    args = dict(transformer_kwargs(GO.config()), num_encoder_layers=2)
    args.update(kw)
    return TransformerASR(**args)


def test_gigaspeech_config_accepted_and_streams():
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _tr()
    assert (tr.d_model, tr.nhead, tr.num_decoder_layers, tr.attention_type) == (768, 8, 0, "RelPosMHAXL")
    for cs, lc in ((32, 4), (16, 8), (8, 2), (16, None)):
        tr.make_streaming_context(DynChunkTrainConfig(chunk_size=cs, left_context_size=lc))


@pytest.mark.parametrize("kw", [dict(attention_type="RoPEMHA"), dict(encoder_module="branchformer"),
                                dict(attention_type="hypermixing"),
                                dict(encoder_module="transformer", attention_type="regularMHA"),
                                dict(num_decoder_layers=1), dict(num_decoder_layers=6)])
def test_head_width_96_refused_elsewhere(kw):
    with pytest.raises(NotImplementedError):
        _tr(**kw)


def test_head_width_80_still_does_not_stream():
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _tr(d_model=640)
    with pytest.raises(NotImplementedError, match="head width 80"):
        tr.make_streaming_context(DynChunkTrainConfig(chunk_size=16, left_context_size=2))


def test_seeded_search_emits_0_1_and_more_tokens_per_frame():
    sd, w_enc, W = GO.weights()
    wav, lens = GO.waveforms()
    enc = GO.encode(sd, wav, lens)
    rows = GO.greedy(W, GO.tn_output(enc, w_enc)[:, :120])
    counts = collections.Counter()
    for r in rows:
        per_frame = collections.Counter(r["frames"])
        counts.update(min(per_frame.get(t, 0), 2) for t in range(120))
    assert counts[0] > 0 and counts[1] > 0 and counts[2] > 0, counts


def test_fp16_operand_error_estimate():
    """The oracle with every GEMM operand rounded to fp16 on the 4 x 10 s batch: about 6.0e-4 rel-L2 against the fp32
    oracle (DESIGN.md section 2a), so the encoder's 1e-3 bar holds at d_model 768."""
    from oracle import asr_oracle as O
    cfg = GO.config()
    sd, _, _ = GO.weights()
    wav, lens = GO.waveforms()
    with torch.no_grad():
        feats = O.full_pipeline_features(wav, lens, sd, dict(cfg, win_length=32))
        ref = O.encode(feats, lens, sd, cfg, "Transformer.")
        q = O.encode(feats, lens, sd, cfg, "Transformer.", q=lambda t: t.half().float())
    r = float((q - ref).norm() / ref.norm())
    print(f"fp16-operand oracle vs fp32 oracle: rel-L2 {r:.2e}")
    assert 4e-4 < r < 7.5e-4
