"""-m gpu tests of the engine handle's lane state (csrc/engine.cu): a clone is a new lane on the source's weights with its
own streams, events, buffers and graphs, and growing a lane buffer drops the graphs that captured pointers into it.
Results are compared with the same handle's or the source's own, not with goldens (those are checked elsewhere)."""
import gc
import os
import sys

import pytest
import torch

from speechbrain_b200 import _lib
from speechbrain_b200.engine import AsrEngine
from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state, seeded_tensor
from speechbrain_b200.utils.shapes import transformer_lm_shapes

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401

pytestmark = pytest.mark.gpu
LM = dict(d_model=128, nhead=2, num_encoder_layers=2, d_ffn=256)
CFG = dict(CONFORMER_LARGE, num_encoder_layers=2, num_decoder_layers=2, lm=LM)
BEAM = dict(beam_size=4, max_steps=12, min_steps=0, bos=1, eos=2, lm_weight=0.6, ctc_weight=0.4, blank_index=0)


def _engine(dev):
    sd = seeded_asr_state(CFG, 0)  # decoder, seq_lin and ctc_lin
    for k, shp in transformer_lm_shapes(CFG["vocab"], LM["d_model"], LM["nhead"], LM["num_encoder_layers"], LM["d_ffn"]).items():
        sd["lm." + k] = seeded_tensor(1, "lm." + k, shp)
    return AsrEngine(CFG, sd, device=dev, parts=("fbank", "cnn", "encoder", "decoder", "lm"))


def _launches():
    return _lib.lib().sbk_launch_count()


def test_clone_after_use_owns_its_streams(dev):
    g = torch.Generator().manual_seed(0)
    wavs = [torch.randn(2, 32000, generator=g).to(dev) for _ in range(2)]
    lens = [torch.tensor([1.0, 0.7], device=dev), torch.tensor([0.8, 1.0], device=dev)]
    enc = torch.randn(2, 100, CFG["d_model"], generator=g).to(dev)
    enc_lens = torch.tensor([1.0, 0.85], device=dev)
    steps = 6

    def run(eng):
        """Group call (poll 0: the whole-group graph on the high-priority decode stream), then a beam search with LM and CTC
        scorers (their branch on the side stream).  Returns the outputs and the launches each call enqueued."""
        preds = [torch.empty(2, steps, dtype=torch.int32, device=dev) for _ in wavs]
        n0 = _launches()
        eng.transcribe_greedy_group_dev(wavs, lens, steps, 1, 2, preds)
        n1 = _launches()
        hist = eng.beam_from_enc(enc, enc_lens, **BEAM)
        return dict(preds=preds, hist=hist, launches=(n1 - n0, _launches() - n1))

    src = _engine(dev)
    # non-default settings a clone inherits: chunked encoder attention changes the encoder states, the separate decoder
    # LayerNorm kernels and the wgmma decode path from one row change the launches of every call
    src.set_poll_interval(0)
    src.set_dynchunk(8, 2)
    src.set_decoder_ln_fusion(False)
    src.set_decoder_tc_min_rows(1)
    ref = run(src)
    torch.cuda.synchronize()
    lanes = [src.clone(), src.clone()]
    del src
    gc.collect()
    streams = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]
    outs = [None, None]
    for i, (eng, s) in enumerate(zip(lanes, streams)):  # both group calls in flight at once, then the two searches
        with torch.cuda.stream(s):
            preds = [torch.empty(2, steps, dtype=torch.int32, device=dev) for _ in wavs]
            n0 = _launches()
            eng.transcribe_greedy_group_dev(wavs, lens, steps, 1, 2, preds)
            outs[i] = dict(preds=preds, launches=[_launches() - n0])
    for i, (eng, s) in enumerate(zip(lanes, streams)):
        with torch.cuda.stream(s):
            n0 = _launches()
            outs[i]["hist"] = eng.beam_from_enc(enc, enc_lens, **BEAM)
            outs[i]["launches"].append(_launches() - n0)
    torch.cuda.synchronize()
    for out in outs:
        assert tuple(out["launches"]) == ref["launches"]
        assert all(torch.equal(a, b) for a, b in zip(out["preds"], ref["preds"]))
        assert len(out["hist"][0]) == len(ref["hist"][0]) > 0
        assert all(torch.equal(a, b) for a, b in zip(out["hist"], ref["hist"]))


def test_buffer_growth_drops_captured_graphs(dev):
    eng = _engine(dev)
    g = torch.Generator().manual_seed(1)
    big = torch.randn(32, 251, CFG["d_model"], generator=g).to(dev)
    enc = torch.randn(2, 100, CFG["d_model"], generator=g).to(dev)
    enc_lens = torch.ones(2, device=dev)
    beam = dict(BEAM, lm_weight=0.0)
    # size the workspace for the large ctc_head call first, so that only the CTC buffer grows below (a workspace growth
    # drops every graph by itself)
    eng.ctc_head(big, want_log_probs=True, want_argmax=False)
    first = eng.beam_from_enc(enc, enc_lens, **beam)  # captures the beam-step graph against the CTC scorer buffer
    eng.ctc_head(big, want_log_probs=False, want_argmax=True)  # arg-max only: the logits grow the CTC buffer
    again = eng.beam_from_enc(enc, enc_lens, **beam)
    assert len(first[0]) > 0
    assert all(torch.equal(a, b) for a, b in zip(first, again))
