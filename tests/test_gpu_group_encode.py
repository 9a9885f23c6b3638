"""-m gpu: a group call encodes its batches several at a time (csrc/engine.cu, group_encode_batches: as many batches as fit in
65536 encoder rows, i.e. 8 batches of 32 x 10 s, the batches spread evenly over that many passes).  Every encoder
kernel works per row or per utterance, so with the decode kernels of a single-batch call at every row count
(set_decoder_tc_min_rows(1 << 30)) the token ids of a group call equal separate transcribe_greedy_dev calls bit for bit:
one pass (G <= 8), a partial last pass (G = 9: 5 + 4 batches) and two full ones (G = 16), each batch with its own
waveforms and ragged lengths."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401

pytestmark = pytest.mark.gpu

B, L, S = 32, 160000, 6  # 32 x 10 s: 251 frames, 8032 encoder rows per batch
PASS = 8                 # batches in one pass of at most 65536 rows
GROUPS = (1, PASS, PASS + 1, 16)


def _engine(base, dev, **kw):
    from speechbrain_b200.engine import AsrEngine
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    cfg = dict(base, num_encoder_layers=2, num_decoder_layers=2, **kw)
    eng = AsrEngine(cfg, seeded_asr_state(cfg, 0), device=dev)
    eng.set_decoder_tc_min_rows(1 << 30)  # the decode kernels of a single-batch call at any row count
    return eng


def _batches(n, seed):
    """n batches of B x L waveforms with their own ragged lengths (zeros past each length), on the host.  Each utterance is
    three tones of its own frequencies and loudness over a little noise: on white noise the seeded 2-layer models give
    nearly the same ids for every utterance, so the ids would not show an utterance reading another one's states."""
    gen = torch.Generator().manual_seed(seed)
    t = torch.arange(L) / 16000.0
    wavs, lens = [], []
    for g in range(n):
        lens_g = 0.3 + 0.7 * torch.rand(B, generator=gen)
        lens_g[g % B] = 1.0
        f = 100 + 5000 * torch.rand(B, 3, generator=gen)
        a = (0.1 + torch.rand(B, 3, generator=gen)) * 10 ** (2 * torch.rand(B, 1, generator=gen))
        w = (a[:, :, None] * torch.sin(2 * math.pi * f[:, :, None] * t)).sum(1) + 0.01 * torch.randn(B, L, generator=gen)
        for b in range(B):
            w[b, int(round(float(lens_g[b]) * L)):] = 0
        wavs.append(w)
        lens.append(lens_g)
    return wavs, lens


def _group(eng, wavs, lens, dev):
    preds = [torch.full((B, S), -7, dtype=torch.int32, device=dev) for _ in wavs]
    eng.transcribe_greedy_group_dev(wavs, lens, S, 1, 2, preds)
    torch.cuda.synchronize()
    return preds


def _singles(eng, wavs, lens):
    out = []
    for w, l_ in zip(wavs, lens):
        pred, _, _, done = eng.transcribe_greedy_dev(w, l_, S, 1, 2)
        assert done == S
        out.append(pred[:, :S].clone())
    torch.cuda.synchronize()
    return out


@pytest.fixture(scope="module", params=("RoPEMHA", "RelPosMHAXL"))
def conformer(request, dev):
    """A Conformer-L-shaped engine, 16 batches on the device and each batch's ids from its own single-batch call."""
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE
    eng = _engine(CONFORMER_LARGE, dev, attention_type=request.param)
    eng.set_poll_interval(0)
    wavs, lens = _batches(16, 11)
    wavs, lens = [w.to(dev) for w in wavs], [l_.to(dev) for l_ in lens]
    ref = _singles(eng, wavs, lens)
    _assert_varied(ref)
    return eng, wavs, lens, ref


def _assert_varied(ref):
    """The reference ids differ between the batches of every pass and between the utterances of every batch, so that a
    wrong length or encoder-state offset inside a pass would change some batch's ids."""
    for g0 in range(0, len(ref), PASS):
        chunk = [r.cpu() for r in ref[g0:g0 + PASS]]
        if len(chunk) > 1:
            assert len({tuple(r.flatten().tolist()) for r in chunk}) == len(chunk), f"pass at batch {g0}: equal batches"
        for g, r in enumerate(chunk):
            assert len({tuple(row.tolist()) for row in r}) > B // 2, f"batch {g0 + g}: too few distinct utterances"


@pytest.mark.parametrize("G", GROUPS)
def test_group_ids_equal_single_batch_calls(conformer, dev, G):
    eng, wavs, lens, ref = conformer
    for _ in range(2):  # capture, then replay of the cached group graph
        preds = _group(eng, wavs[:G], lens[:G], dev)
        for g in range(G):
            assert torch.equal(preds[g], ref[g]), f"G={G} batch {g}"


def test_host_entry_equals_device_entry_at_a_pass_boundary(conformer, dev):
    eng, wavs, lens, ref = conformer
    G = PASS + 1
    wavs_h = [w.cpu().pin_memory() for w in wavs[:G]]
    lens_h = [l_.cpu().pin_memory() for l_ in lens[:G]]
    dev_ids = _group(eng, wavs[:G], lens[:G], dev)
    for poll in (8, 0):  # eager launches, then the whole call as one CUDA graph
        eng.set_poll_interval(poll)
        out = [torch.full((B, S), -7, dtype=torch.int32).pin_memory() for _ in range(G)]
        eng.transcribe_greedy_group_host_async(wavs_h, lens_h, S, 1, 2, out)
        torch.cuda.synchronize()
        for g in range(G):
            assert torch.equal(out[g], dev_ids[g].cpu()) and torch.equal(out[g], ref[g].cpu()), f"poll={poll} batch {g}"


def test_one_encoder_pass_per_chunk(conformer, dev):
    """Eager launches (sbk_launch_count) of a group call: Fbank and the lengths per batch, the CNN and encoder once per pass,
    one decode loop."""
    from speechbrain_b200._lib import lib
    eng, wavs, lens, _ = conformer
    eng.set_poll_interval(8)  # S < 8: exactly S steps, no early exit

    def launches(fn):
        fn()  # warm-up: workspace and step graph for this shape
        torch.cuda.synchronize()
        n0 = lib().sbk_launch_count()
        fn()
        torch.cuda.synchronize()
        return lib().sbk_launch_count() - n0

    n = {G: launches(lambda G=G: _group(eng, wavs[:G], lens[:G], dev)) for G in (1, 2, PASS, PASS + 1, 16)}
    encode = launches(lambda: eng.transcribe_greedy_dev(wavs[0], lens[0], 0, 1, 2))  # Fbank, lengths, one encoder pass
    per_batch = n[2] - n[1]
    assert 0 < per_batch < encode
    assert n[PASS] - n[1] == (PASS - 1) * per_batch                # one pass
    assert n[PASS + 1] - n[PASS] == encode                          # a second pass, with one more batch
    assert n[16] - n[PASS + 1] == (16 - PASS - 1) * per_batch      # still two passes
    eng.set_poll_interval(0)


@pytest.mark.parametrize("model", ("branchformer", "transformer", "hyperconformer"))
def test_other_encoders_group_ids_equal_single_batch_calls(dev, model):
    from speechbrain_b200.utils import seeded_init as si
    base = {"branchformer": si.BRANCHFORMER_LARGE, "transformer": si.TRANSFORMER_LARGE,
            "hyperconformer": si.HYPERCONFORMER_22M}[model]
    eng = _engine(base, dev)
    eng.set_poll_interval(0)
    G = PASS + 1
    wavs, lens = _batches(G, 12)
    wavs, lens = [w.to(dev) for w in wavs], [l_.to(dev) for l_ in lens]
    ref = _singles(eng, wavs, lens)
    _assert_varied(ref)
    preds = _group(eng, wavs, lens, dev)
    for g in range(G):
        assert torch.equal(preds[g], ref[g]), f"{model} batch {g}"


def test_empty_batch_is_an_error(conformer, dev):
    """B = 0 or L = 0 is refused with an error before any workspace or pass-size arithmetic, through both group entries."""
    import ctypes

    from speechbrain_b200._lib import lib
    eng, wavs, lens, _ = conformer
    with pytest.raises(RuntimeError):
        eng.transcribe_greedy_group_dev([torch.empty(0, L, device=dev)], [torch.empty(0, device=dev)], S, 1, 2,
                                        [torch.empty(0, S, dtype=torch.int32, device=dev)])
    pred = torch.empty(B, S, dtype=torch.int32, device=dev)
    pred_h = torch.empty(B, S, dtype=torch.int32).pin_memory()
    wav_h, len_h = wavs[0].cpu().pin_memory(), lens[0].cpu().pin_memory()
    VP = ctypes.c_void_p * 2
    done = ctypes.c_int()
    st = eng._sp()
    for b_, l_ in ((0, L), (B, 0)):  # valid buffers, empty shape
        w, r, p = (VP(wavs[0].data_ptr(), wavs[1].data_ptr()), VP(lens[0].data_ptr(), lens[1].data_ptr()),
                   VP(pred.data_ptr(), pred.data_ptr()))
        assert lib().sbk_asr_transcribe_greedy_group_dev(eng._h, 2, w, r, b_, l_, S, 1, 2, p, ctypes.byref(done), st) != 0
        w, r, p = (VP(wav_h.data_ptr(), wav_h.data_ptr()), VP(len_h.data_ptr(), len_h.data_ptr()),
                   VP(pred_h.data_ptr(), pred_h.data_ptr()))
        assert lib().sbk_asr_transcribe_greedy_group_host_async(eng._h, 2, w, r, b_, l_, S, 1, 2, p, None, ctypes.byref(done),
                                                                st) != 0
    torch.cuda.synchronize()
    ids = _group(eng, wavs[:2], lens[:2], dev)  # the handle still works
    assert all(torch.equal(a, b) for a, b in zip(ids, _singles(eng, wavs[:2], lens[:2])))
