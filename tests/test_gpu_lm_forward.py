"""-m gpu: TransformerLM.forward (whole-sequence prefill on the device) vs the REFERENCE fixture, the fp32 oracle and the
engine's KV-cached step path (position by position, and summed as AsrEngine.lm_rescore does), plus its standalone
properties.  Logits are compared on every position, pad positions included, and some batches hold id 0 inside the valid
length: the key-padding mask removes keys that real positions would otherwise see."""
import os
import sys

import pytest
import torch

from oracle import asr_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev  # noqa: E402,F401

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

pytestmark = pytest.mark.gpu

CFG = dict(d_model=768, nhead=12, num_encoder_layers=12, d_ffn=3072)


def _lm(act="gelu", seed=1):
    from speechbrain_b200.lobes.models.transformer.TransformerLM import TransformerLM
    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    lm = TransformerLM(vocab=5000, d_model=768, nhead=12, num_encoder_layers=12, num_decoder_layers=0, d_ffn=3072, dropout=0.0,
                       activation=torch.nn.GELU if act == "gelu" else torch.nn.ReLU, normalize_before=False)
    sd = seeded_state_dict(lm, seed=seed)
    lm.load_state_dict(sd)
    return lm, sd


@pytest.fixture(scope="module")
def gelu_lm():
    return _lm("gelu")


def _batch(n, s, seed, full=True, interior_pad=0.0):
    """Ragged batch: bos = 1, ids in [3, 5000), padded with 0; the first row spans all s positions.  interior_pad: share of
    the positions after bos, inside each valid length, that hold id 0 (SentencePiece's <unk> in the recipes)."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, s + 1, (n,), generator=g)
    if full:
        lens[0] = s
    tokens = torch.zeros(n, s, dtype=torch.long)
    for i, L in enumerate(lens.tolist()):
        tokens[i, 0] = 1
        tokens[i, 1:L] = torch.randint(3, 5000, (L - 1,), generator=g)
        if interior_pad > 0 and L > 1:
            tokens[i, 1:L][torch.rand(L - 1, generator=g) < interior_pad] = 0
    return tokens, lens


def _check_vs(logits, ref, what):
    """Per sequence on all its positions (pad positions too): rel-L2 <= 2e-3; arg-max identical where ref's top-1/top-2
    margin >= 5e-3."""
    logits, ref = logits.double().cpu(), ref.double().cpu()
    worst = 0.0
    for i in range(ref.shape[0]):
        a, b = logits[i], ref[i]
        worst = max(worst, float((a - b).norm() / b.norm()))
        top2 = b.topk(2, dim=-1).values
        sure = (top2[:, 0] - top2[:, 1]) >= 5e-3
        assert torch.equal(a.argmax(-1)[sure], b.argmax(-1)[sure]), f"{what}: arg-max differs in sequence {i}"
    print(f"{what}: worst per-sequence rel-L2 {worst:.2e}")
    assert worst <= 2e-3, what


def test_lm_forward_reference_golden(dev, gelu_lm):
    lm, sd = gelu_lm
    gold = torch.load(os.path.join(GOLDEN, "lm_forward.pt"))
    tokens, lens = gold["tokens"], gold["lengths"]
    logits = lm(tokens.to(dev)).cpu()
    assert logits.shape == (tokens.shape[0], tokens.shape[1], 5000) and logits.dtype == torch.float32
    valid = torch.arange(tokens.shape[1]).unsqueeze(0) < lens.unsqueeze(1)
    assert ((tokens == 0) & valid).sum() >= 3  # the fixture holds id 0 inside valid lengths
    assert torch.isfinite(logits).all()
    assert (logits.logsumexp(-1) - gold["logsumexp"]).abs().max() < 5e-2  # every position, pad positions included
    top_v, top_i = logits.topk(8, dim=-1)
    margin = gold["top_values"][..., 0] - gold["top_values"][..., 1]
    sure = margin >= 5e-3
    assert torch.equal(top_i[..., 0][sure], gold["top_ids"][..., 0][sure].long())
    idx = gold["sample_idx"].long()
    sample = logits[idx[:, 0], idx[:, 1]].double()
    for k in range(idx.shape[0]):
        ref = gold["sample_logits"][k].double()
        assert float((sample[k] - ref).norm() / ref.norm()) <= 2e-3, tuple(idx[k].tolist())
    with torch.no_grad():
        oracle = O.transformer_lm_forward(tokens, sd, dict(CFG, activation="gelu"))
    _check_vs(logits, oracle, "golden batch vs oracle")


@pytest.mark.parametrize("act,n,s,seed,interior_pad", [
    ("gelu", 4, 1, 11, 0.0),      # s = 1
    ("gelu", 3, 70, 12, 0.0),     # s not a multiple of the 64-key attention block
    ("gelu", 2, 300, 13, 0.0),    # s above 256: five key blocks
    ("gelu", 1, 50, 14, 0.0),     # n = 1
    ("gelu", 64, 48, 15, 0.0),    # n = 64
    ("relu", 5, 90, 16, 0.0),     # ReLU LM
    ("gelu", 6, 150, 17, 0.15),   # id 0 inside the valid lengths, over three key blocks
    ("relu", 3, 64, 18, 0.3),     # the same, one whole block
])
def test_lm_forward_vs_oracle(dev, act, n, s, seed, interior_pad):
    lm, sd = _lm(act)
    tokens, lens = _batch(n, s, seed, interior_pad=interior_pad)
    if interior_pad:
        valid = torch.arange(s).unsqueeze(0) < lens.unsqueeze(1)
        assert ((tokens[:, 1:] == 0) & valid[:, 1:]).sum() >= 5
    logits = lm(tokens.to(dev))
    assert torch.isfinite(logits).all()
    with torch.no_grad():
        ref = O.transformer_lm_forward(tokens, sd, dict(CFG, activation=act))
    _check_vs(logits, ref, f"{act} n={n} s={s} interior id-0 share {interior_pad}")


@pytest.mark.parametrize("n,s,seed", [(5, 70, 41), (64, 24, 42)])  # 64 rows: the step's projections on the wgmma GEMM
def test_lm_forward_equals_step_path_position_by_position(dev, gelu_lm, n, s, seed):
    """The whole-sequence forward and the KV-cached step (the beam search's LM scorer / the rescorer) give the same logits
    at every position of a batch with id 0 inside the valid lengths and as trailing padding."""
    lm, _ = gelu_lm
    tokens, lens = _batch(n, s, seed, interior_pad=0.2)
    td = tokens.to(dev)
    fwd = lm(td)
    step = lm._get_engine(dev).lm_step_logits(td)
    assert torch.isfinite(step).all()
    _check_vs(fwd, step, f"forward vs step path n={n} s={s}")


@pytest.mark.parametrize("temperature", [1.0, 1.15])
def test_lm_forward_agrees_with_step_path(dev, gelu_lm, temperature):
    """Sum over positions of log_softmax(forward / T) at the next token (pad column excluded from the normalisation, as
    the rescorer does) == the engine's KV-cached teacher-forced step path, within 1e-2 per sequence."""
    lm, _ = gelu_lm
    tokens, lens = _batch(12, 40, 21)
    td = tokens.to(dev)
    logits = lm(td).double()
    lp = torch.log_softmax(logits / temperature, dim=-1)
    lp[:, :, 0] = float("-inf")
    tgt = lp[:, :-1].gather(2, td[:, 1:].unsqueeze(2)).squeeze(2) - lp[:, :-1].logsumexp(-1)
    mask = (torch.arange(tokens.shape[1], device=dev).unsqueeze(0) < lens.to(dev).unsqueeze(1))[:, 1:]
    ours = torch.nansum(tgt * mask, dim=-1).cpu()
    step = lm._get_engine(dev).lm_rescore(td, lens, temperature, 0).double().cpu()
    print("forward", ours.tolist(), "step", step.tolist())
    assert (ours - step).abs().max() < 1e-2


def test_lm_forward_batch_invariance_and_determinism(dev, gelu_lm):
    lm, _ = gelu_lm
    gold = torch.load(os.path.join(GOLDEN, "lm_forward.pt"))
    tokens, lens = gold["tokens"].to(dev), gold["lengths"]
    a = lm(tokens)
    b = lm(tokens)
    assert torch.equal(a, b)  # bit-identical reruns
    for i, L in enumerate(lens.tolist()):
        alone = lm(tokens[i:i + 1, :L])
        assert (alone[0] - a[i, :L]).abs().max() <= 1e-5, i


def test_lm_forward_picks_up_load_state_dict(dev):
    lm, sd = _lm("gelu")
    tokens, _ = _batch(2, 20, 31)
    before = lm(tokens.to(dev))
    sd2 = dict(sd)
    sd2["output_proj.layers.2.w.bias"] = sd["output_proj.layers.2.w.bias"] + 1.0
    lm.load_state_dict(sd2)
    after = lm(tokens.to(dev))
    assert (after - before - 1.0).abs().max() < 1e-4  # the vocabulary bias is added in fp32


def test_lm_forward_errors(dev, gelu_lm):
    lm, _ = gelu_lm
    with pytest.raises(RuntimeError):
        lm(torch.ones(1, 4, dtype=torch.long))  # CPU tensor
    with pytest.raises(ValueError):
        lm(torch.ones(1, lm.max_length + 1, dtype=torch.long, device=dev))
    with pytest.raises(IndexError):
        lm(torch.full((1, 3), 5000, dtype=torch.long, device=dev))
    eng = lm._get_engine(dev)
    with pytest.raises(RuntimeError, match="max_len"):  # the C ABI's own check
        eng.lm_forward(torch.ones(1, eng.cfg.get("max_length", 2500) + 1, dtype=torch.int32, device=dev))
    with pytest.raises(RuntimeError, match="65535"):
        eng.lm_forward(torch.ones(65536, 1, dtype=torch.int32, device=dev))
    # the C ABI does not range-check ids on the host: an id >= vocab reads nothing out of bounds, it turns its sequence into
    # NaN (its NaN value rows reach every query of the key block through 0 * NaN); the other sequences are unaffected
    out = eng.lm_forward(torch.tensor([[1, 5000, 3, 4], [1, 3, 4, 5]], dtype=torch.int32, device=dev))
    assert torch.isnan(out[0, 1:]).all() and torch.isfinite(out[1]).all()
