"""-m gpu: the chunk-by-chunk streaming encoder (TransformerASR.encode_streaming on per-layer device caches).

Bars: the streamed encoder output equals the masked full-sequence run encode(..., dynchunktrain_config) within 3e-4
rel-L2 (same maths; the chunk's keys are grouped into other 64-key blocks, so the online softmax sums in another order).
A finite-context stream's per-chunk work does not grow with its length (equal kernel-launch counts at chunks 5 and 60, and
a chunk past max_length frames equal to a fresh stream fed only that chunk's receptive field).  Reruns, reset and a stream
inside a batch are bit-identical."""
import os
import pytest
import sys
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import dev, rel  # noqa: E402,F401

pytestmark = pytest.mark.gpu


_MODELS = {}


def _model(dev, base, att, n_layers):
    import bench
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, CONFORMER_SMALL, seeded_asr_state
    key = (base, att, n_layers)
    if key not in _MODELS:
        cfg = dict(CONFORMER_LARGE if base == "large" else CONFORMER_SMALL, attention_type=att, num_encoder_layers=n_layers,
                   num_decoder_layers=1)
        _MODELS[key] = bench.build_product_asr(cfg, seeded_asr_state(cfg, 0), dev).transformer
    return _MODELS[key]


def _stream(tr, src, dc, ctx=None):
    ctx = ctx or tr.make_streaming_context(dc)
    cs = dc.chunk_size
    return torch.cat([tr.encode_streaming(src[:, t:t + cs].contiguous(), ctx) for t in range(0, src.shape[1], cs)], dim=1), ctx


@pytest.mark.parametrize("base,att,cs,lc,B", [
    ("large", "RoPEMHA", 24, 8, 1),      # the model card's DynChunkTrainConfig(24, 8): cache of 192 frames
    ("large", "RoPEMHA", 16, None, 5),   # infinite left context, the ring grows
    ("large", "RoPEMHA", 8, 0, 2),       # no left context: the chunk and the convolution carry only
    ("large", "RelPosMHAXL", 8, 2, 5),
    ("large", "RelPosMHAXL", 6, None, 1),
    ("small", "RelPosMHAXL", 16, 4, 2),  # head width 36 (Conformer-S)
])
def test_streaming_equals_masked(dev, base, att, cs, lc, B):
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _model(dev, base, att, 3)
    gen = torch.Generator().manual_seed(cs * 10 + B)
    T = 14 * cs + 5  # a short last chunk
    src = torch.randn(B, T, 640, generator=gen).to(dev)
    dc = DynChunkTrainConfig(cs, lc)
    full = tr.encode(src, None, dynchunktrain_config=dc)
    out, ctx = _stream(tr, src, dc)
    r = rel(out.cpu(), full.cpu())
    per_chunk = max(rel(out[:, t:t + cs].cpu(), full[:, t:t + cs].cpu()) for t in range(0, T, cs))
    print(f"[stream {base} {att} ({cs}, {lc}) B={B}] rel vs masked {r:.2e}, worst chunk {per_chunk:.2e}")
    assert out.shape == full.shape and r < 3e-4 and per_chunk < 6e-4
    layer = ctx.encoder_context.layers[0]
    kept = T if lc is None else min(T, lc * cs)
    assert ctx.history.shape == (B, kept, tr.d_model) and layer.mha_left_context.shape == (B, kept, tr.d_model)
    assert layer.dcconv_left_context.shape == (B, (tr.kernel_size - 1) // 2, tr.d_model)
    assert layer.mha_left_context_size == (None if lc is None else lc * cs)


def test_cache_cost_is_constant(dev):
    """A finite-context stream: equal launch counts per chunk at chunk 5 and chunk 60, bounded memory, and a chunk past
    max_length frames (RoPE positions beyond the full-sequence table) equal to a fresh stream fed only the frames that
    chunk can depend on."""
    from speechbrain_b200._lib import lib
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _model(dev, "large", "RoPEMHA", 2)
    cs, lc = 8, 2
    dc = DynChunkTrainConfig(cs, lc)
    n_chunks = 330  # 2640 frames > max_length = 2500
    gen = torch.Generator().manual_seed(7)
    src = torch.randn(1, n_chunks * cs, 640, generator=gen).to(dev)
    ctx = tr.make_streaming_context(dc)
    deltas, outs = {}, []
    for k in range(n_chunks):
        n0 = lib().sbk_launch_count()
        outs.append(tr.encode_streaming(src[:, k * cs:(k + 1) * cs].contiguous(), ctx))
        deltas[k] = lib().sbk_launch_count() - n0
    print(f"[stream cost] launches per chunk at 5: {deltas[5]}, at 60: {deltas[60]}, at {n_chunks - 1}: {deltas[n_chunks - 1]}")
    assert deltas[5] == deltas[60] == deltas[n_chunks - 1] > 0
    assert ctx.history.shape[1] == lc * cs
    # receptive field of a chunk: per layer lc chunks of attention or the convolution's 15 frames, so 2 layers < 8 chunks
    R = 8
    first = n_chunks - 1 - R
    fresh, _ = _stream(tr, src[:, first * cs:].contiguous(), dc)
    r = rel(fresh[:, -cs:].cpu(), outs[-1].cpu())
    print(f"[stream cost] chunk {n_chunks - 1} (frames {(n_chunks - 1) * cs}..) vs a fresh stream over its receptive field: {r:.2e}")
    assert r < 3e-4


def test_bit_identical_reruns_reset_and_batch(dev):
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _model(dev, "large", "RelPosMHAXL", 2)
    dc = DynChunkTrainConfig(16, 2)
    gen = torch.Generator().manual_seed(3)
    src = torch.randn(4, 16 * 9, 640, generator=gen).to(dev)
    a, ctx = _stream(tr, src, dc)
    b, _ = _stream(tr, src, dc)
    assert torch.equal(a, b)
    ctx.reset()
    assert ctx.history is None
    c, _ = _stream(tr, src, dc, ctx)
    assert torch.equal(a, c)
    for i in range(4):  # a stream alone equals the same stream inside the batch of 4
        alone, _ = _stream(tr, src[i:i + 1].contiguous(), dc)
        assert torch.equal(alone, a[i:i + 1])


def test_rejections_before_device_work(dev):
    from speechbrain_b200._lib import lib
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    tr = _model(dev, "large", "RoPEMHA", 2)
    dc = DynChunkTrainConfig(8, 1)
    ctx = tr.make_streaming_context(dc)
    gen = torch.Generator().manual_seed(1)
    src = torch.randn(2, 40, 640, generator=gen)
    tr.encode_streaming(src[:, :8].to(dev), ctx)
    torch.cuda.synchronize()
    n0 = lib().sbk_launch_count()
    with pytest.raises(RuntimeError, match="chunk size"):  # longer than the chunk size
        tr.encode_streaming(src[:, 8:17].contiguous().to(dev), ctx)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        tr.encode_streaming(src[:, 8:16].contiguous(), ctx)
    assert lib().sbk_launch_count() == n0 and ctx.history.shape[1] == 8
    tr.encode_streaming(src[:, 8:13].contiguous().to(dev), ctx)  # a short chunk ends the stream
    n0 = lib().sbk_launch_count()
    with pytest.raises(RuntimeError, match="last chunk"):
        tr.encode_streaming(src[:, 13:21].contiguous().to(dev), ctx)
    assert lib().sbk_launch_count() == n0
    from speechbrain_b200.lobes.models.transformer.TransformerASR import TransformerASR
    for kw in (dict(encoder_module="transformer", attention_type="regularMHA", d_model=256, nhead=4),
               dict(encoder_module="branchformer", attention_type="RelPosMHAXL", d_model=256, nhead=4),
               dict(encoder_module="conformer", attention_type="hypermixing", d_model=256, nhead=4)):
        other = TransformerASR(5000, 640, num_encoder_layers=1, num_decoder_layers=1, normalize_before=True, causal=False,
                               d_ffn=512, **kw)
        with pytest.raises(NotImplementedError):
            other.make_streaming_context(dc)


@pytest.mark.parametrize("pos0", [0, 10 ** 7, 10 ** 9])
def test_rope_ring_write_far_into_a_stream(dev, pos0):
    """Keys rotated once by their stream position give the scores of the reference's window-local rotation, however far
    into the stream (10^9 frames is about 1.3 years of audio): float64 scores of the kernel's fp16 q / k against float64
    scores of q and k rotated by their window positions 0..n-1."""
    import ctypes
    import math

    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    H, dh, n, cap, slot0 = 2, 64, 16, 24, 20  # the chunk's rows wrap around the ring
    d = H * dh
    gen = torch.Generator().manual_seed(11)
    qkv = torch.randn(n, 3 * d, generator=gen)
    inv = torch.exp(torch.arange(0, dh, 2, dtype=torch.float32) * -(math.log(10000.0) / dh))
    scale = 1.0 / math.sqrt(d)
    q = torch.empty(n, d, dtype=torch.float16, device=dev)
    kv = torch.zeros(1, cap, 2 * d, dtype=torch.float16, device=dev)
    qkv_d, inv_d = qkv.to(dev), inv.to(dev)
    check(lib().sbk_stream_qkv_test(ptr(qkv_d), 1, n, H, dh, ptr(inv_d), ctypes.c_longlong(pos0), ctypes.c_float(scale),
                                    ptr(q), ptr(kv), cap, slot0, stream_ptr(dev)), "sbk_stream_qkv_test")
    slots = [(slot0 + i) % cap for i in range(n)]
    ring = kv[0, slots].double().cpu().view(n, H, 2, dh)
    qh = q.double().cpu().view(n, H, dh)

    def rotate(x, pos):  # x [n, dh], adjacent pairs rotated by pos * inv_freq in float64
        ang = pos[:, None].double() * inv.double()[None, :]
        c, s = torch.cos(ang), torch.sin(ang)
        x0, x1 = x[:, 0::2], x[:, 1::2]
        out = torch.empty_like(x)
        out[:, 0::2], out[:, 1::2] = x0 * c - x1 * s, x1 * c + x0 * s
        return out
    win = torch.arange(n)
    worst = 0.0
    for h in range(H):
        blk = qkv.double().view(n, H, 3, dh)[:, h]
        ref = (rotate(blk[:, 0], win) * scale) @ rotate(blk[:, 1], win).T
        got = qh[:, h] @ ring[:, h, 0].T
        worst = max(worst, rel(got, ref))
        assert torch.equal(ring[:, h, 1], blk[:, 2].half().double())  # values pass through
    print(f"[ring write pos0={pos0}] scores vs window-local float64 rotation: rel {worst:.2e}")
    assert worst < 1e-3


@pytest.mark.parametrize("name", ["rope_24_8", "rope_8_2", "rope_16_1", "relpos_16_2"])
def test_encoder_vs_reference_golden(dev, name):
    """Every chunk of the 12-layer Conformer-L stream against the reference's encode_streaming
    (tests/golden/streaming.pt, tools/make_streaming_golden.py): per-frame output norms and one whole chunk taken after
    the caches filled, rel-L2 <= 1e-3."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import make_streaming_golden as MG

    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    g = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "streaming.pt"))["cases"][name]
    src, T = MG.case_input(g)
    assert abs(float(src.double().abs().sum()) - g["src_checksum"]) < 1e-6 * g["src_checksum"]
    tr = _model(dev, "large", g["att"], 12)
    dc = DynChunkTrainConfig(g["chunk"], g["left"])
    ctx = tr.make_streaming_context(dc)
    src = src.to(dev)
    worst = 0.0
    for k, t in enumerate(range(0, T, g["chunk"])):
        out = tr.encode_streaming(src[:, t:t + g["chunk"]].contiguous(), ctx).cpu()
        worst = max(worst, rel(out.double().norm(dim=-1), g["frame_norms"][k]))
        if k == g["full_chunk_index"]:
            full = rel(out, g["full_chunk"])
    print(f"[golden {name}] worst chunk frame-norm rel {worst:.2e}; chunk {g['full_chunk_index']} rel-L2 {full:.2e}")
    assert worst < 1e-3 and full < 1e-3
