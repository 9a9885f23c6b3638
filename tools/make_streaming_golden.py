"""Generate tests/golden/streaming.pt by RUNNING THE REFERENCE TransformerASR.encode_streaming (speechbrain.lobes.models.
transformer.TransformerASR, Conformer.py forward_streaming with its per-layer mha / dcconv left contexts) chunk by chunk.

How to run it: oracle/goldens.py.  Models: the Conformer-L encoder (12 layers, d_model 512) with seeded weights (seeded_init.seeded_asr_state, seed 0), RoPEMHA
with DynChunkTrainConfig (24, 8), (8, 2) and (16, 1), and RelPosMHAXL with (16, 2).  Input: a 2-stream batch of encoder-input
frames [2, T, 640] from a seed (checksummed), 14 full chunks and a short last one, so the (24, 8) caches fill.  Per case
it stores the per-frame L2 norms of every chunk's output and the whole output of one chunk taken after the caches filled.
The reference rejects an unlimited left context, so every case has a finite one."""
import torch

from oracle import goldens as G

CASES = [dict(name="rope_24_8", att="RoPEMHA", chunk=24, left=8, seed=101),
         dict(name="rope_8_2", att="RoPEMHA", chunk=8, left=2, seed=102),
         dict(name="rope_16_1", att="RoPEMHA", chunk=16, left=1, seed=103),
         dict(name="relpos_16_2", att="RelPosMHAXL", chunk=16, left=2, seed=104)]
B, FULL_CHUNKS, SHORT = 2, 14, 5


def case_input(case):
    """The encoder input of a case [B, T, 640] and its frame count."""
    T = FULL_CHUNKS * case["chunk"] + SHORT
    g = torch.Generator().manual_seed(case["seed"])
    return torch.randn(B, T, 640, generator=g), T


def case_cfg(case):
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE
    return dict(CONFORMER_LARGE, attention_type=case["att"], num_decoder_layers=1)


def main():
    import speechbrain  # noqa: F401
    from speechbrain.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain.utils.dynamic_chunk_training import DynChunkTrainConfig

    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    out = dict(weight_seed=0, B=B, full_chunks=FULL_CHUNKS, short=SHORT, cases={})
    for case in CASES:
        cfg = case_cfg(case)
        tr = TransformerASR(input_size=cfg["input_size"], tgt_vocab=cfg["vocab"], d_model=cfg["d_model"], nhead=cfg["nhead"],
                            num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=cfg["num_decoder_layers"],
                            d_ffn=cfg["d_ffn"], dropout=0.1, activation=torch.nn.GELU, encoder_module="conformer",
                            attention_type=case["att"], normalize_before=True, causal=False)
        sd = seeded_asr_state(cfg, 0)
        res = tr.load_state_dict({k[len("Transformer."):]: v for k, v in sd.items() if k.startswith("Transformer.")},
                                 strict=False)
        assert not res.unexpected_keys and all(".pe" in k or "inv_freq" in k for k in res.missing_keys), res  # fixed tables
        tr.eval()
        src, T = case_input(case)
        dc = DynChunkTrainConfig(case["chunk"], case["left"])
        ctx = tr.make_streaming_context(dc)
        norms, outs = [], []
        with torch.no_grad():
            for t in range(0, T, case["chunk"]):
                o = tr.encode_streaming(src[:, t:t + case["chunk"]], ctx)
                outs.append(o)
                norms.append(o.double().norm(dim=-1).float())
            full = tr.encode(src, None, dynchunktrain_config=dc)
        stream = torch.cat(outs, dim=1)
        r = G.rel(stream, full)
        keep = FULL_CHUNKS - 2  # a chunk after every cache has filled
        print(f"[{case['name']}] {len(outs)} chunks; reference streaming vs its masked encode rel {r:.2e}; "
              f"layer 0 left context {tuple(ctx.encoder_context.layers[0].mha_left_context.shape)}")
        assert r < 1e-5
        out["cases"][case["name"]] = dict(case, src_checksum=float(src.double().abs().sum()), frame_norms=norms,
                                          full_chunk_index=keep, full_chunk=outs[keep].clone())
    G.save(out, "streaming.pt")


if __name__ == "__main__":
    main()
