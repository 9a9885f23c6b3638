"""CPU checks of tests/golden/streaming.pt (the reference's chunk-by-chunk TransformerASR.encode_streaming,
tools/make_streaming_golden.py): the inputs regenerate from their seeds, and every case holds one output per chunk with the
reference's left-context sizes."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_streaming_golden as MG  # noqa: E402


def test_golden_inputs_and_layout():
    gd = torch.load(os.path.join(ROOT, "tests", "golden", "streaming.pt"))
    assert sorted(gd["cases"]) == sorted(c["name"] for c in MG.CASES)
    for case in MG.CASES:
        g = gd["cases"][case["name"]]
        src, T = MG.case_input(case)
        assert abs(float(src.double().abs().sum()) - g["src_checksum"]) < 1e-6 * g["src_checksum"]
        n_chunks = -(-T // case["chunk"])
        assert len(g["frame_norms"]) == n_chunks and g["frame_norms"][-1].shape == (MG.B, MG.SHORT)
        assert g["full_chunk"].shape == (MG.B, case["chunk"], 512)
        assert g["full_chunk_index"] * case["chunk"] >= case["left"] * case["chunk"]  # taken after the caches filled
        assert torch.isfinite(g["full_chunk"]).all()
