"""mirrors.py maps each recipe config onto the TransformerASR keywords the way the device engine reads them back, no GPU
needed: for every config in utils/seeded_init, the mirror's engine_cfg() names the config's encoder module, attention
type and three activations, and the mirror loads the config's whole seeded state."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mirrors import build_mirror, seeded  # noqa: E402
from speechbrain_b200.utils import seeded_init as S  # noqa: E402

CONFIGS = {v["name"]: v for v in vars(S).values() if isinstance(v, dict) and "name" in v}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_mirror_reads_the_recipe_config(name):
    cfg = CONFIGS[name]
    # one layer of each kind: the mapping does not depend on depth, and the full xlarge alone is 480M weights
    small = dict(cfg, num_encoder_layers=1, num_decoder_layers=min(cfg["num_decoder_layers"], 1))
    got = build_mirror(small, seeded(small)).tr.engine_cfg()
    want = dict(encoder_module=cfg.get("encoder_module", "conformer"), attention_type=cfg["attention_type"],
                decoder_activation=cfg["decoder_activation"], conformer_activation=cfg.get("conformer_activation", "swish"),
                branchformer_activation=cfg.get("branchformer_activation", "gelu"))
    assert {k: got[k] for k in want} == want
