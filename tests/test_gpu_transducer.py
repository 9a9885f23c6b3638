"""Transducer greedy search on the device (csrc/transducer.cu through decoders/transducer.py) against the fp32 CPU oracle
(tests/transducer_oracle.py), walked along the device's decisions: every device decision is the oracle's arg-max or a
near-tie (oracle top-1 / top-2 margin < 5e-3) and the row's summed score is within 1e-2, or 1e-4 relative for rows whose
score sums over a thousand or more tokens (fp16 weights: the per-token error accumulates)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import transducer_oracle as TO  # noqa: E402
from mirrors import build_mirror  # noqa: E402
from parity import normalizer_ckpt, write_pretrained_dir  # noqa: E402

pytestmark = pytest.mark.gpu

MARGIN, SCORE_TOL = 5e-3, 1e-2


def build(J, H, V, blank, seed=1):
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.nnet.embedding import Embedding
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.RNN import LSTM
    from speechbrain_b200.nnet.transducer.transducer_joint import Transducer_joint
    emb = Embedding(num_embeddings=V, consider_as_one_hot=True, blank_id=blank)
    dec = LSTM(input_shape=[None, None, V - 1], hidden_size=H, num_layers=1)
    proj = Linear(input_size=H, n_neurons=J, bias=False)
    lin = Linear(input_size=J, n_neurons=V, bias=False)
    W = TO.seeded_weights(seed, J, H, V, blank)
    mods = {"emb": emb, "dec": dec, "proj_dec": proj, "transducer_lin": lin}
    for prefix, m in mods.items():
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in W.items() if k.startswith(prefix + ".")})
    s = TransducerBeamSearcher([emb, dec, proj], Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU), [lin],
                               blank_id=blank, beam_size=1, nbest=1)
    return s, W, mods


def run_device(s, tn, m, state=None):
    r = s.device_search(tn.device).greedy(tn.contiguous(), s.blank_id, m, state, want_frames=True, want_stats=True)
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in r.items()}


def check_rows(O, tn, blank, m, r, rows):
    for b in rows:
        n = int(r["n_tokens"][b])
        toks, frs = r["tokens"][b, :n].tolist(), r["frames"][b, :n].tolist()
        o = O.row(tn[b], blank, m, forced=(toks, frs))
        assert o["tokens"] == toks, f"row {b}: the forced walk did not follow the device path"
        for (t, tok, lp, am, top1, top2) in o["decisions"]:
            if tok != am:
                assert top1 - top2 < MARGIN, f"row {b} frame {t}: device {tok}, oracle arg-max {am}, margin {top1 - top2}"
        tol = max(SCORE_TOL, 1e-4 * abs(o["score"]))
        assert abs(float(r["logp_sum"][b]) - o["score"]) <= tol, (b, float(r["logp_sum"][b]), o["score"])
        if frs:
            assert int(torch.bincount(torch.tensor(frs)).max()) <= m + 1


CASES = [  # (recipe, B, T, blank, max_symbols_per_step)
    ("librispeech", 4, 251, 0, 5),
    ("librispeech", 1, 1, 0, 5),
    ("librispeech", 3, 17, "last", 1),
    ("commonvoice", 32, 251, 0, 5),
    ("commonvoice", 3, 17, 0, 0),
    ("voxpopuli", 96, 17, "last", 5),
    ("voxpopuli", 1, 3000, 0, 5),
]


@pytest.mark.parametrize("recipe,B,T,blank,m", CASES)
def test_search_matches_oracle(recipe, B, T, blank, m):
    J, H, V = TO.RECIPE_SIZES[recipe]
    blank = V - 1 if blank == "last" else blank
    s, W, _ = build(J, H, V, blank)
    tn = TO.seeded_tn(7, B, T, W)
    r = run_device(s, tn.cuda(), m)
    O = TO.Oracle(W)
    rows = range(B) if B <= 4 else [0, 1, B // 2, B - 1]
    check_rows(O, tn, blank, m, r, rows)
    rounds, barriers = r["stats"].tolist()
    decisions = []  # per row: T blanks and tokens, minus the frames that ended at the symbol cap (no trailing blank)
    for b in range(B):
        n = int(r["n_tokens"][b])
        per_frame = torch.bincount(r["frames"][b, :n].long(), minlength=T) if n else torch.zeros(T, dtype=torch.long)
        decisions.append(T + n - int((per_frame == m + 1).sum()))
    assert rounds == max(decisions) and barriers >= rounds


def test_cap_every_frame():
    """Blank suppressed: every frame hits the cap, exactly (m + 1) * T tokens per row."""
    J, H, V = TO.RECIPE_SIZES["voxpopuli"]
    for m in (0, 1, 5):
        s, W, mods = build(J, H, V, 0)
        w = mods["transducer_lin"].w.weight
        with torch.no_grad():
            w[0] = -50.0 / J ** 0.5 * torch.ones(J)
        tn = TO.seeded_tn(8, 3, 17, W).abs()   # GELU(positive) > 0: the blank logit is strongly negative
        r = run_device(s, tn.cuda(), m)
        assert r["n_tokens"].tolist() == [(m + 1) * 17] * 3


def test_row_independence_and_reruns():
    J, H, V = TO.RECIPE_SIZES["librispeech"]
    s, W, _ = build(J, H, V, 0)
    tn = TO.seeded_tn(9, 32, 251, W).cuda()
    a = run_device(s, tn, 5)
    b = run_device(s, tn, 5)
    for k in ("tokens", "n_tokens", "logp_sum", "h", "c", "out_pn"):
        assert torch.equal(a[k], b[k]), k
    for row in (0, 17, 31):
        one = run_device(s, tn[row:row + 1], 5)
        n = int(a["n_tokens"][row])
        assert int(one["n_tokens"][0]) == n
        assert torch.equal(one["tokens"][0, :n], a["tokens"][row, :n])
        for k in ("logp_sum", "h", "c", "out_pn"):
            assert torch.equal(one[k][0], a[k][row]), (row, k)


def test_streaming_state_carry():
    from speechbrain_b200.decoders.transducer import TransducerGreedySearcherStreamingContext
    J, H, V = TO.RECIPE_SIZES["librispeech"]
    s, W, _ = build(J, H, V, 0)
    tn = TO.seeded_tn(10, 3, 251, W).cuda()
    hyps, score, _, _, (out_pn, (h, c)) = s.transducer_greedy_decode(tn, return_hidden=True)
    ctx = TransducerGreedySearcherStreamingContext()
    got = [[] for _ in range(3)]
    for t0 in range(0, 251, 16):
        for b, hyp in enumerate(s.transducer_greedy_decode_streaming(tn[:, t0:t0 + 16], ctx)):
            got[b] += hyp
    assert got == hyps
    p2, (h2, c2) = ctx.hidden
    assert torch.equal(p2, out_pn) and torch.equal(h2, h) and torch.equal(c2, c)
    assert out_pn.shape == (3, 1, J) and h.shape == (1, 3, H)
    O = TO.Oracle(W)
    ref_hyps, ref_score, _ = O.batch(tn.cpu(), 0, 5)
    assert abs(float(score) - float(ref_score)) <= 1e-2 * max(1.0, float(ref_score))


def test_load_state_dict_after_first_use():
    J, H, V = TO.RECIPE_SIZES["voxpopuli"]
    s, W, mods = build(J, H, V, 0)
    tn = TO.seeded_tn(11, 2, 17, W).cuda()
    s(tn)
    W2 = TO.seeded_weights(5, J, H, V, 0)
    mods["transducer_lin"].load_state_dict({"w.weight": W2["transducer_lin.w.weight"]})
    mods["dec"].load_state_dict({k[4:]: v for k, v in W2.items() if k.startswith("dec.")})
    s(tn)
    W3 = dict(W, **{k: v for k, v in W2.items() if k.startswith(("dec.", "transducer_lin."))})
    assert s.builds == 2
    r = run_device(s, tn, 5)
    check_rows(TO.Oracle(W3), tn.cpu(), 0, 5, r, range(2))


def test_rejections_before_device_work():
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.transducer.transducer_joint import Transducer_joint
    J, H, V = TO.RECIPE_SIZES["voxpopuli"]
    s, W, mods = build(J, H, V, 0)
    joint = Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU)
    dec = [mods["emb"], mods["dec"], mods["proj_dec"]]
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(dec, joint, [mods["transducer_lin"]], blank_id=0, beam_size=4)
    with pytest.raises(NotImplementedError):
        Transducer_joint(joint="concat", nonlinearity=torch.nn.GELU)
    gru = torch.nn.GRU(V - 1, H, batch_first=True)
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher([mods["emb"], gru, mods["proj_dec"]], joint, [mods["transducer_lin"]], blank_id=0, beam_size=1)
    from speechbrain_b200.nnet.RNN import LSTM
    wide = [mods["emb"], LSTM(input_size=V - 1, hidden_size=1088), Linear(input_size=1088, n_neurons=J, bias=False)]
    with pytest.raises(NotImplementedError):
        TransducerBeamSearcher(wide, joint, [mods["transducer_lin"]], blank_id=0, beam_size=1)
    assert s.builds == 0


def _fixture_e2e():
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import make_transducer_golden as MG
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transducer.pt"))["e2e"]
    cfg, sd, w_enc, W, wav, lens = MG.e2e_inputs()
    assert abs(float(wav.double().abs().sum()) - fx["wav_checksum"]) <= 1e-9 * fx["wav_checksum"]
    return fx, cfg, sd, w_enc, W, wav, lens


def _transducer_modules(cfg, sd, w_enc, W):
    """The reference's EncoderDecoderASR layout for the LibriSpeech transducer recipe: encoder = LengthsCapableSequential(
    Fbank, InputNormalization, ConvolutionFrontEnd, EncoderWrapper(12-layer RoPEMHA Conformer), proj_enc), decoder =
    TransducerBeamSearcher(beam_size=1)."""
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.lobes.models.transformer.TransformerASR import EncoderWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.nnet.embedding import Embedding
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.RNN import LSTM
    from speechbrain_b200.nnet.transducer.transducer_joint import Transducer_joint
    mirror = build_mirror(cfg, sd)
    proj_enc = Linear(input_size=512, n_neurons=640, bias=False)
    proj_enc.load_state_dict({"w.weight": w_enc})
    emb = Embedding(num_embeddings=1000, consider_as_one_hot=True, blank_id=0)
    dec = LSTM(input_shape=[None, None, 999], hidden_size=512, num_layers=1)
    proj_dec = Linear(input_size=512, n_neurons=640, bias=False)
    lin = Linear(input_size=640, n_neurons=1000, bias=False)
    for prefix, m in (("emb", emb), ("dec", dec), ("proj_dec", proj_dec), ("transducer_lin", lin)):
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in W.items() if k.startswith(prefix + ".")})
    s = TransducerBeamSearcher([emb, dec, proj_dec], Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU), [lin],
                               blank_id=0, beam_size=1, nbest=1)
    enc = LengthsCapableSequential(mirror.fb, mirror.norm, mirror.cnn, EncoderWrapper(mirror.tr), proj_enc)
    return dict(encoder=enc, decoder=s), dict(CNN=mirror.cnn, Transformer=mirror.tr, proj_enc=proj_enc, emb=emb, dec=dec,
                                               proj_dec=proj_dec, transducer_lin=lin)


def device_decisions(r, b, T, m, blank=0):
    """(frame, token) of every decision of row b, blanks included, from the device's tokens and their frames."""
    n = int(r["n_tokens"][b])
    toks, frs = r["tokens"][b, :n].tolist(), r["frames"][b, :n].tolist()
    out, k = [], 0
    for t in range(T):
        c = 0
        while k < n and frs[k] == t:
            out.append((t, toks[k]))
            k += 1
            c += 1
        if c < m + 1:
            out.append((t, blank))
    return out


def test_encoder_decoder_asr_transducer_end_to_end():
    """The LibriSpeech transducer recipe model against the reference run stored in the fixture: tn_output per-frame norms
    within 1e-3 rel-L2 (padded frames included), every row's decisions equal to the reference's up to its first decision
    with a reference margin < 5e-3, and from there the oracle walked along the device's decisions (check_rows)."""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    fx, cfg, sd, w_enc, W, wav, lens = _fixture_e2e()
    mods, _ = _transducer_modules(cfg, sd, w_enc, W)
    asr = EncoderDecoderASR(modules=mods, hparams={"tokenizer": None, "transducer_beam_search": True},
                            run_opts={"device": "cuda:0"})
    tn = asr.encode_batch(wav.cuda(), lens.cuda())
    B, T, _ = tn.shape
    ref_norms = fx["tn_norms"]
    assert tuple(ref_norms.shape) == (B, T) == (4, 251)
    rel = float((tn.double().norm(dim=-1).cpu() - ref_norms.double()).norm() / ref_norms.double().norm())
    assert rel < 1e-3, rel
    words, hyps = asr.transcribe_batch(wav.cuda(), lens.cuda())
    assert sum(len(h) for h in fx["tokens"]) > 0
    r = run_device(asr.mods["decoder"], tn, fx["m"])
    assert hyps == [r["tokens"][b, :int(r["n_tokens"][b])].tolist() for b in range(B)]
    assert words == [" ".join(map(str, h)) for h in hyps]
    for b in range(B):
        ref = [tuple(x) for x in fx["decisions"][b].tolist()]
        margins = fx["margins"][b].tolist()
        k = next((i for i, mg in enumerate(margins) if mg < MARGIN), len(ref))
        got = device_decisions(r, b, T, fx["m"])
        assert got[:k] == ref[:k], f"row {b}: differs from the reference before its first near-tie (decision {k})"
        if k == len(ref):
            assert hyps[b] == fx["tokens"][b]
    check_rows(TO.Oracle(W), tn.cpu(), 0, fx["m"], r, range(B))


HPARAMS = """
blank_index: 0
activation: !name:torch.nn.GELU
normalizer: !new:speechbrain.processing.features.InputNormalization
    norm_type: global
compute_features: !new:speechbrain.lobes.features.Fbank
    sample_rate: 16000
    n_fft: 512
    n_mels: 80
    win_length: 32
CNN: !new:speechbrain.lobes.models.convolution.ConvolutionFrontEnd
    input_shape: (8, 10, 80)
    num_blocks: 2
    num_layers_per_block: 1
    out_channels: (64, 32)
    kernel_sizes: (3, 3)
    strides: (2, 2)
    residuals: (False, False)
Transformer: !new:speechbrain.lobes.models.transformer.TransformerASR.TransformerASR
    input_size: 640
    tgt_vocab: 1000
    d_model: 512
    nhead: 8
    num_encoder_layers: 12
    num_decoder_layers: 0
    d_ffn: 2048
    dropout: 0.1
    activation: !ref <activation>
    encoder_module: conformer
    attention_type: RoPEMHA
    normalize_before: True
    causal: False
enc: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
    transformer: !ref <Transformer>
proj_enc: !new:speechbrain.nnet.linear.Linear
    input_size: 512
    n_neurons: 640
    bias: False
proj_dec: !new:speechbrain.nnet.linear.Linear
    input_size: 512
    n_neurons: 640
    bias: False
emb: !new:speechbrain.nnet.embedding.Embedding
    num_embeddings: 1000
    consider_as_one_hot: True
    blank_id: !ref <blank_index>
dec: !new:speechbrain.nnet.RNN.LSTM
    input_shape: [null, null, 999]
    hidden_size: 512
    num_layers: 1
    re_init: True
Tjoint: !new:speechbrain.nnet.transducer.transducer_joint.Transducer_joint
    joint: sum
    nonlinearity: !ref <activation>
transducer_lin: !new:speechbrain.nnet.linear.Linear
    input_size: 640
    n_neurons: 1000
    bias: False
decoder: !new:speechbrain.decoders.transducer.TransducerBeamSearcher
    decode_network_lst: [!ref <emb>, !ref <dec>, !ref <proj_dec>]
    tjoint: !ref <Tjoint>
    classifier_network: [!ref <transducer_lin>]
    blank_id: !ref <blank_index>
    beam_size: 1
    nbest: 1
encoder: !new:speechbrain.nnet.containers.LengthsCapableSequential
    input_shape: [null, null, 80]
    compute_features: !ref <compute_features>
    normalize: !ref <normalizer>
    cnn: !ref <CNN>
    transformer_encoder: !ref <enc>
    proj_enc: !ref <proj_enc>
tokenizer: null
transducer_beam_search: True
asr_model: !new:torch.nn.ModuleList
    - [!ref <CNN>, !ref <Transformer>, !ref <proj_enc>, !ref <emb>, !ref <dec>, !ref <proj_dec>, !ref <transducer_lin>]
modules:
    encoder: !ref <encoder>
    decoder: !ref <decoder>
pretrainer: !new:speechbrain.utils.parameter_transfer.Pretrainer
    loadables:
        normalizer: !ref <normalizer>
        asr: !ref <asr_model>
    paths:
        asr: <save_dir>/asr.ckpt
"""


def test_from_hparams_local_directory_matches_direct_construction(tmp_path):
    """A pretrained-model directory with the transducer recipe's module names (hyperparams.yaml, asr.ckpt in the
    ModuleList key layout, normalizer.ckpt) loads through from_hparams and transcribes like direct construction."""
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    fx, cfg, sd, w_enc, W, wav, lens = _fixture_e2e()
    mods, parts = _transducer_modules(cfg, sd, w_enc, W)
    order = ["CNN", "Transformer", "proj_enc", "emb", "dec", "proj_dec", "transducer_lin"]
    ck = {f"{i}.{k}": v for i, n in enumerate(order) for k, v in parts[n].state_dict().items()}
    tmp = write_pretrained_dir(tmp_path, HPARAMS, dict(asr=ck, normalizer=normalizer_ckpt(sd)))
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    assert isinstance(loaded.mods["decoder"], TransducerBeamSearcher) and loaded.transducer_beam_search
    direct = EncoderDecoderASR(modules=mods, hparams={"tokenizer": None, "transducer_beam_search": True},
                               run_opts={"device": "cuda:0"})
    w1, t1 = loaded.transcribe_batch(wav.cuda(), lens.cuda())
    w2, t2 = direct.transcribe_batch(wav.cuda(), lens.cuda())
    assert t1 == t2 and w1 == w2 and sum(len(t) for t in t1) > 0
