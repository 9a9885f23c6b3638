"""-m gpu tests of GigaSpeech's Conformer-Transducer encoder (12 layers, d_model 768, RelPosMHAXL with 8 heads of 96).

Kernel level, through sbk_encoder_attention_window_test (sbk_encoder_attention_test keeps refusing head width 96), on the
inputs, float64 references and bars of test_gpu_encoder_kernels.py:
- the full-sequence form at head width 96 with RelPosMHAXL: the full-context T list, the Dynamic Chunk windows and T up to
  2500 (max_len); reruns are bit-identical and an utterance alone equals its rows in the batch;
- the stream form (one chunk's queries against a ring of cached keys and values) at 96 and at every width already streamed
  (64, 36, 32; RoPE / plain at 64 and 32): wrapped and unwrapped rings, one and several query tiles, compared with the same
  float64 reference over the window.  Ring slots outside the window hold +-3e4, so a read past the window shows.

Model level, on seeded weights (gigaspeech_oracle.py), against the fp32 CPU oracle recomputed here:
- wav -> encoder states, all frames and valid frames, rel-L2 <= ENC_BAR, with full context and with DynChunkTrainConfig
  (16, 2); a rerun is bit-identical and an utterance alone equals its rows in the batch;
- the streaming encoder (TransformerASR.encode_streaming) equals the masked full-sequence run within 3e-4 per stream, at
  the recipe README's (32, 4), (16, 8) and (8, 2) and with an unlimited left context; reruns, reset and a stream inside a
  batch of 4 are bit-identical;
- the greedy transducer search on proj_enc of the device's encoder states: decisions equal to the oracle's on the oracle's
  states up to the first near-tie, and the oracle walked along the device's path accepts every decision
  (test_gpu_transducer.check_rows, with a score bound for long low-confidence paths); the beam-10 search (state_beam = expand_beam = 2.3) replayed decision by decision
  through the beam oracle (test_gpu_transducer_beam.check_replay)."""
import ctypes
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gigaspeech_oracle as GO  # noqa: E402
import test_gpu_encoder_kernels as EKT  # noqa: E402
import test_gpu_transducer as GT  # noqa: E402
import test_gpu_transducer_beam as BT  # noqa: E402
import transducer_oracle as TO  # noqa: E402
from parity import check_alone_vs_batch, check_encoder, dev, rel  # noqa: E402,F401

ENC_BAR = 1e-3
STREAM_BAR = 3e-4

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ kernel at head width 96
def _att_win(qkv, B, T, H, dh, lens, relpos, u, w, P, scale, chunk=0, left=-1, kv=None, cap=0, start=0, nq=0):
    from speechbrain_b200._lib import check, lib, ptr, stream_ptr
    rows = B * (nq if kv is not None else T)
    out = torch.full((rows, H * dh), float("nan"), dtype=torch.float16, device=qkv.device)
    check(lib().sbk_encoder_attention_window_test(ptr(qkv), ptr(kv), B, T, H, dh, ptr(lens), int(relpos), ptr(u), ptr(w),
                                                  ptr(P), ctypes.c_float(scale), chunk, left, cap, start, nq, ptr(out),
                                                  stream_ptr(qkv.device)),
          "sbk_encoder_attention_window_test")
    return out


def _run96(dev, name, B, T, H, lens, seed, chunk=0, left=-1):
    lens_dev = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    lens_t = None if lens is None else torch.tensor(lens)
    qkv, (u, w, P), scale = EKT._att_inputs(B, T, H, 96, lens_t, True, seed, dev)
    out = _att_win(qkv, B, T, H, 96, lens_dev, True, u, w, P, scale, chunk, left)
    ref = EKT._att_ref(qkv, B, T, H, 96, lens_t, True, u, w, P, scale, chunk, left)
    seen = EKT._att_check(name, out, ref, lens_t, True, chunk, left)
    assert torch.equal(out, _att_win(qkv, B, T, H, 96, lens_dev, True, u, w, P, scale, chunk, left)), f"{name}: rerun differs"
    return qkv, (u, w, P), scale, out, seen


@pytest.mark.parametrize("T", [1, 17, 63, 64, 65, 251, 1000])
def test_attention96_full_context(dev, T):
    """B = 3 with lengths {T, not a multiple of 64, 1}; H = 8 at T = 251; the middle utterance alone is bit-identical to its
    rows in the batch; T = 65 and 251 also run without lengths"""
    H = 8 if T == 251 else 2
    lens = [T, EKT._ragged_len(T), 1]
    name = f"dh=96 relpos T={T}"
    qkv, (u, w, P), scale, out, _ = _run96(dev, name, 3, T, H, lens, T * 131 + 96 * 7 + 1)
    alone = _att_win(qkv[T:2 * T].contiguous(), 1, T, H, 96, torch.tensor(lens[1:2], dtype=torch.int32, device=dev), True,
                     u, w, P, scale)
    assert torch.equal(alone, out[T:2 * T]), f"{name}: B = 1 differs from the batch"
    if T in (65, 251):
        _run96(dev, name + " no lens", 2, T, H, None, T * 17 + 97)


@pytest.mark.parametrize("T", [251, 300])
@pytest.mark.parametrize("chunk,left", EKT.WINDOWS)
def test_attention96_dynamic_chunk(dev, chunk, left, T):
    lens = [T, EKT._ragged_len(T), 20]
    _, _, _, _, seen = _run96(dev, f"dh=96 relpos T={T} chunk={chunk} left={left}", 3, T, 2, lens,
                              T * 7 + chunk * 101 + left + 97, chunk, left)
    if left >= 0:
        assert not seen[2].all(), "the case should hold rows without a visible key"


@pytest.mark.parametrize("T", [1036, 1037, 1500, 2500])
def test_attention96_relpos_long(dev, T):
    _run96(dev, f"dh=96 relpos long T={T}", 2, T, 2, [T, EKT._ragged_len(T)], T + 96)


def test_attention96_built_for_relpos_only(dev):
    from speechbrain_b200._lib import lib, ptr, stream_ptr
    T, H = 16, 2
    qkv = torch.zeros(T, 3 * H * 128, dtype=torch.float16, device=dev)
    out = torch.zeros(T, H * 128, dtype=torch.float16, device=dev)
    uv = torch.zeros(H * 128, device=dev)
    P = torch.zeros(T, H * 128, dtype=torch.float16, device=dev)
    st = stream_ptr(dev)
    new = lambda dh, rp: lib().sbk_encoder_attention_window_test(ptr(qkv), None, 1, T, H, dh, None, rp, ptr(uv), ptr(uv),  # noqa: E731
                                                                 ptr(P), ctypes.c_float(0.1), 0, -1, 0, 0, 0, ptr(out), st)
    old = lambda dh, rp: lib().sbk_encoder_attention_test(ptr(qkv), 1, T, H, dh, None, rp, ptr(uv), ptr(uv), ptr(P),  # noqa: E731
                                                          ctypes.c_float(0.1), 0, -1, ptr(out), st)
    assert new(96, 1) == 0 and new(96, 0) != 0 and new(128, 1) != 0 and new(48, 1) != 0
    assert old(96, 1) != 0 and old(96, 0) != 0 and old(80, 1) == 0


# (W window rows, nq queries, cap, start): the first chunk, a wrapped ring, several query tiles, a window that fills the ring
RINGS = [(16, 16, 32, 0), (48, 16, 64, 40), (150, 16, 160, 100), (200, 100, 256, 250), (320, 64, 320, 7)]
STREAMED = [(96, True), (64, True), (36, True), (32, True), (64, False), (32, False)]


@pytest.mark.parametrize("W,nq,cap,start", RINGS)
@pytest.mark.parametrize("dh,relpos", STREAMED)
def test_attention_stream_form(dev, dh, relpos, W, nq, cap, start):
    """one chunk's nq queries against the window's W keys / values in a ring of cap slots from slot start, against the
    float64 reference over the window (every key visible); H = 8 on the (150, 16) ring"""
    B, H = 2, 8 if W == 150 else 2
    d = H * dh
    name = f"stream dh={dh} {'relpos' if relpos else 'plain'} W={W} nq={nq} cap={cap} start={start}"
    qkv, (u, w, P), scale = EKT._att_inputs(B, W, H, dh, None, relpos, W * 13 + dh + cap + relpos, dev)
    x = qkv.view(B, W, H, 3 * dh)
    q = x[:, W - nq:, :, :dh].reshape(B * nq, d).contiguous()
    g = torch.Generator().manual_seed(cap + start)
    ring = (3e4 * torch.sign(torch.randn(B, cap, H, 2 * dh, generator=g))).half().to(dev)  # slots outside the window
    slots = (start + torch.arange(W, device=dev)) % cap
    ring[:, slots] = x[:, :, :, dh:]
    ring = ring.view(B, cap, 2 * d).contiguous()
    out = _att_win(q, B, W, H, dh, None, relpos, u, w, P, scale, kv=ring, cap=cap, start=start, nq=nq)
    ref = EKT._att_ref(qkv, B, W, H, dh, None, relpos, u, w, P, scale)[:, W - nq:]
    EKT._att_check(name, out, ref, None, relpos)
    again = _att_win(q, B, W, H, dh, None, relpos, u, w, P, scale, kv=ring, cap=cap, start=start, nq=nq)
    assert torch.equal(out, again), f"{name}: rerun differs"


# ------------------------------------------------------------------------------------------------ model level
_CASE = {}


def _case(dev):
    """the seeded model on the device (TransformerASR mirror and AsrEngine), its weights, the waveforms and the oracle's
    encoder states and proj_enc output"""
    if not _CASE:
        from mirrors import build_mirror
        from speechbrain_b200.engine import AsrEngine
        cfg = GO.config()
        sd, w_enc, W = GO.weights()
        wav, lens = GO.waveforms()
        enc = GO.encode(sd, wav, lens)
        _CASE.update(cfg=cfg, sd=sd, w_enc=w_enc, W=W, wav=wav, lens=lens, enc=enc, T=enc.shape[1],
                     tn=GO.tn_output(enc, w_enc), eng=AsrEngine(cfg, sd, device=str(dev)), tr=build_mirror(cfg, sd).tr)
    return _CASE


def test_encoder_full_context(dev):
    c = _case(dev)
    wav, lens = c["wav"].to(dev), c["lens"].to(dev)
    enc = c["eng"].encode_wav(wav, lens)
    torch.cuda.synchronize()
    check_encoder("gigaspeech", enc.cpu(), c["enc"], [round(float(x) * c["T"]) for x in c["lens"]], ENC_BAR)
    assert torch.equal(enc, c["eng"].encode_wav(wav, lens)), "rerun differs"
    check_alone_vs_batch(lambda w, ln: (c["eng"].encode_wav(w, ln),), wav, lens, 1e-5, relative=True)


def test_encoder_dynamic_chunk(dev):
    """the masked full-sequence encode with DynChunkTrainConfig(16, 2) against the oracle's masked encode"""
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    c = _case(dev)
    ref = GO.encode(c["sd"], c["wav"], c["lens"], dynchunk=GO.DYNCHUNK)
    src = _front_end(dev, c)
    out = c["tr"].encode(src, c["lens"].to(dev), dynchunktrain_config=DynChunkTrainConfig(*GO.DYNCHUNK))
    check_encoder("gigaspeech dynchunk (16, 2)", out.cpu(), ref, [round(float(x) * c["T"]) for x in c["lens"]], ENC_BAR)


def _front_end(dev, c):
    """the mirror front end (Fbank -> global CMVN -> ConvolutionFrontEnd) of the batch on the device: [B, T, 640]"""
    from mirrors import build_mirror
    if "mirror" not in c:
        c["mirror"] = build_mirror(c["cfg"], c["sd"])
    x = c["mirror"].front_end()(c["wav"].to(dev), c["lens"].to(dev))
    return x.reshape(x.shape[0], x.shape[1], -1)


def _stream(tr, src, dc, ctx=None):
    ctx = ctx or tr.make_streaming_context(dc)
    cs = dc.chunk_size
    return torch.cat([tr.encode_streaming(src[:, t:t + cs].contiguous(), ctx) for t in range(0, src.shape[1], cs)], dim=1), ctx


@pytest.mark.parametrize("cs,lc", [(32, 4), (16, 8), (8, 2), (16, None)])
def test_streaming_equals_masked(dev, cs, lc):
    """chunk by chunk on the device equals the masked full-sequence run, per stream, on the batch's front-end output"""
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    c = _case(dev)
    src = _front_end(dev, c)[:3, :150].contiguous()  # the first 6 s of three rows: a short last chunk at 16 and 32
    dc = DynChunkTrainConfig(cs, lc)
    full = c["tr"].encode(src, None, dynchunktrain_config=dc)
    out, _ = _stream(c["tr"], src, dc)
    worst = max(rel(out[b].cpu(), full[b].cpu()) for b in range(src.shape[0]))
    print(f"MEASURE gigaspeech stream ({cs}, {lc}) vs masked full sequence: worst stream rel-L2 {worst:.2e}")
    assert out.shape == full.shape and worst < STREAM_BAR


def test_streaming_reruns_reset_and_batch(dev):
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    c = _case(dev)
    src = _front_end(dev, c)[:, :128].contiguous()
    dc = DynChunkTrainConfig(16, 8)
    a, ctx = _stream(c["tr"], src, dc)
    b, _ = _stream(c["tr"], src, dc)
    ctx.reset()
    d, _ = _stream(c["tr"], src, dc, ctx)
    assert torch.equal(a, b) and torch.equal(a, d)
    alone, _ = _stream(c["tr"], src[2:3].contiguous(), dc)
    assert torch.equal(alone, a[2:3])


def test_transducer_greedy_and_beam(dev):
    """greedy: the device's decisions on its own proj_enc output equal the oracle's on the oracle's up to the first
    near-tie, and the oracle walked along the device's path accepts every decision; beam 10: replayed through the oracle"""
    c = _case(dev)
    enc = c["eng"].encode_wav(c["wav"].to(dev), c["lens"].to(dev))
    tn = GO.tn_output(enc, c["w_enc"].to(dev)).contiguous()
    s, _ = _searcher(c, 1)
    r = GT.run_device(s, tn, GO.MAX_SYMBOLS)
    ref = GO.greedy(c["W"], c["tn"])
    B, T = tn.shape[:2]
    n_tok = 0
    for b in range(B):
        got = GT.device_decisions(r, b, T, GO.MAX_SYMBOLS)
        dec = ref[b]["decisions"]
        cut = next((i for i, d in enumerate(dec) if d[4] - d[5] < GT.MARGIN), len(dec))
        assert got[:cut] == [(d[0], d[1]) for d in dec[:cut]], f"row {b}: differs before its first near-tie ({cut})"
        n_tok += int(r["n_tokens"][b])
    _check_rows(c["W"], tn.cpu(), r, range(B))
    assert n_tok > 0
    sb, _ = _searcher(c, GO.BEAM)
    rb = BT.run_device(sb, tn)
    BT.check_replay(c["W"], tn.cpu(), sb, rb, range(B))
    print(f"MEASURE gigaspeech greedy tokens per row {[int(x) for x in r['n_tokens']]}, beam-10 best lengths "
          f"{[int(x) for x in rb['lens'][:, 0]]}")


def _check_rows(W, tn, r, rows):
    """test_gpu_transducer.check_rows with a score bound of max(1e-2, 2e-4 |score|): at this blank gain a row emits a
    about 90 low-confidence tokens, and the fp16 operands' error in each log-probability adds up along the path with one
    sign (1.25e-4 of the score measured on row 0, -259.54 against -259.57)"""
    O = TO.Oracle(W)
    for b in rows:
        n = int(r["n_tokens"][b])
        toks, frs = r["tokens"][b, :n].tolist(), r["frames"][b, :n].tolist()
        o = O.row(tn[b], GO.BLANK, GO.MAX_SYMBOLS, forced=(toks, frs))
        assert o["tokens"] == toks, f"row {b}: the forced walk did not follow the device path"
        for (t, tok, lp, am, top1, top2) in o["decisions"]:
            if tok != am:
                assert top1 - top2 < GT.MARGIN, f"row {b} frame {t}: device {tok}, oracle arg-max {am}, margin {top1 - top2}"
        tol = max(GT.SCORE_TOL, 2e-4 * abs(o["score"]))
        print(f"MEASURE gigaspeech greedy row {b}: {n} tokens, score {float(r['logp_sum'][b]):.4f} vs oracle "
              f"{o['score']:.4f} (bound {tol:.3e})")
        assert abs(float(r["logp_sum"][b]) - o["score"]) <= tol, (b, float(r["logp_sum"][b]), o["score"])


def _searcher(c, beam):
    """the recipe's searcher on the model's prediction network and classifier (GT.build's modules, reloaded)"""
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    g, _, mods = GT.build(GO.J, GO.H, GO.V, GO.BLANK, GO.PN_SEED)
    for prefix, m in mods.items():
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in c["W"].items() if k.startswith(prefix + ".")})
    if beam == 1:
        return g, c["W"]
    return TransducerBeamSearcher(list(g.decode_network_lst), g.tjoint, list(g.classifier_network), blank_id=GO.BLANK,
                                  beam_size=beam, nbest=1, state_beam=GO.STATE_BEAM, expand_beam=GO.EXPAND_BEAM), c["W"]


# ------------------------------------------------------------------------------------------------ against the reference
_ASR = {}


def _fixture():
    fx = torch.load(os.path.join(GO.GOLDEN, "gigaspeech.pt"))
    assert fx["spm_checksum"] == sum(GO.sp_model().serialized_model_proto())
    return fx


def _streaming_asr():
    if not _ASR:
        _ASR["v"] = GO.streaming_asr()
    return _ASR["v"]


@pytest.mark.parametrize("name", ["32_4", "16_8", "8_2"])
def test_streaming_asr_against_the_reference(name):
    """test_gpu_streaming_asr.test_against_the_reference on this model: front end (norms within 2e-3 of the reference's,
    bit-identical to the offline front end), proj_enc (1e-3 against the reference's norms and the oracle), decisions up
    to the first near-tie then accepted by the oracle walk, and the strings"""
    import streaming_asr_oracle as SO
    import test_gpu_streaming_asr as SA
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    g = _fixture()["streaming"][name]
    asr, m, sd, w_enc, W, wav = _streaming_asr()
    fea = asr.hparams.fea_streaming_extractor
    chunk, left = g["chunk"], g["left"]
    assert (fea.get_required_padding(), fea.properties.window_size, fea.properties.stride) == (g["pad"], g["window_size"],
                                                                                                 g["stride"])
    cfg = DynChunkTrainConfig(chunk, left)
    assert asr.get_chunk_size_frames(cfg) == g["chunk_samples"]
    res, _ = SA._stream(asr, wav, cfg)
    assert len(res) == len(g["tokens"])
    trim = fea.get_output_count_per_pad_frame()
    worst_fe = 0.0
    for k, win in enumerate(SO.windows(wav, chunk)):
        got = res[k][0]
        off = fea.cnn(fea.normalize(fea.fbank(win.cuda())))
        off = off.reshape(off.shape[0], off.shape[1], -1)[:, trim:off.shape[1] - trim].cpu()
        assert torch.equal(got, off), f"chunk {k}: differs from the offline front end"
        worst_fe = max(worst_fe, rel(got.norm(dim=-1), g["feat_norms"][k]))
    whole = range(1, len(res) - 1)
    worst_tn = max(rel(res[k][1].norm(dim=-1), g["tn_norms"][k]) for k in whole)
    o = SO.run(wav, sd, GO.config(), w_enc, W, chunk, left, GO.sp_model())
    worst_or = max(rel(res[k][1], o[k][1]) for k in whole)
    print(f"MEASURE gigaspeech stream asr {name}: {len(res)} chunks; front end norms vs reference {worst_fe:.2e}; "
          f"proj_enc norms vs reference {worst_tn:.2e}, vs oracle {worst_or:.2e}")
    assert worst_fe < 2e-3 and worst_tn < 1e-3 and worst_or < 1e-3
    B = wav.shape[0]
    tn = torch.cat([r[1] for r in res], dim=1)
    T = tn.shape[1]
    toks = [sum((r[2][b] for r in res), []) for b in range(B)]
    r = GT.run_device(asr.hparams.decoding_function.args[0], tn.cuda(), SO.MAX_SYMBOLS)
    assert toks == [r["tokens"][b, :int(r["n_tokens"][b])].tolist() for b in range(B)]
    offsets = [sum(x[1].shape[1] for x in res[:k]) for k in range(len(res))]
    for b in range(B):
        ref = [(int(t) + offsets[k], int(tok)) for k in range(len(res)) for t, tok in g["decisions"][k][b].tolist()]
        margins = [mg for k in range(len(res)) for mg in g["margins"][k][b].tolist()]
        cut = next((i for i, mg in enumerate(margins) if mg < GT.MARGIN), len(ref))
        got = GT.device_decisions(r, b, T, SO.MAX_SYMBOLS)
        assert got[:cut] == ref[:cut], f"row {b}: differs from the reference before its first near-tie (decision {cut})"
        for k in range(len(res)):
            if all(res[j][2][b] == g["tokens"][j][b] for j in range(k + 1)):
                assert res[k][3][b] == g["words"][k][b], (b, k)
        if cut == len(ref):
            assert "".join(x[3][b] for x in res) == "".join(w[b] for w in g["words"])
    _check_rows(W, tn, r, range(B))


def test_streaming_asr_reruns_and_batch():
    import test_gpu_streaming_asr as SA
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    asr, _, _, _, _, wav = _streaming_asr()
    cfg = DynChunkTrainConfig(16, 8)
    wav4 = torch.cat([wav, wav[:1].flip(1)], dim=0)
    a, _ = SA._stream(asr, wav4, cfg)
    b, _ = SA._stream(asr, wav4, cfg)
    for x, y in zip(a, b):
        assert torch.equal(x[0], y[0]) and torch.equal(x[1], y[1]) and x[2] == y[2] and x[3] == y[3]
    alone, _ = SA._stream(asr, wav4[3:4], cfg)
    for x, y in zip(a, alone):
        assert torch.equal(x[1][3:4], y[1]) and x[2][3] == y[2][0]


def test_offline_against_the_reference_and_from_hparams(tmp_path):
    """the encoder and proj_enc per-frame norms against the reference's (1e-3), the Dynamic Chunk encode's, and the greedy
    decisions up to the first near-tie; EncoderDecoderASR.from_hparams on the recipe-layout directory (beam 10) transcribes
    like the same modules constructed directly"""
    from parity import normalizer_ckpt, write_pretrained_dir
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.inference.ASR import EncoderDecoderASR
    from speechbrain_b200.lobes.models.transformer.TransformerASR import EncoderWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.utils.dynamic_chunk_training import DynChunkTrainConfig
    g = _fixture()["offline"]
    sd, w_enc, W = GO.weights()
    wav, lens = GO.waveforms()
    m = GO.modules(sd, w_enc, W)
    enc_mod = LengthsCapableSequential(m["fb"], m["norm"], m["CNN"], EncoderWrapper(m["Transformer"]), m["proj_enc"])
    with torch.no_grad():
        src = LengthsCapableSequential(m["fb"], m["norm"], m["CNN"])(wav.cuda(), lens.cuda())
        enc = m["Transformer"].encode(src, lens.cuda())
        enc_dc = m["Transformer"].encode(src, lens.cuda(), dynchunktrain_config=DynChunkTrainConfig(*g["dynchunk"]))
        tn = m["proj_enc"](enc)
    r_enc, r_dc, r_tn = (rel(x.norm(dim=-1).cpu(), y) for x, y in ((enc, g["enc_norms"]), (enc_dc, g["dynchunk_enc_norms"]),
                                                                    (tn, g["tn_norms"])))
    print(f"MEASURE gigaspeech offline vs reference norms: encoder {r_enc:.2e}, dynchunk {r_dc:.2e}, proj_enc {r_tn:.2e}")
    assert max(r_enc, r_dc, r_tn) < ENC_BAR
    r = GT.run_device(m["searcher"], tn.contiguous(), GO.MAX_SYMBOLS)
    for b in range(tn.shape[0]):
        ref = [tuple(x) for x in g["decisions"][b].tolist()]
        cut = next((i for i, mg in enumerate(g["margins"][b].tolist()) if mg < GT.MARGIN), len(ref))
        assert GT.device_decisions(r, b, tn.shape[1], GO.MAX_SYMBOLS)[:cut] == ref[:cut], b
    beam = TransducerBeamSearcher([m["emb"], m["dec"], m["proj_dec"]], m["searcher"].tjoint, [m["transducer_lin"]],
                                  blank_id=GO.BLANK, beam_size=GO.BEAM, nbest=1, state_beam=GO.STATE_BEAM,
                                  expand_beam=GO.EXPAND_BEAM)
    if g["beam"]["min_margin"] >= GT.MARGIN:  # otherwise the replay of test_transducer_greedy_and_beam covers it
        rb = BT.run_device(beam, tn.contiguous())
        assert [BT.device_nbest(rb, b)[0] for b in range(tn.shape[0])] == [t[0] for t in g["beam"]["tokens"]]
    tmp = write_pretrained_dir(tmp_path, GO.HPARAMS, dict(asr=GO.asr_ckpt(m), normalizer=normalizer_ckpt(sd)))
    loaded = EncoderDecoderASR.from_hparams(source=tmp, run_opts={"device": "cuda:0"})
    direct = EncoderDecoderASR(modules={"encoder": enc_mod, "decoder": beam},
                               hparams={"tokenizer": None, "transducer_beam_search": True}, run_opts={"device": "cuda:0"})
    w1, t1 = loaded.transcribe_batch(wav.cuda(), lens.cuda())
    w2, t2 = direct.transcribe_batch(wav.cuda(), lens.cuda())
    assert t1 == t2 and w1 == w2 and sum(len(t) for t in t1) > 0
