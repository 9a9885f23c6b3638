"""The fixture writers' shared pieces: oracle/make_goldens.py and tools/make_*_golden.py run the reference and write
tests/golden/*.pt with these.

Running the writers
-------------------
Every writer imports the reference package, whose speechbrain/core.py needs two names from HyperPyYAML;
baseline/stubs/hyperpyyaml.py stands in for it.  From the repository root, with <reference> the reference checkout:

    PYTHONPATH=baseline/stubs:<reference>:. python oracle/make_goldens.py [case ...]
    PYTHONPATH=baseline/stubs:<reference>:. python tools/make_<name>_golden.py

make_goldens.py without arguments writes fbank, norm, L_rope, L_relpos, S_relpos, beam, beam_topk, beam_lm, beam_ctc,
rescore and beam_len.  The other cases take minutes of CPU each and run only when named: bench_L_rope, bench_L_relpos,
bench_S_relpos, bench_extra, dynchunk, beam_cov, beam66, scaled and ctc_greedy.  Some cases start from a fixture that is
already committed: the beam cases, dynchunk, scaled and ctc_greedy read conformer_large_*.pt, bench_extra reads
bench_conformer_large_rope_10s.pt, and the CTC beam writers read branchformer.pt.  Each writer asserts that its oracle
equals the reference before it writes anything.

Importing this module or a writer does not import the reference (tests import the writers' case lists); every function
that needs it imports it when called.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
if os.path.join(ROOT, "tests") not in sys.path:  # the writers check the reference against the oracles under tests/
    sys.path.append(os.path.join(ROOT, "tests"))

BOS, EOS = 1, 2
LM_TEMPERATURE = 1.15
CFG_LM = dict(d_model=768, nhead=12, num_encoder_layers=12, d_ffn=3072, activation="gelu")


def rel(a, b):
    """rel-L2 of a against b, in float64"""
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def load(name):
    return torch.load(os.path.join(GOLDEN, name))


def save(obj, name):
    path = os.path.join(GOLDEN, name)
    torch.save(obj, path)
    print(path, os.path.getsize(path))


def seeded_wav(seed, shape, lens=None, checksum=None):
    """A fixture's waveform, generated from its seed: [B, L] normal samples, row b zeroed past round(lens[b] L) (lens None:
    all ones); the checksum (sum of |x|) pins the RNG stream"""
    B, L = shape
    wav = torch.randn(B, L, generator=torch.Generator().manual_seed(seed))
    lens = torch.ones(B) if lens is None else lens
    for b in range(B):
        wav[b, int(round(float(lens[b]) * L)):] = 0
    if checksum is not None:
        assert abs(float(wav.double().abs().sum()) - checksum) / checksum < 1e-9, "regenerated waveform differs from the fixture's"
    return wav, lens


def wav_case(seed, B, L, lens):
    """seeded_wav for the Python float lengths lens: (wav, wav_lens, the fixture record of both)"""
    wav, _ = seeded_wav(seed, (B, L), lens)
    wav_lens = torch.tensor(lens)
    return wav, wav_lens, dict(wav_seed=seed, wav_shape=(B, L), wav_lens=wav_lens, wav_checksum=float(wav.double().abs().sum()))


class Reference:
    """The reference's Fbank, global CMVN, CNN front end, TransformerASR, seq_lin (when the recipe decodes) and ctc_lin on
    seeded weights (seed 0); sd is the flat state with the CMVN statistics, cfg the oracle's config"""

    def __init__(self, fb, norm, mods, sd, cfg):
        self.fb, self.norm, self.mods, self.sd, self.cfg = fb, norm, mods, sd, cfg

    @torch.no_grad()
    def cnn(self, wav, wav_lens):
        return self.mods["CNN"](self.norm(self.fb(wav), wav_lens))

    @torch.no_grad()
    def encode(self, wav, wav_lens):
        return self.mods["Transformer"].encode(self.cnn(wav, wav_lens), wav_lens)

    def keys(self, name="Transformer"):
        """the state_dict key -> shape list of one module"""
        return [(k, tuple(v.shape)) for k, v in self.mods[name].state_dict().items()]


def build_reference(cfg, attention_type=None, cnn_blocks=2, transform=None, **transformer_kw):
    """Reference of a recipe config (win_length in ms, or win in samples at sample_rate).  cnn_blocks: the 2-block
    conformer front end or the 3-block transformer one; transformer_kw: TransformerASR keywords besides the sizes
    (encoder_module, activations, positional_encoding, Branchformer sizes); transform(sd): rescales the seeded weights
    before they are loaded.  seq_lin exists when the config has decoder layers."""
    import speechbrain  # noqa: F401
    from speechbrain.lobes.features import Fbank
    from speechbrain.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain.nnet.linear import Linear
    from speechbrain.processing.features import InputNormalization

    from speechbrain_b200.utils.seeded_init import seeded_state_dict, seeded_tensor
    win = cfg["win_length"] if "win_length" in cfg else cfg["win"] * 1000 // cfg["sample_rate"]
    fb = Fbank(n_fft=cfg["n_fft"], n_mels=cfg["n_mels"], win_length=win)
    norm = InputNormalization(norm_type="global", update_until_epoch=4)
    if cnn_blocks == 2:
        cnn = ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1,
                                  out_channels=cfg["cnn_channels"], kernel_sizes=(3, 3), strides=(2, 2),
                                  residuals=(False, False))
    else:
        cnn = ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=3, num_layers_per_block=1, out_channels=(64, 64, 64),
                                  kernel_sizes=(5, 5, 1), strides=(2, 2, 1), residuals=(False, False, True))
    attention_type = attention_type or cfg["attention_type"]
    transformer_kw = dict(dict(activation=torch.nn.GELU, encoder_module="conformer"), **transformer_kw)
    tr = TransformerASR(input_size=cfg["input_size"], tgt_vocab=cfg["vocab"], d_model=cfg["d_model"], nhead=cfg["nhead"],
                        num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=cfg["num_decoder_layers"],
                        d_ffn=cfg["d_ffn"], dropout=0.1, attention_type=attention_type, normalize_before=True, causal=False,
                        **transformer_kw)
    mods = dict(CNN=cnn, Transformer=tr, ctc_lin=Linear(input_size=cfg["d_model"], n_neurons=cfg["vocab"]))
    if cfg["num_decoder_layers"] > 0:
        mods["seq_lin"] = Linear(input_size=cfg["d_model"], n_neurons=cfg["vocab"])
    mods = torch.nn.ModuleDict(mods)
    sd = seeded_state_dict(mods, seed=0)
    if transform is not None:
        sd = transform(sd)
    mods.load_state_dict(sd)
    mods.eval()
    norm.glob_mean = seeded_tensor(0, "normalize.glob_mean", (cfg["n_mels"],)) * 3.0 - 20.0
    norm.glob_std = seeded_tensor(0, "normalize.glob_std", (cfg["n_mels"],)) * 8.0
    norm.count = 1
    norm.eval()
    sd["normalize.glob_mean"], sd["normalize.glob_std"] = norm.glob_mean, norm.glob_std
    return Reference(fb, norm, mods, sd, dict(cfg, attention_type=attention_type, win_length=win))


def frame_summary(x, abs_len, head, near=(-2, -1, 0, 1), tail=(2, 1), norm_key="frame_norm"):
    """x [B, T, ...] as the fixtures keep it: the L2 norm of every frame, and the full rows of sampled frames (b, t): the
    first ones (head), the middle one, abs_len[b] + near around each valid length and T - tail at the end"""
    B, T = x.shape[:2]
    x = x.reshape(B, T, -1)
    idx = set()
    for b in range(B):
        n = int(abs_len[b])
        ts = tuple(head) + (T // 2,) + tuple(n + d for d in near) + tuple(T - d for d in tail)
        idx |= {(b, t) for t in ts if 0 <= t < T}
    sample_idx = torch.tensor(sorted(idx), dtype=torch.long)
    return {norm_key: x.double().norm(dim=-1).float(), "sample_idx": sample_idx.to(torch.int32),
            "sample_rows": x[sample_idx[:, 0], sample_idx[:, 1]].clone()}


@torch.no_grad()
def reference_greedy(ref, enc, wav_lens, max_decode_ratio):
    """the token lists of the reference's S2STransformerGreedySearcher"""
    from speechbrain.decoders.seq2seq import S2STransformerGreedySearcher
    gs = S2STransformerGreedySearcher(modules=[ref.mods["Transformer"], ref.mods["seq_lin"]], bos_index=BOS, eos_index=EOS,
                                      min_decode_ratio=0.0, max_decode_ratio=max_decode_ratio)
    return gs(enc, wav_lens)[0]


@torch.no_grad()
def greedy_case(ref, enc, wav_lens, n_steps, tag):
    """n_steps greedy steps of the reference and of the oracle, asserted equal: (hyps, the oracle's logits [B, S, V])"""
    from oracle import asr_oracle as O
    ratio = (n_steps + 0.5) / enc.shape[1]
    hyps = reference_greedy(ref, enc, wav_lens, ratio)
    ohyps, _, _, _, ologits = O.greedy_search(enc, wav_lens, ref.sd, ref.cfg, ref.sd["seq_lin.w.weight"],
                                              ref.sd["seq_lin.w.bias"], BOS, EOS, 0.0, ratio, "Transformer.",
                                              return_logits=True)
    assert ohyps == hyps, "oracle greedy != reference greedy"
    print(f"[{tag}] greedy {ologits.shape[1]} steps, oracle equal")
    return hyps, ologits


def greedy_record(hyps, logits, lp=None, chosen_lp=True):
    """a fixture's greedy entries: token lists, arg-max tokens, top-1 / top-2 logit margins and (chosen_lp) the log-prob of
    each chosen token (lp: the log-probs, default log_softmax(logits))"""
    top2 = logits.topk(2, dim=-1).values
    tok = logits.argmax(-1)
    out = dict(greedy_hyps=hyps, greedy_tokens=tok.int(), greedy_margin=(top2[..., 0] - top2[..., 1]).clone())
    if chosen_lp:
        lp = torch.log_softmax(logits, -1) if lp is None else lp
        out["greedy_chosen_lp"] = lp.gather(-1, tok.unsqueeze(-1)).squeeze(-1).clone()
    print(f"   greedy min top1-top2 margin {float(out['greedy_margin'].min()):.4f}")
    return out


def reference_lm(vocab=5000):
    """the recipes' 12 x 768 TransformerLM of the reference on seeded weights (seed 1): (module, state dict)"""
    from speechbrain.lobes.models.transformer.TransformerLM import TransformerLM

    from speechbrain_b200.utils.seeded_init import seeded_state_dict
    lm = TransformerLM(vocab=vocab, d_model=768, nhead=12, num_encoder_layers=12, num_decoder_layers=0, d_ffn=3072,
                       dropout=0.0, activation=torch.nn.GELU, normalize_before=False)
    sd_lm = seeded_state_dict(lm, seed=1)
    lm.load_state_dict(sd_lm)
    lm.eval()
    return lm, sd_lm


@torch.no_grad()
def run_beam(ref, enc, wav_lens, kwargs, max_decode_ratio, eos_bias=0.0, scorers=None, lm=None, coverage_threshold=None,
             topk=None, bar=1e-4, rank0=False, check=True, tag="beam"):
    """One S2STransformerBeamSearcher case: seq_lin's EOS bias raised by eos_bias (random weights rarely end a
    hypothesis otherwise), the searcher built with kwargs and, when topk, return_topk=True.  scorers: an ordered
    {name: weight} of full scorers ("transformerlm" with lm = reference_lm(), "ctc", "length", "coverage" with
    coverage_threshold), built in that order.  With check, the oracle runs the same search and must return the same
    hypotheses (all of them, or with rank0 the best one per utterance) and scores within bar.  seq_lin's bias is restored
    afterwards; returns the reference's (hyps, lens, scores, log_probs)."""
    from speechbrain.decoders.scorer import CoverageScorer, CTCScorer, LengthScorer, ScorerBuilder, TransformerLMScorer
    from speechbrain.decoders.seq2seq import S2STransformerBeamSearcher

    from oracle import asr_oracle as O
    sd, vocab = ref.sd, ref.cfg["vocab"]
    full, okw = [], {}
    for name, w in (scorers or {}).items():
        if name == "transformerlm":
            full.append(TransformerLMScorer(language_model=lm[0], temperature=LM_TEMPERATURE))
            okw["lm"] = dict(sd=lm[1], cfg=CFG_LM, weight=w, temperature=LM_TEMPERATURE)
        elif name == "ctc":
            full.append(CTCScorer(eos_index=EOS, blank_index=0, ctc_fc=ref.mods["ctc_lin"]))
            okw["ctc"] = dict(w=sd["ctc_lin.w.weight"], b=sd["ctc_lin.w.bias"], weight=w, blank_index=0)
        elif name == "length":
            full.append(LengthScorer(vocab))
            okw["length_weight"] = w
        else:
            full.append(CoverageScorer(vocab, threshold=coverage_threshold))
            okw["coverage"] = dict(weight=w, threshold=coverage_threshold)
    scorer = ScorerBuilder(full_scorers=full, weights=dict(scorers)) if scorers else None
    if topk:
        okw.update(topk=topk, return_topk=True)
    bias = sd["seq_lin.w.bias"].clone()
    bias[EOS] += eos_bias
    ref.mods["seq_lin"].w.bias.copy_(bias)
    bs = S2STransformerBeamSearcher(modules=[ref.mods["Transformer"], ref.mods["seq_lin"]], bos_index=BOS, eos_index=EOS,
                                    max_decode_ratio=max_decode_ratio, scorer=scorer,
                                    **(dict(return_topk=True, topk=topk) if topk else {}), **kwargs)
    out = bs(enc, wav_lens)
    if check:
        o = O.beam_search(enc, wav_lens, sd, ref.cfg, sd["seq_lin.w.weight"], bias, BOS, EOS,
                          max_decode_ratio=max_decode_ratio, prefix="Transformer.", **okw, **kwargs)
        if rank0:
            same = torch.equal(o[0][:, 0], out[0][:, 0])
        elif topk:
            same = torch.equal(o[0], out[0]) and torch.allclose(o[1], out[1])
        else:
            same = o[0] == out[0]
        err = float((o[2] - out[2]).abs().max())
        print(f"[{tag}] reference scores {out[2].tolist()} | oracle hypotheses equal: {same}, score err {err:.2e} (bar {bar})")
        assert same and err < bar, tag
    ref.mods["seq_lin"].w.bias.copy_(sd["seq_lin.w.bias"])
    return out
