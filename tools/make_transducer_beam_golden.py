"""Generate tests/golden/transducer_beam.pt by RUNNING THE REFERENCE TransducerBeamSearcher(beam_size > 1)
(speechbrain.decoders.transducer.transducer_beam_search_decode, no language model) on the seeded recipe-shaped prediction
networks of tests/transducer_oracle.py.

How to run it: oracle/goldens.py.  Weights and tn_output are regenerated from seeds (seeded_weights / seeded_tn); the
fixture stores the case parameters, a checksum of tn_output and the outputs only.  Per case: the reference's n-best tokens
and normalised scores per utterance, its number of pops (prediction-network + joint evaluations), and the smallest margin
of every kind of comparison the search made (key max, top-K boundary, expand_beam, state_beam, final sort), taken from the
fp32 oracle (tests/transducer_beam_oracle.py) after asserting that the oracle returns the reference's n-best tokens and
scores within 1e-5.

The "e2e" case is the LibriSpeech transducer model of tests/golden/transducer.pt (make_transducer_golden.e2e_inputs(),
4 x 10 s ragged) searched with beam 10, nbest 1."""
import collections

import torch

import make_transducer_golden as MG
from oracle import goldens as G  # also puts tests/, where the oracles live, on sys.path

import transducer_beam_oracle as BO  # noqa: E402
import transducer_oracle as TO  # noqa: E402

SB, EB = 2.3, 2.3


def case_list():
    return [
        dict(name="librispeech", recipe="librispeech", blank="first", B=4, T=251, seed=31, beam=10, nbest=1, sb=SB, eb=EB),
        dict(name="voxpopuli_last", recipe="voxpopuli", blank="last", B=3, T=120, seed=32, beam=10, nbest=1, sb=SB, eb=EB),
        dict(name="commonvoice_nbest", recipe="commonvoice", blank="first", B=3, T=120, seed=33, beam=4, nbest=4, sb=1.0,
             eb=4.0),
        dict(name="t1", recipe="librispeech", blank="first", B=2, T=1, seed=34, beam=10, nbest=1, sb=SB, eb=EB),
        dict(name="t17", recipe="voxpopuli", blank="first", B=3, T=17, seed=35, beam=10, nbest=2, sb=SB, eb=EB),
        # short searches whose every comparison is at least 2e-3 from flipping: the device must give their tokens exactly
        dict(name="wide_librispeech", recipe="librispeech", blank="first", B=2, T=4, seed=48, beam=10, nbest=1, sb=SB,
             eb=EB),
        dict(name="wide_voxpopuli", recipe="voxpopuli", blank="last", B=2, T=3, seed=41, beam=4, nbest=2, sb=SB, eb=EB),
    ]


def case_inputs(case):
    """(weights, tn_output, blank) of a case, regenerated"""
    J, H, V = TO.RECIPE_SIZES[case["recipe"]]
    blank = 0 if case["blank"] == "first" else V - 1
    W = TO.seeded_weights(case["seed"], J, H, V, blank)
    tn = TO.seeded_tn(case["seed"] + 1000, case["B"], case["T"], W)
    return W, tn, blank


def run_reference(W, tn, blank, beam, nbest, sb, eb):
    """the reference beam search: (its return value, pops per utterance)"""
    s, _ = MG.reference_searcher(W, blank)
    s.beam_size, s.nbest, s.state_beam, s.expand_beam = beam, nbest, sb, eb
    s.searcher = s.transducer_beam_search_decode
    pops = collections.Counter()
    orig = s._joint_forward_step

    def rec(h_i, out_PN):
        pops[h_i.storage_offset() // (tn.shape[1] * tn.shape[2])] += 1
        return orig(h_i, out_PN)
    s._joint_forward_step = rec
    with torch.no_grad():
        out = s.transducer_beam_search_decode(tn)
    return out, [pops[b] for b in range(tn.shape[0])]


def check_and_record(W, tn, blank, case):
    (best, score, nb, nbs), pops = run_reference(W, tn, blank, case["beam"], case["nbest"], case["sb"], case["eb"])
    o_best, o_score, o_nb, o_nbs, rows = BO.BeamOracle(W).batch(tn, blank, case["beam"], case["nbest"], case["sb"],
                                                                  case["eb"])
    assert o_nb == nb, case["name"]
    for a, b in zip(o_nbs, nbs):
        assert len(a) == len(b) and all(abs(x - float(y)) <= 1e-5 for x, y in zip(a, b)), (case["name"], a, b)
    assert [r["pops"] for r in rows] == pops, (case["name"], pops)
    margins = {k: min(r["margins"][k] for r in rows) for k in BO.KINDS}
    max_pf = max(r["max_pops_per_frame"] for r in rows)
    print(case["name"], "lens", [len(h) for h in best], "pops", pops, "max pops/frame", max_pf, "margins",
          {k: f"{v:.2e}" for k, v in margins.items()})
    return dict(tokens=nb, scores=[[float(x) for x in s] for s in nbs], score=float(score), pops=pops,
                max_pops_per_frame=max_pf, margins=margins, min_margin=min(margins.values()))


def e2e_case():
    cfg, sd, w_enc, W, wav, lens = MG.e2e_inputs()
    tn = e2e_tn(cfg, sd, w_enc, wav, lens)
    case = dict(name="e2e", beam=10, nbest=1, sb=SB, eb=EB)
    return dict(case, wav_checksum=float(wav.double().abs().sum()), tn_checksum=float(tn.double().abs().sum()),
                **check_and_record(W, tn, 0, case))


def e2e_tn(cfg, sd, w_enc, wav, lens):
    """the reference tn_output of the e2e model (the encoder of make_transducer_golden.e2e_case)"""
    from speechbrain.lobes.features import Fbank
    from speechbrain.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain.processing.features import InputNormalization
    fb = Fbank(n_fft=512, n_mels=80, win_length=32)
    norm = InputNormalization(norm_type="global")
    norm.glob_mean, norm.glob_std, norm.count = sd["normalize.glob_mean"], sd["normalize.glob_std"], 1
    norm.eval()
    cnn = ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1, out_channels=(64, 32),
                              kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
    cnn.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("CNN.")})
    cnn.eval()
    tr = TransformerASR(input_size=640, tgt_vocab=1000, d_model=512, nhead=8, num_encoder_layers=12, num_decoder_layers=0,
                        d_ffn=2048, dropout=0.1, activation=torch.nn.GELU, encoder_module="conformer",
                        attention_type="RoPEMHA", normalize_before=True, causal=False)
    tr.load_state_dict({k[len("Transformer."):]: v for k, v in sd.items() if k.startswith("Transformer.")}, strict=False)
    tr.eval()
    with torch.no_grad():
        enc = tr.encode(cnn(norm(fb(wav), lens)), lens)
        return (enc @ w_enc.T).contiguous()


def main():
    torch.set_num_threads(8)
    out = {"cases": []}
    for case in case_list():
        W, tn, blank = case_inputs(case)
        out["cases"].append(dict(case, checksum=float(tn.double().abs().sum()), **check_and_record(W, tn, blank, case)))
    out["e2e"] = e2e_case()
    G.save(out, "transducer_beam.pt")


if __name__ == "__main__":
    main()
