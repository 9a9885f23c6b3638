"""Generate tests/golden/transducer.pt by RUNNING THE REFERENCE TransducerBeamSearcher(beam_size=1) (speechbrain.decoders.
transducer) with the reference Embedding / LSTM / Linear / Transducer_joint modules on seeded recipe-shaped weights.

How to run it: oracle/goldens.py.  The weights and tn_output of every case are regenerated from seeds (tests/transducer_oracle.seeded_weights / seeded_tn;
the fixture keeps the seeds, the weight rescale and a checksum).  Per case it stores the reference's tokens, its score
(exp of the summed log-probs, averaged over the batch) and, per joint evaluation, the top-two log-probs of every row
(the reference margins); for the streaming case the tokens of chunked calls and the final (out_PN, h, c) norms.  It
asserts that the oracle (tests/transducer_oracle.py) gives the same tokens and the score to 1e-6, and that the cases
have frames with 0, 1 and >= 2 emissions.

The "e2e" entry is the LibriSpeech transducer recipe model in the EncoderDecoderASR layout: the 12-layer RoPEMHA Conformer
(d_model 512, seeded_init.seeded_asr_state with E2E["seed"]), proj_enc 512 -> 640 (bias-free, seeded, scaled by
E2E["enc_scale"]) and the 640 / 512 / 1000 prediction network and classifier (seeded_weights with E2E["blank_gain"]),
run by the reference on a 4 x 10 s ragged batch [1.0, 0.9, 0.6, 0.3] (waveforms from a seed, checksummed).  It stores
the per-frame norms of the reference tn_output (padded frames included), the tokens, the score, and every row's
decisions (frame, token, top-1 / top-2 log-prob margin) as the reference took them.  The blank gain is the rescale that
makes this search emit 0, 1 and >= 2 tokens per frame (asserted)."""
import collections

import torch

from oracle import goldens as G  # also puts tests/, where the oracles live, on sys.path

import transducer_oracle as TO  # noqa: E402


def case_list():
    cases = []
    for recipe in ("librispeech", "commonvoice", "voxpopuli"):
        for blank in ("first", "last"):
            cases.append(dict(name=f"{recipe}_{blank}", recipe=recipe, blank=blank, m=5, B=4, T=120, seed=11))
    cases += [
        dict(name="m0", recipe="voxpopuli", blank="first", m=0, B=3, T=120, seed=12),
        dict(name="m1", recipe="voxpopuli", blank="last", m=1, B=3, T=120, seed=13),
        dict(name="t1", recipe="librispeech", blank="first", m=5, B=3, T=1, seed=14),
        dict(name="cap", recipe="voxpopuli", blank="first", m=2, B=2, T=20, seed=15, suppress_blank=True),
        dict(name="stream", recipe="librispeech", blank="first", m=5, B=3, T=100, seed=16, chunk=16),
    ]
    return cases


def case_inputs(case):
    """(weights, tn_output) of a case, regenerated."""
    J, H, V = TO.RECIPE_SIZES[case["recipe"]]
    blank = 0 if case["blank"] == "first" else V - 1
    W = TO.seeded_weights(case["seed"], J, H, V, blank)
    tn = TO.seeded_tn(case["seed"] + 1000, case["B"], case["T"], W)
    if case.get("suppress_blank"):
        W["transducer_lin.w.weight"][blank] = -50.0 / J ** 0.5
        tn = tn.abs()
    return W, tn, blank


def reference_searcher(W, blank):
    import speechbrain as sb
    from speechbrain.decoders.transducer import TransducerBeamSearcher
    from speechbrain.nnet.transducer.transducer_joint import Transducer_joint
    V, J = W["transducer_lin.w.weight"].shape
    H = W["dec.rnn.weight_hh_l0"].shape[1]
    emb = sb.nnet.embedding.Embedding(num_embeddings=V, consider_as_one_hot=True, blank_id=blank)
    dec = sb.nnet.RNN.LSTM(input_shape=[None, None, V - 1], hidden_size=H, num_layers=1)
    proj = sb.nnet.linear.Linear(input_size=H, n_neurons=J, bias=False)
    lin = sb.nnet.linear.Linear(input_size=J, n_neurons=V, bias=False)
    for prefix, m in (("emb", emb), ("dec", dec), ("proj_dec", proj), ("transducer_lin", lin)):
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in W.items() if k.startswith(prefix + ".")})
        m.eval()
    s = TransducerBeamSearcher([emb, dec, proj], Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU), [lin],
                               blank_id=blank, beam_size=1, nbest=1)
    keys = {p: sorted(m.state_dict()) for p, m in (("emb", emb), ("dec", dec), ("proj_dec", proj),
                                                   ("transducer_lin", lin))}
    return s, keys


E2E = dict(seed=21, pn_seed=23, wav_seed=22, lens=[1.0, 0.9, 0.6, 0.3], L=160000, enc_scale=1.0, blank_gain=1.0, m=5)


def e2e_inputs():
    """(encoder state dict, proj_enc weight, prediction-network weights, wav, lens) of the end-to-end case."""
    from speechbrain_b200.utils.seeded_init import CONFORMER_LARGE, seeded_asr_state, seeded_tensor
    cfg = dict(CONFORMER_LARGE, num_decoder_layers=0, vocab=1000)
    sd = seeded_asr_state(cfg, E2E["seed"])
    w_enc = seeded_tensor(E2E["seed"], "proj_enc.w.weight", (640, 512)) * E2E["enc_scale"]
    W = TO.seeded_weights(E2E["pn_seed"], 640, 512, 1000, 0, blank_gain=E2E["blank_gain"])
    wav, lens, _ = G.wav_case(E2E["wav_seed"], len(E2E["lens"]), E2E["L"], E2E["lens"])
    return cfg, sd, w_enc, W, wav, lens


def row_decisions(calls, B, blank, m):
    """Per row, the decisions the reference took, from its recorded joint calls [(frame, top-2 values [B, 2], arg-max [B])]:
    in every frame a row's decisions are the calls up to its first blank (its later calls repeat that blank)."""
    out = []
    for b in range(B):
        dec, t_done = [], -1
        for t, top2, am in calls:
            if t == t_done:
                continue
            tok = int(am[b])
            dec.append((t, tok, float(top2[b, 0] - top2[b, 1])))
            if tok == blank:
                t_done = t
        out.append(torch.tensor([[d[0], d[1]] for d in dec], dtype=torch.int32))
        out[-1] = (out[-1], torch.tensor([d[2] for d in dec], dtype=torch.float32))
    return out


def e2e_case():
    from speechbrain.lobes.features import Fbank
    from speechbrain.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain.processing.features import InputNormalization
    cfg, sd, w_enc, W, wav, lens = e2e_inputs()
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
    s, _ = reference_searcher(W, 0)
    calls = []
    orig = s._joint_forward_step

    def rec(h_i, out_PN):
        lp = orig(h_i, out_PN)
        flat = lp.squeeze(1).squeeze(1)
        calls.append((h_i.storage_offset() // h_i.shape[-1], flat.topk(2, dim=-1).values.clone(), flat.argmax(-1).clone()))
        return lp
    s._joint_forward_step = rec
    with torch.no_grad():
        enc = tr.encode(cnn(norm(fb(wav), lens)), lens)
        tn = (enc @ w_enc.T).contiguous()
        hyps, score, _, _ = s.transducer_greedy_decode(tn, max_symbols_per_step=E2E["m"])
    # frames = tn_output[:, t] views: storage offset t * J
    assert [c[0] for c in calls] == sorted(c[0] for c in calls) and calls[-1][0] == tn.shape[1] - 1
    o_hyps, o_score, rows = TO.Oracle(W).batch(tn, 0, E2E["m"])
    assert o_hyps == hyps and abs(float(o_score) - float(score)) <= 1e-6 * max(1.0, abs(float(score)))
    hist = collections.Counter()
    for r in rows:
        c = collections.Counter(r["frames"])
        hist.update(min(c.get(t, 0), 2) for t in range(tn.shape[1]))
    assert all(hist[k] > 0 for k in (0, 1, 2)), hist
    dec = row_decisions(calls, tn.shape[0], 0, E2E["m"])
    for b, r in enumerate(rows):   # the per-row decisions replay the reference's tokens
        assert [int(t) for (f, t) in dec[b][0].tolist() if t != 0] == hyps[b]
    print("e2e tokens", [len(h) for h in hyps], "score", float(score), "frames by emissions", dict(hist))
    return dict(E2E, wav_checksum=float(wav.double().abs().sum()), tn_norms=tn.double().norm(dim=-1).float(),
                tokens=hyps, score=float(score), decisions=[d[0] for d in dec], margins=[d[1] for d in dec],
                emission_hist=dict(hist))


def main():
    torch.set_num_threads(8)
    out = {"cases": [], "keys": None}
    total = collections.Counter()
    for case in case_list():
        W, tn, blank = case_inputs(case)
        s, keys = reference_searcher(W, blank)
        out["keys"] = keys
        tops = []
        orig = s._joint_forward_step

        def rec(h_i, out_PN, orig=orig):
            lp = orig(h_i, out_PN)
            tops.append(lp.squeeze(1).squeeze(1).topk(2, dim=-1).values.clone())
            return lp
        s._joint_forward_step = rec
        entry = dict(case, checksum=float(tn.double().abs().sum()))
        with torch.no_grad():
            if "chunk" in case:
                from speechbrain.decoders.transducer import TransducerGreedySearcherStreamingContext
                ctx = TransducerGreedySearcherStreamingContext()
                hyps = [[] for _ in range(case["B"])]
                for t0 in range(0, case["T"], case["chunk"]):
                    for b, h in enumerate(s.transducer_greedy_decode_streaming(tn[:, t0:t0 + case["chunk"]], ctx)):
                        hyps[b] += h
                p, (h, c) = ctx.hidden
                entry["state_norms"] = [p.reshape(case["B"], -1).norm(dim=-1), h[0].norm(dim=-1), c[0].norm(dim=-1)]
                score = None
            else:
                hyps, score, _, _ = s.transducer_greedy_decode(tn, max_symbols_per_step=case["m"])
        entry["tokens"] = hyps
        entry["score"] = None if score is None else float(score)
        entry["top2"] = torch.stack(tops) if tops else torch.zeros(0)
        # the oracle equals the reference
        o_hyps, o_score, rows = TO.Oracle(W).batch(tn, blank, case["m"])
        assert o_hyps == hyps, case["name"]
        if score is not None:
            assert abs(float(o_score) - float(score)) <= 1e-6 * max(1.0, abs(float(score))), (case["name"], o_score, score)
        hist = collections.Counter()
        for r in rows:
            c = collections.Counter(r["frames"])
            hist.update(min(c.get(t, 0), 2) for t in range(case["T"]))
        entry["emission_hist"] = dict(hist)
        total.update(hist)
        if case.get("suppress_blank"):
            assert all(len(h) == (case["m"] + 1) * case["T"] for h in hyps)
        print(case["name"], "tokens", [len(h) for h in hyps], "score", entry["score"], "frames by emissions", dict(hist))
        out["cases"].append(entry)
    assert all(total[k] > 0 for k in (0, 1, 2)), total   # frames with 0, 1 and >= 2 emissions
    out["e2e"] = e2e_case()
    G.save(out, "transducer.pt")


if __name__ == "__main__":
    main()
