"""Generate tests/golden/gigaspeech.pt (and the SentencePiece model tests/golden/gigaspeech_spm.model) by RUNNING THE
REFERENCE modules of GigaSpeech's Conformer-Transducer, wired as recipes/GigaSpeech/ASR/transducer/hparams/
conformer_transducer.yaml's model and its commented inference block wire them: Fbank(n_fft 512, win 32 ms), global
InputNormalization, the 2-block (64, 32) ConvolutionFrontEnd, TransformerASR(d_model 768, 8 heads, 12 Conformer layers,
d_ffn 2048, RelPosMHAXL, num_decoder_layers 0) in an EncoderWrapper, proj_enc 768 -> 512 without bias, and a
TransducerBeamSearcher over Embedding(1024, one-hot) -> LSTM 512 -> proj_dec 512 and a GELU sum joint -> 1024 tokens.

How to run it: oracle/goldens.py.  Weights: tests/gigaspeech_oracle.weights (seeded; the blank gain there makes the greedy
search emit 0, 1 and >= 2 tokens on some frames, asserted here).

Offline, on the 4 x 10 s ragged batch [1.0, 0.9, 0.6, 0.3]: per-frame norms of the encoder states and of proj_enc; the greedy
tokens, decisions (frame, token) and top-1 / top-2 margins as the reference's joint calls took them; the beam-10 best
hypotheses and scores (state_beam = expand_beam = 2.3, nbest 1); one Dynamic Chunk encode at (16, 2) as per-frame norms.
Streaming: the reference StreamingASR chunk by chunk on the first 6 s of three rows at the recipe README's (32, 4), (16, 8)
and (8, 2), with what make_streaming_asr_golden.py records per chunk.  And the reference state_dict keys and shapes of
every module.

Before writing, it asserts that the CPU oracles equal the reference: the encoder (tests/gigaspeech_oracle.py), the greedy
search (tests/transducer_oracle.py), the beam search (tests/transducer_beam_oracle.py) and StreamingASR
(tests/streaming_asr_oracle.run)."""
import collections
import functools
import io
import os
import random

import torch

from oracle import goldens as G  # also puts tests/ on sys.path

import gigaspeech_oracle as GO  # noqa: E402
import make_transducer_beam_golden as MB  # noqa: E402  (tools/ is the script's directory)
import make_transducer_golden as MT  # noqa: E402
import streaming_asr_oracle as SO  # noqa: E402
import transducer_oracle as TO  # noqa: E402

CASES = {"32_4": (32, 4), "16_8": (16, 8), "8_2": (8, 2)}


def train_spm():
    import sentencepiece as spm
    if not os.path.exists(GO.SPM_MODEL):
        rng = random.Random(1)
        words = ["".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(2, 9))) for _ in range(4000)]
        lines = [" ".join(rng.choice(words) for _ in range(12)) for _ in range(5000)]
        buf = io.BytesIO()
        spm.SentencePieceTrainer.train(sentence_iterator=iter(lines), model_writer=buf, vocab_size=GO.V, model_type="unigram",
                                       character_coverage=1.0, bos_id=-1, eos_id=-1, unk_id=0, num_threads=1, minloglevel=2)
        with open(GO.SPM_MODEL, "wb") as f:
            f.write(buf.getvalue())
    sp = GO.sp_model()
    assert sp.vocab_size() == GO.V
    return sp


def reference_modules(sd, w_enc, W):
    import speechbrain as sb
    from speechbrain.lobes.features import Fbank
    from speechbrain.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain.lobes.models.transformer.TransformerASR import TransformerASR
    from speechbrain.processing.features import InputNormalization
    cfg = GO.config()
    fb = Fbank(sample_rate=16000, n_fft=512, n_mels=80, win_length=32)
    norm = InputNormalization(norm_type="global")
    norm.glob_mean, norm.glob_std, norm.count = sd["normalize.glob_mean"], sd["normalize.glob_std"], 1
    norm.eval()
    cnn = ConvolutionFrontEnd(input_shape=(8, 10, 80), num_blocks=2, num_layers_per_block=1, out_channels=(64, 32),
                              kernel_sizes=(3, 3), strides=(2, 2), residuals=(False, False))
    cnn.load_state_dict({k[4:]: v for k, v in sd.items() if k.startswith("CNN.")})
    cnn.eval()
    tr = TransformerASR(input_size=640, tgt_vocab=GO.V, d_model=cfg["d_model"], nhead=cfg["nhead"],
                        num_encoder_layers=cfg["num_encoder_layers"], num_decoder_layers=0, d_ffn=cfg["d_ffn"],
                        dropout=0.1, activation=torch.nn.GELU, encoder_module="conformer", attention_type="RelPosMHAXL",
                        normalize_before=True, causal=False, max_length=2500)
    missing, unexpected = tr.load_state_dict({k[len("Transformer."):]: v for k, v in sd.items()
                                              if k.startswith("Transformer.")}, strict=False)
    assert not unexpected and all(k.startswith("positional_encoding") for k in missing), (missing, unexpected)
    tr.eval()
    proj_enc = sb.nnet.linear.Linear(input_size=cfg["d_model"], n_neurons=GO.J, bias=False)
    proj_enc.load_state_dict({"w.weight": w_enc})
    searcher, pn_keys = MT.reference_searcher(W, GO.BLANK)
    shapes = {"CNN": cnn, "Transformer": tr, "proj_enc": proj_enc}
    keys = {p: {k: list(v.shape) for k, v in m.state_dict().items()} for p, m in shapes.items()}
    for p, m in zip(("emb", "dec", "proj_dec"), searcher.decode_network_lst):
        keys[p] = {k: list(v.shape) for k, v in m.state_dict().items()}
    keys["transducer_lin"] = {k: list(v.shape) for k, v in searcher.classifier_network[0].state_dict().items()}
    return fb, norm, cnn, tr, proj_enc, searcher, keys


def record_joint(searcher):
    calls = []
    orig = searcher._joint_forward_step

    def rec(h_i, out_PN):
        lp = orig(h_i, out_PN)
        flat = lp.squeeze(1).squeeze(1)
        calls.append((h_i.storage_offset() // h_i.shape[-1], flat.topk(2, dim=-1).values.clone(), flat.argmax(-1).clone()))
        return lp
    searcher._joint_forward_step = rec
    return calls, orig


def offline(sd, w_enc, W):
    from speechbrain.utils.dynamic_chunk_training import DynChunkTrainConfig
    fb, norm, cnn, tr, proj_enc, searcher, keys = reference_modules(sd, w_enc, W)
    wav, lens = GO.waveforms()
    with torch.no_grad():
        src = cnn(norm(fb(wav), lens))
        enc = tr.encode(src, lens)
        enc_dc = tr.encode(src, lens, dynchunktrain_config=DynChunkTrainConfig(*GO.DYNCHUNK))
        tn = proj_enc(enc).contiguous()
        calls, orig = record_joint(searcher)
        hyps, score, _, _ = searcher.transducer_greedy_decode(tn, max_symbols_per_step=GO.MAX_SYMBOLS)
        searcher._joint_forward_step = orig
    o_enc = GO.encode(sd, wav, lens)
    o_dc = GO.encode(sd, wav, lens, dynchunk=GO.DYNCHUNK)
    assert G.rel(o_enc, enc) < 1e-5 and G.rel(o_dc, enc_dc) < 1e-5, (G.rel(o_enc, enc), G.rel(o_dc, enc_dc))
    rows = GO.greedy(W, tn)
    assert [r["tokens"] for r in rows] == hyps
    hist = collections.Counter()
    for r in rows:
        c = collections.Counter(r["frames"])
        hist.update(min(c.get(t, 0), 2) for t in range(tn.shape[1]))
    assert all(hist[k] > 0 for k in (0, 1, 2)), hist
    dec = MT.row_decisions(calls, tn.shape[0], GO.BLANK, GO.MAX_SYMBOLS)
    beam = MB.check_and_record(W, tn, GO.BLANK, dict(name="gigaspeech beam 10", beam=GO.BEAM, nbest=1, sb=GO.STATE_BEAM,
                                                     eb=GO.EXPAND_BEAM))
    print("offline: T", tn.shape[1], "greedy tokens", [len(h) for h in hyps], "frames by emissions", dict(hist))
    return dict(wav_checksum=float(wav.double().abs().sum()), enc_norms=enc.double().norm(dim=-1).float(),
                tn_norms=tn.double().norm(dim=-1).float(), dynchunk=GO.DYNCHUNK,
                dynchunk_enc_norms=enc_dc.double().norm(dim=-1).float(), tokens=hyps, score=float(score),
                decisions=[d[0] for d in dec], margins=[d[1] for d in dec], emission_hist=dict(hist), beam=beam), keys


def streaming(sd, w_enc, W, sp):
    import speechbrain as sb  # noqa: F401
    from speechbrain.decoders.transducer import TransducerBeamSearcher, TransducerGreedySearcherStreamingContext
    from speechbrain.inference.ASR import StreamingASR
    from speechbrain.lobes.features import StreamingFeatureWrapper
    from speechbrain.lobes.models.transformer.TransformerASR import EncoderWrapper
    from speechbrain.nnet.containers import LengthsCapableSequential
    from speechbrain.tokenizers.SentencePiece import SentencePieceDecoderStreamingContext, spm_decode_preserve_leading_space
    from speechbrain.utils.dynamic_chunk_training import DynChunkTrainConfig
    from speechbrain.utils.filter_analysis import stack_filter_properties
    wav = GO.waveforms()[0][:3, :SO.L_AUDIO].contiguous()
    out = {}
    for name, (chunk, left) in CASES.items():
        fb, norm, cnn, tr, proj_enc, searcher, _ = reference_modules(sd, w_enc, W)
        fea = StreamingFeatureWrapper(LengthsCapableSequential(fb, norm, cnn), stack_filter_properties([fb, cnn]))
        fea.eval()
        hp = dict(fea_streaming_extractor=fea, make_decoder_streaming_context=TransducerGreedySearcherStreamingContext,
                  decoding_function=functools.partial(TransducerBeamSearcher.transducer_greedy_decode_streaming, searcher),
                  make_tokenizer_streaming_context=SentencePieceDecoderStreamingContext,
                  tokenizer_decode_streaming=spm_decode_preserve_leading_space, tokenizer=sp)
        asr = StreamingASR(modules={"enc": EncoderWrapper(tr), "proj_enc": proj_enc}, hparams=hp, run_opts={"device": "cpu"})
        asr.mods.eval()
        dc = DynChunkTrainConfig(chunk, left)
        assert asr.get_chunk_size_frames(dc) == SO.chunk_samples(chunk)
        assert fea.get_required_padding() == SO.PAD and fea.properties.stride == SO.STRIDE
        feats = []
        orig_fwd = fea.forward

        def rec_fwd(*a, **k):
            y = orig_fwd(*a, **k)
            feats.append(y.clone())
            return y
        fea.forward = rec_fwd
        calls, _ = record_joint(searcher)
        ctx = asr.make_streaming_context(dc)
        B = wav.shape[0]
        rec = dict(chunk=chunk, left=left, pad=fea.get_required_padding(), chunk_samples=asr.get_chunk_size_frames(dc),
                   window_size=fea.properties.window_size, stride=fea.properties.stride, feat_norms=[], tn_norms=[],
                   tokens=[], decisions=[], margins=[], words=[])
        with torch.no_grad():
            for ch in SO.chunks(wav, chunk):
                feats.clear()
                calls.clear()
                x = asr.encode_chunk(ctx, ch)
                words, toks = asr.decode_chunk(ctx, x)
                dec = MT.row_decisions(calls, B, GO.BLANK, SO.MAX_SYMBOLS)
                rec["feat_norms"].append(feats[0].reshape(B, feats[0].shape[1], -1).double().norm(dim=-1).float())
                rec["tn_norms"].append(x.double().norm(dim=-1).float())
                rec["tokens"].append(toks)
                rec["decisions"].append([d[0] for d in dec])
                rec["margins"].append([d[1] for d in dec])
                rec["words"].append(words)
        o = SO.run(wav, sd, GO.config(), w_enc, W, chunk, left, sp)
        assert [c[2] for c in o] == rec["tokens"], name
        assert [c[3] for c in o] == rec["words"], name
        tn_rel = max(G.rel(c[1].norm(dim=-1), n) for c, n in zip(o, rec["tn_norms"]))
        assert tn_rel < 1e-5, (name, tn_rel)
        print(name, "chunks", len(rec["tokens"]), "tokens per row", [sum(len(t[b]) for t in rec["tokens"]) for b in range(B)],
              "text", ["".join(w[b] for w in rec["words"])[:30] for b in range(B)])
        out[name] = rec
    return out


def main():
    torch.set_num_threads(8)
    sp = train_spm()
    sd, w_enc, W = GO.weights()
    off, keys = offline(sd, w_enc, W)
    out = dict(offline=off, streaming=streaming(sd, w_enc, W, sp), keys=keys, wav_rows=3, audio_samples=SO.L_AUDIO,
               max_symbols=GO.MAX_SYMBOLS, spm_checksum=sum(sp.serialized_model_proto()))
    G.save(out, "gigaspeech.pt")


if __name__ == "__main__":
    main()
