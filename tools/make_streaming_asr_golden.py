"""Generate tests/golden/streaming_asr.pt (and the SentencePiece model tests/golden/streaming_asr_spm.model) by RUNNING THE
REFERENCE StreamingASR (speechbrain.inference.ASR, built with modules= / hparams= directly) chunk by chunk.

How to run it: oracle/goldens.py.  The model is transducer.pt's "e2e" one (make_transducer_golden.e2e_inputs: 12-layer
RoPEMHA Conformer, proj_enc 512 -> 640, 640 / 512 / 1000 prediction network), plus the same model with RelPosMHAXL
attention (seeded_asr_state of that config with the same seed).  The audio is the first 6 s of the e2e batch's first three
rows (lengths 1.0, 0.9, 0.6 of 10 s), with the recommended zero chunks appended and split into chunks of
get_chunk_size_frames samples (tests/streaming_asr_oracle.chunks).  Cases: RoPE at DynChunkTrainConfig (24, 8), (16, 2)
and (8, 0) (the reference cannot stream with an unlimited left context: its
Conformer layer compares the None left-context size with 0), RelPos at (16, 2).

Per case and chunk it stores the filter properties and the pad / chunk sample counts, the wrapper output's and the
proj_enc output's per-frame norms, each row's tokens, decisions (frame, token) and top-1 / top-2 margins as the reference's
joint calls took them, and each row's detokenised string.  It asserts that the CPU oracle (tests/streaming_asr_oracle.py)
gives the reference's tokens and strings.

The tokenizer is a 1000-piece unigram SentencePiece model trained here on seeded synthetic text (written only when
absent, so the committed model stays what the fixture was made with)."""
import functools
import io
import os
import random

import torch

from oracle import goldens as G  # also puts tests/ on sys.path

import make_transducer_golden as MT  # noqa: E402  (tools/ is the script's directory)
import streaming_asr_oracle as SO  # noqa: E402


def train_spm():
    import sentencepiece as spm
    if not os.path.exists(SO.SPM_MODEL):
        rng = random.Random(0)
        words = ["".join(rng.choice("abcdefghijklmnopqrstuvwxyz") for _ in range(rng.randint(2, 8))) for _ in range(3000)]
        lines = [" ".join(rng.choice(words) for _ in range(12)) for _ in range(4000)]
        buf = io.BytesIO()
        spm.SentencePieceTrainer.train(sentence_iterator=iter(lines), model_writer=buf, vocab_size=1000, model_type="unigram",
                                       character_coverage=1.0, bos_id=-1, eos_id=-1, unk_id=0, num_threads=1, minloglevel=2)
        with open(SO.SPM_MODEL, "wb") as f:
            f.write(buf.getvalue())
    sp = SO.sp_model()
    assert sp.vocab_size() == 1000
    return sp


def model_inputs(att):
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    cfg, sd, w_enc, W, wav, _ = MT.e2e_inputs()
    if att != cfg["attention_type"]:
        cfg = dict(cfg, attention_type=att)
        sd = seeded_asr_state(cfg, MT.E2E["seed"])
    return cfg, sd, w_enc, W, wav[:3, :SO.L_AUDIO].contiguous()


def reference_asr(cfg, sd, w_enc, W, sp):
    import speechbrain as sb
    from speechbrain.decoders.transducer import TransducerBeamSearcher, TransducerGreedySearcherStreamingContext
    from speechbrain.inference.ASR import StreamingASR
    from speechbrain.lobes.features import Fbank, StreamingFeatureWrapper
    from speechbrain.lobes.models.convolution import ConvolutionFrontEnd
    from speechbrain.lobes.models.transformer.TransformerASR import EncoderWrapper, TransformerASR
    from speechbrain.nnet.containers import LengthsCapableSequential
    from speechbrain.processing.features import InputNormalization
    from speechbrain.tokenizers.SentencePiece import SentencePieceDecoderStreamingContext, spm_decode_preserve_leading_space
    from speechbrain.utils.filter_analysis import stack_filter_properties
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
                        attention_type=cfg["attention_type"], normalize_before=True, causal=False)
    tr.load_state_dict({k[len("Transformer."):]: v for k, v in sd.items() if k.startswith("Transformer.")}, strict=False)
    tr.eval()
    proj_enc = sb.nnet.linear.Linear(input_size=512, n_neurons=640, bias=False)
    proj_enc.load_state_dict({"w.weight": w_enc})
    searcher, _ = MT.reference_searcher(W, 0)
    fea = StreamingFeatureWrapper(LengthsCapableSequential(fb, norm, cnn), stack_filter_properties([fb, cnn]))
    fea.eval()
    hp = dict(fea_streaming_extractor=fea, make_decoder_streaming_context=TransducerGreedySearcherStreamingContext,
              decoding_function=functools.partial(TransducerBeamSearcher.transducer_greedy_decode_streaming, searcher),
              make_tokenizer_streaming_context=SentencePieceDecoderStreamingContext,
              tokenizer_decode_streaming=spm_decode_preserve_leading_space, tokenizer=sp)
    asr = StreamingASR(modules={"enc": EncoderWrapper(tr), "proj_enc": proj_enc}, hparams=hp, run_opts={"device": "cpu"})
    asr.mods.eval()
    return asr, fea, searcher


def run_case(name, sp):
    from speechbrain.utils.dynamic_chunk_training import DynChunkTrainConfig
    att, chunk, left = SO.CASES[name]
    cfg, sd, w_enc, W, wav = model_inputs(att)
    asr, fea, searcher = reference_asr(cfg, sd, w_enc, W, sp)
    dc = DynChunkTrainConfig(chunk, left)
    assert asr.get_chunk_size_frames(dc) == SO.chunk_samples(chunk)
    assert fea.get_required_padding() == SO.PAD and fea.properties.stride == SO.STRIDE
    feats, calls = [], []
    orig_fwd, orig_joint = fea.forward, searcher._joint_forward_step

    def rec_fwd(*a, **k):
        y = orig_fwd(*a, **k)
        feats.append(y.clone())
        return y

    def rec_joint(h_i, out_PN):
        lp = orig_joint(h_i, out_PN)
        flat = lp.squeeze(1).squeeze(1)
        calls.append((h_i.storage_offset() // h_i.shape[-1], flat.topk(2, dim=-1).values.clone(), flat.argmax(-1).clone()))
        return lp
    fea.forward, searcher._joint_forward_step = rec_fwd, rec_joint
    ctx = asr.make_streaming_context(dc)
    B = wav.shape[0]
    rec = dict(att=att, chunk=chunk, left=left, pad=fea.get_required_padding(), chunk_samples=asr.get_chunk_size_frames(dc),
               window_size=fea.properties.window_size, stride=fea.properties.stride, feat_norms=[], tn_norms=[], tokens=[],
               decisions=[], margins=[], words=[])
    with torch.no_grad():
        for ch in SO.chunks(wav, chunk):
            feats.clear()
            calls.clear()
            x = asr.encode_chunk(ctx, ch)
            words, toks = asr.decode_chunk(ctx, x)
            dec = MT.row_decisions(calls, B, 0, SO.MAX_SYMBOLS)
            rec["feat_norms"].append(feats[0].reshape(B, feats[0].shape[1], -1).double().norm(dim=-1).float())
            rec["tn_norms"].append(x.double().norm(dim=-1).float())
            rec["tokens"].append(toks)
            rec["decisions"].append([d[0] for d in dec])
            rec["margins"].append([d[1] for d in dec])
            rec["words"].append(words)
    o = SO.run(wav, sd, cfg, w_enc, W, chunk, left, sp)
    assert [c[2] for c in o] == rec["tokens"], name
    assert [c[3] for c in o] == rec["words"], name
    fe = max(G.rel(c[0].norm(dim=-1), n) for c, n in zip(o, rec["feat_norms"]))
    print(name, "chunks", len(rec["tokens"]), "tokens per row", [sum(len(t[b]) for t in rec["tokens"]) for b in range(B)],
          "oracle front-end norm rel", f"{fe:.1e}", "text", ["".join(w[b] for w in rec["words"])[:40] for b in range(B)])
    return rec


def main():
    torch.set_num_threads(8)
    sp = train_spm()
    out = dict(cases={}, wav_rows=3, audio_samples=SO.L_AUDIO, max_symbols=SO.MAX_SYMBOLS,
               spm_checksum=sum(sp.serialized_model_proto()))
    for name in SO.CASES:
        out["cases"][name] = run_case(name, sp)
    G.save(out, "streaming_asr.pt")


if __name__ == "__main__":
    main()
