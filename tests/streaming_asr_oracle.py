"""CPU oracle of StreamingASR.transcribe_chunk (inference/ASR.py:1156-1363) for the Conformer-Transducer, built on the
front-end, encoder and transducer oracles: per chunk the StreamingFeatureWrapper window [last 2 * pad samples | chunk]
(zeros before the first) through Fbank -> global CMVN -> ConvolutionFrontEnd, pad / stride frames trimmed off each side;
the encoder as the masked full-sequence run (DynChunkTrainConfig) over the concatenated chunk features, which is what
chunk-by-chunk streaming computes; proj_enc; the greedy transducer search carried across chunks; and the SentencePiece
streaming detokeniser.  Also the fixture's shared inputs: the chunking and the 1000-piece SentencePiece model."""
import os

import torch

import transducer_oracle as TO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SPM_MODEL = os.path.join(GOLDEN, "streaming_asr_spm.model")
PAD, STRIDE = 1280, 640  # upalign((1473 - 1) // 2, 640) for Fbank(n_fft=512, win_length=32) + the 2-block front end
L_AUDIO = 96000          # the first 6 s of transducer.pt's "e2e" waveforms
MAX_SYMBOLS = 5
CASES = {"rope_24_8": ("RoPEMHA", 24, 8), "rope_16_2": ("RoPEMHA", 16, 2), "rope_8_0": ("RoPEMHA", 8, 0),
         "relpos_16_2": ("RelPosMHAXL", 16, 2)}


def sp_model():
    """The committed 1000-piece unigram SentencePiece model (id 0 = <unk>, the transducer's blank)."""
    import sentencepiece as spm
    return spm.SentencePieceProcessor(model_file=SPM_MODEL)


def chunk_samples(chunk_size):
    """StreamingASR.get_chunk_size_frames: (stride - 1) * chunk_size samples."""
    return (STRIDE - 1) * chunk_size


def chunks(wav, chunk_size):
    """The audio with the recommended zero chunks (upalign(pad, n) / n of them) appended, split into chunks of n samples:
    only the last chunk is short."""
    n = chunk_samples(chunk_size)
    k = -(-PAD // n)
    full = torch.cat([wav, torch.zeros(wav.shape[0], k * n)], dim=1)
    return [full[:, t:t + n].contiguous() for t in range(0, full.shape[1], n)]


def windows(wav, chunk_size):
    carry = torch.zeros(wav.shape[0], 2 * PAD)
    for ch in chunks(wav, chunk_size):
        win = torch.cat([carry, ch], dim=1)
        carry = win[:, -2 * PAD:]
        yield win


def front_end(win, sd):
    """The wrapper's output for one window [B, 2 * pad + n] -> [B, frames, 640]."""
    from oracle import asr_oracle as O
    f = O.fbank(win, n_fft=512, n_mels=80, win_length_ms=32)
    f = O.input_norm(f, None, "global", sd["normalize.glob_mean"], sd["normalize.glob_std"])
    y = O.cnn_frontend(f, sd, "CNN.")
    trim = PAD // STRIDE
    return y.reshape(y.shape[0], y.shape[1], -1)[:, trim:y.shape[1] - trim]


def detokenise(sp, hyps, ctx):
    """spm_decode_preserve_leading_space (tokenizers/SentencePiece.py:527-577); ctx a one-element list (symbols emitted)."""
    proto = sp.decode([hyps], out_type="immutable_proto")[0]
    text = proto.text
    if len(proto.pieces) >= 1:
        if ctx[0] > 0 and proto.pieces[0].piece.startswith("▁"):
            text = " " + text
        ctx[0] += len(proto.pieces)
    return text


def run(wav, sd, cfg, w_enc, W, chunk_size, left, sp):
    """Per chunk: wrapper output, proj_enc output, tokens per row, text per row."""
    from oracle import asr_oracle as O
    feats = [front_end(win, sd) for win in windows(wav, chunk_size)]
    src = torch.cat(feats, dim=1)
    enc = O.encode(src, torch.ones(src.shape[0]), sd, cfg, "Transformer.", dynchunk=(chunk_size, left))
    tn = enc @ w_enc.T
    oracle = TO.Oracle(W)
    B = wav.shape[0]
    state = [None] * B
    tctx = [[0] for _ in range(B)]
    out, t0 = [], 0
    for f in feats:
        n = f.shape[1]
        toks, words = [], []
        for b in range(B):
            r = oracle.row(tn[b, t0:t0 + n], 0, MAX_SYMBOLS, state=state[b])
            state[b] = r["state"]
            toks.append(r["tokens"])
            words.append(detokenise(sp, r["tokens"], tctx[b]))
        out.append((f, tn[:, t0:t0 + n], toks, words))
        t0 += n
    return out
