"""StreamingASR built from this package's mirrors on the LibriSpeech transducer model of transducer.pt's "e2e" entry (or the
same model with RelPosMHAXL attention), the way the recipe's inference block wires it; shared by the GPU tests and
tools/streaming_asr_e2e.py.  The tokenizer is the committed 1000-piece SentencePiece model."""
import functools
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from streaming_asr_oracle import sp_model  # noqa: E402,F401


def model_inputs(att="RoPEMHA"):
    """(cfg, sd, w_enc, W, wav) of the fixture's model with attention ``att`` and its waveforms (first three rows, 6 s)."""
    import make_transducer_golden as MT
    import streaming_asr_oracle as SO
    from speechbrain_b200.utils.seeded_init import seeded_asr_state
    cfg, sd, w_enc, W, wav, _ = MT.e2e_inputs()
    if att != cfg["attention_type"]:
        cfg = dict(cfg, attention_type=att)
        sd = seeded_asr_state(cfg, MT.E2E["seed"])
    return cfg, sd, w_enc, W, wav[:3, :SO.L_AUDIO].contiguous()


def modules(cfg, sd, w_enc, W):
    """The recipe's modules: (fbank, normalize, cnn, EncoderWrapper, proj_enc, greedy TransducerBeamSearcher)."""
    from mirrors import build_mirror
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.lobes.models.transformer.TransformerASR import EncoderWrapper
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
    return mirror.fb, mirror.norm, mirror.cnn, EncoderWrapper(mirror.tr), proj_enc, s


def build(att="RoPEMHA", device="cuda:0"):
    """(StreamingASR, cfg, sd, w_enc, W, wav)."""
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher, TransducerGreedySearcherStreamingContext
    from speechbrain_b200.inference.ASR import StreamingASR
    from speechbrain_b200.lobes.features import StreamingFeatureWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.tokenizers.SentencePiece import SentencePieceDecoderStreamingContext, spm_decode_preserve_leading_space
    from speechbrain_b200.utils.filter_analysis import stack_filter_properties
    cfg, sd, w_enc, W, wav = model_inputs(att)
    fb, norm, cnn, enc, proj_enc, searcher = modules(cfg, sd, w_enc, W)
    fea = StreamingFeatureWrapper(LengthsCapableSequential(fb, norm, cnn), stack_filter_properties([fb, cnn]))
    hp = dict(fea_streaming_extractor=fea, make_decoder_streaming_context=TransducerGreedySearcherStreamingContext,
              decoding_function=functools.partial(TransducerBeamSearcher.transducer_greedy_decode_streaming, searcher),
              make_tokenizer_streaming_context=SentencePieceDecoderStreamingContext,
              tokenizer_decode_streaming=spm_decode_preserve_leading_space, tokenizer=sp_model())
    asr = StreamingASR(modules={"enc": enc, "proj_enc": proj_enc}, hparams=hp, run_opts={"device": device})
    return asr, cfg, sd, w_enc, W, wav
