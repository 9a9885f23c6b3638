"""The GigaSpeech Conformer-Transducer (utils/seeded_init.GIGASPEECH_TRANSDUCER: 12 Conformer layers at d_model 768 with
RelPosMHAXL, 8 heads of 96, no decoder layers; proj_enc 768 -> 512, LSTM 512, joint 512 with GELU over 1024 tokens, blank 0)
on seeded weights, and its fp32 CPU oracle: oracle/asr_oracle.py for the front end and the encoder (full context or a
Dynamic Chunk mask), transducer_oracle.py for the greedy search and transducer_beam_oracle.py for the beam search.

The offline batch is 4 x 10 s ragged [1.0, 0.9, 0.6, 0.3] (conformer640_oracle.waveforms).  The seeded encoder's output
has a large component common to every frame, so the classifier's blank row decides nearly alone: BLANK_GAIN is the value
at which the greedy search emits 0, 1 and >= 2 tokens on some frames (0.6 emits on every frame, 0.8 almost never).
"""
import os

import torch

import conformer640_oracle as CO
import transducer_oracle as TO
from mirrors import seeded
from oracle import asr_oracle as O

SEED, PN_SEED = 0, 31
J, H, V, BLANK = 512, 512, 1024, 0
ENC_SCALE, BLANK_GAIN, MAX_SYMBOLS = 1.0, 0.7, 5
BEAM, STATE_BEAM, EXPAND_BEAM = 10, 2.3, 2.3
DYNCHUNK = (16, 2)  # chunk 16 frames, 2 chunks of left context
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SPM_MODEL = os.path.join(GOLDEN, "gigaspeech_spm.model")


def sp_model():
    """The committed 1024-piece unigram SentencePiece model (id 0 = <unk>, the transducer's blank)."""
    import sentencepiece as spm
    return spm.SentencePieceProcessor(model_file=SPM_MODEL)


def config():
    from speechbrain_b200.utils.seeded_init import GIGASPEECH_TRANSDUCER
    return GIGASPEECH_TRANSDUCER


def weights():
    """(sd, w_enc [512, 768], W): the encoder state, proj_enc's weight and the prediction network and classifier."""
    from speechbrain_b200.utils.seeded_init import seeded_tensor
    cfg = config()
    sd = seeded(cfg, SEED)
    w_enc = seeded_tensor(SEED, "proj_enc.w.weight", (J, cfg["d_model"])) * ENC_SCALE
    W = TO.seeded_weights(PN_SEED, J, H, V, BLANK, blank_gain=BLANK_GAIN)
    return sd, w_enc, W


def waveforms():
    return CO.waveforms()


@torch.no_grad()
def encode(sd, wav, lens, dynchunk=None):
    """fp32 encoder states [B, T, 768] (dynchunk = (chunk, left chunks): the masked full-sequence run)"""
    cfg = config()
    feats = O.full_pipeline_features(wav, lens, sd, dict(cfg, win_length=cfg["win"] * 1000 // cfg["sample_rate"]))
    return O.encode(feats, lens, sd, cfg, CO.PREFIX, dynchunk=dynchunk)


def tn_output(enc, w_enc):
    return enc @ w_enc.T


def greedy(W, tn):
    """the oracle's greedy search of each row over every frame, padded ones included, as TransducerBeamSearcher runs it"""
    oracle = TO.Oracle(W)
    return [oracle.row(tn[b], BLANK, MAX_SYMBOLS) for b in range(tn.shape[0])]


# ------------------------------------------------------------------------------------------------ this package's modules
def modules(sd, w_enc, W):
    """The recipe's modules from this package's mirrors: (fbank, normalize, cnn, Transformer, proj_enc, emb, dec, proj_dec,
    transducer_lin, greedy TransducerBeamSearcher)."""
    from mirrors import build_mirror
    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher
    from speechbrain_b200.nnet.embedding import Embedding
    from speechbrain_b200.nnet.linear import Linear
    from speechbrain_b200.nnet.RNN import LSTM
    from speechbrain_b200.nnet.transducer.transducer_joint import Transducer_joint
    mirror = build_mirror(config(), sd)
    proj_enc = Linear(input_size=config()["d_model"], n_neurons=J, bias=False)
    proj_enc.load_state_dict({"w.weight": w_enc})
    emb = Embedding(num_embeddings=V, consider_as_one_hot=True, blank_id=BLANK)
    dec = LSTM(input_shape=[None, None, V - 1], hidden_size=H, num_layers=1)
    proj_dec = Linear(input_size=H, n_neurons=J, bias=False)
    lin = Linear(input_size=J, n_neurons=V, bias=False)
    for prefix, m in (("emb", emb), ("dec", dec), ("proj_dec", proj_dec), ("transducer_lin", lin)):
        m.load_state_dict({k[len(prefix) + 1:]: v for k, v in W.items() if k.startswith(prefix + ".")})
    s = TransducerBeamSearcher([emb, dec, proj_dec], Transducer_joint(joint="sum", nonlinearity=torch.nn.GELU), [lin],
                               blank_id=BLANK, beam_size=1, nbest=1)
    return dict(fb=mirror.fb, norm=mirror.norm, CNN=mirror.cnn, Transformer=mirror.tr, proj_enc=proj_enc, emb=emb, dec=dec,
                proj_dec=proj_dec, transducer_lin=lin, searcher=s)


def streaming_asr(device="cuda:0"):
    """(StreamingASR built as the recipe's commented inference block wires it, the modules, sd, w_enc, W, wav of the first 6 s
    of three rows)"""
    import functools

    from speechbrain_b200.decoders.transducer import TransducerBeamSearcher, TransducerGreedySearcherStreamingContext
    from speechbrain_b200.inference.ASR import StreamingASR
    from speechbrain_b200.lobes.features import StreamingFeatureWrapper
    from speechbrain_b200.lobes.models.transformer.TransformerASR import EncoderWrapper
    from speechbrain_b200.nnet.containers import LengthsCapableSequential
    from speechbrain_b200.tokenizers.SentencePiece import SentencePieceDecoderStreamingContext, spm_decode_preserve_leading_space
    from speechbrain_b200.utils.filter_analysis import stack_filter_properties
    sd, w_enc, W = weights()
    m = modules(sd, w_enc, W)
    fea = StreamingFeatureWrapper(LengthsCapableSequential(m["fb"], m["norm"], m["CNN"]), stack_filter_properties([m["fb"], m["CNN"]]))
    hp = dict(fea_streaming_extractor=fea, make_decoder_streaming_context=TransducerGreedySearcherStreamingContext,
              decoding_function=functools.partial(TransducerBeamSearcher.transducer_greedy_decode_streaming, m["searcher"]),
              make_tokenizer_streaming_context=SentencePieceDecoderStreamingContext,
              tokenizer_decode_streaming=spm_decode_preserve_leading_space, tokenizer=sp_model())
    asr = StreamingASR(modules={"enc": EncoderWrapper(m["Transformer"]), "proj_enc": m["proj_enc"]}, hparams=hp,
                       run_opts={"device": device})
    import streaming_asr_oracle as SO
    return asr, m, sd, w_enc, W, waveforms()[0][:3, :SO.L_AUDIO].contiguous()


CKPT_ORDER = ["CNN", "Transformer", "proj_enc", "emb", "dec", "proj_dec", "transducer_lin"]


def asr_ckpt(m):
    """asr.ckpt in the recipe's ModuleList key layout"""
    return {f"{i}.{k}": v for i, n in enumerate(CKPT_ORDER) for k, v in m[n].state_dict().items()}


# The recipe's model block (conformer_transducer.yaml) with its offline EncoderDecoderASR inference block, the layout of a
# pretrained-model directory; STREAMING_HPARAMS is the commented StreamingASR block of the same file.
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
    tgt_vocab: 1024
    d_model: 768
    nhead: 8
    num_encoder_layers: 12
    num_decoder_layers: 0
    d_ffn: 2048
    dropout: 0.1
    activation: !ref <activation>
    encoder_module: conformer
    attention_type: RelPosMHAXL
    normalize_before: True
    causal: False
enc: !new:speechbrain.lobes.models.transformer.TransformerASR.EncoderWrapper
    transformer: !ref <Transformer>
proj_enc: !new:speechbrain.nnet.linear.Linear
    input_size: 768
    n_neurons: 512
    bias: False
proj_dec: !new:speechbrain.nnet.linear.Linear
    input_size: 512
    n_neurons: 512
    bias: False
emb: !new:speechbrain.nnet.embedding.Embedding
    num_embeddings: 1024
    consider_as_one_hot: True
    blank_id: !ref <blank_index>
dec: !new:speechbrain.nnet.RNN.LSTM
    input_shape: [null, null, 1023]
    hidden_size: 512
    num_layers: 1
    re_init: True
Tjoint: !new:speechbrain.nnet.transducer.transducer_joint.Transducer_joint
    joint: sum
    nonlinearity: !ref <activation>
transducer_lin: !new:speechbrain.nnet.linear.Linear
    input_size: 512
    n_neurons: 1024
    bias: False
decoder: !new:speechbrain.decoders.transducer.TransducerBeamSearcher
    decode_network_lst: [!ref <emb>, !ref <dec>, !ref <proj_dec>]
    tjoint: !ref <Tjoint>
    classifier_network: [!ref <transducer_lin>]
    blank_id: !ref <blank_index>
    beam_size: 10
    nbest: 1
    state_beam: 2.3
    expand_beam: 2.3
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

STREAMING_HPARAMS = HPARAMS.replace("tokenizer: null\n", "").replace("transducer_beam_search: True\n", "").replace(
    "    beam_size: 10\n    nbest: 1\n    state_beam: 2.3\n    expand_beam: 2.3\n", "    beam_size: 1\n    nbest: 1\n").replace(
    "modules:\n    encoder: !ref <encoder>\n    decoder: !ref <decoder>\n", "") + """
Greedysearcher: !ref <decoder>
tokenizer: !apply:gigaspeech_oracle.sp_model
make_tokenizer_streaming_context: !name:speechbrain.tokenizers.SentencePiece.SentencePieceDecoderStreamingContext
tokenizer_decode_streaming: !name:speechbrain.tokenizers.SentencePiece.spm_decode_preserve_leading_space
make_decoder_streaming_context: !name:speechbrain.decoders.transducer.TransducerGreedySearcherStreamingContext
decoding_function: !name:speechbrain.decoders.transducer.TransducerBeamSearcher.transducer_greedy_decode_streaming
    - !ref <Greedysearcher>
fea_streaming_extractor: !new:speechbrain.lobes.features.StreamingFeatureWrapper
    module: !new:speechbrain.nnet.containers.LengthsCapableSequential
        - !ref <compute_features>
        - !ref <normalizer>
        - !ref <CNN>
    properties: !apply:speechbrain.utils.filter_analysis.stack_filter_properties
        - [!ref <compute_features>, !ref <CNN>]
modules:
    enc: !ref <enc>
    proj_enc: !ref <proj_enc>
"""
