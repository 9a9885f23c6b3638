"""Python handle on the C-ABI model engine (sbk_asr_*): repacks a reference-keyed state_dict once and
runs the fused device pipeline.  Used by the nn.Module mirrors and by EncoderDecoderASR."""
import ctypes
import itertools
import math

import torch

from . import _lib
from ._lib import check, lib, ptr, stream_ptr


def stft_window(n_fft, win_length_samples):
    """torch.hamming_window (periodic), centre-padded to n_fft like torch.stft does
    (reference: processing/features.py:139,159-170)."""
    w = torch.hamming_window(win_length_samples)
    if win_length_samples < n_fft:
        left = (n_fft - win_length_samples) // 2
        w = torch.nn.functional.pad(w, (left, n_fft - win_length_samples - left))
    return w.contiguous()


def mel_filter_matrix(n_mels, n_fft, sample_rate=16000, f_min=0, f_max=None):
    """The (n_fft//2+1, n_mels) triangular matrix of processing/features.py:487-507,620-650, built with the
    same torch ops so the filter values are bit-identical to the reference's."""
    if f_max is None:
        f_max = sample_rate // 2
    n_stft = n_fft // 2 + 1
    to_mel = lambda hz: 2595 * math.log10(1 + hz / 700)
    mel = torch.linspace(to_mel(f_min), to_mel(f_max), n_mels + 2)
    hz = 700 * (10 ** (mel / 2595) - 1)
    band = (hz[1:] - hz[:-1])[:-1]
    f_central = hz[1:-1]
    all_freqs = torch.linspace(0, sample_rate // 2, n_stft)
    all_freqs_mat = all_freqs.repeat(f_central.shape[0], 1)
    f_central_mat = f_central.repeat(all_freqs_mat.shape[1], 1).transpose(0, 1)
    band_mat = band.repeat(all_freqs_mat.shape[1], 1).transpose(0, 1)
    slope = (all_freqs_mat - f_central_mat) / band_mat
    m = torch.max(torch.zeros(1), torch.min(slope + 1.0, -slope + 1.0)).transpose(0, 1)
    return m.contiguous()


class FbankHandle:
    """sbk_fbank_* handle."""

    def __init__(self, n_fft, hop, n_mels, window, mel_matrix, amin=1e-10, top_db=80.0):
        self.n_fft, self.hop, self.n_mels = n_fft, hop, n_mels
        self._h = ctypes.c_void_p()
        w = window.float().contiguous().cpu()
        mm = mel_matrix.float().contiguous().cpu()
        check(lib().sbk_fbank_create(n_fft, hop, n_mels, ptr(w), ptr(mm), ctypes.c_float(amin), ctypes.c_float(top_db),
                                     ctypes.byref(self._h)), "sbk_fbank_create")

    def __del__(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().sbk_fbank_destroy(self._h)
            self._h = None

    def forward(self, wav):
        _lib.require_cuda(wav, "Fbank")
        wav = wav.float().contiguous()
        B, L = wav.shape
        T = 1 + L // self.hop
        out = torch.empty(B, T, self.n_mels, device=wav.device, dtype=torch.float32)
        scratch = torch.empty(B, device=wav.device, dtype=torch.int32)
        with torch.cuda.device(wav.device):
            check(lib().sbk_fbank_forward(self._h, ptr(wav), B, L, ptr(out), ptr(scratch), stream_ptr(wav.device)),
                  "sbk_fbank_forward")
        return out


class AsrEngine:
    """One repacked model on one GPU.  ``cfg`` keys: n_fft, hop, win (samples), n_mels, cnn_channels, input_size,
    d_model, nhead, num_encoder_layers, num_decoder_layers, d_ffn, vocab, kernel_size, attention_type
    ("RoPEMHA"|"RelPosMHAXL"|"hypermixing"|"regularMHA", hypermixing with the Conformer only, regularMHA with the Transformer
    only), decoder_activation ("gelu"|"relu"|"swish"), max_length; encoder_module ("conformer" (default) | "branchformer" |
    "transformer") with csgu_linear_units and branchformer_activation ("gelu" (default) | "relu"); cnn_blocks (2 (default),
    or 3: the Transformer recipes' front-end, cnn_channels (64, 64)); conformer_activation ("swish" (default) | "gelu": the
    Conformer's FFN and convolution-module activation).
    ``state``: {reference key with recipe prefix: CPU fp32 tensor}."""

    def __init__(self, cfg, state, device="cuda", parts=("fbank", "cnn", "encoder", "decoder")):
        self.cfg = dict(cfg)
        self.parts = tuple(parts)
        self.device = torch.device(device)
        c = _lib.sbk_asr_config()
        c.n_fft, c.hop, c.n_mels = cfg["n_fft"], cfg["hop"], cfg["n_mels"]
        c.cnn_c1, c.cnn_c2 = cfg["cnn_channels"]
        c.input_size, c.d_model, c.nhead = cfg["input_size"], cfg["d_model"], cfg["nhead"]
        c.num_encoder_layers, c.num_decoder_layers = cfg["num_encoder_layers"], cfg["num_decoder_layers"]
        c.d_ffn, c.vocab, c.kernel_size = cfg["d_ffn"], cfg["vocab"], cfg.get("kernel_size", 31)
        att = cfg["attention_type"]
        att_types = {"RoPEMHA": _lib.SBK_ATT_ROPE, "RelPosMHAXL": _lib.SBK_ATT_RELPOS, "hypermixing": _lib.SBK_ATT_HYPERMIX,
                     "regularMHA": _lib.SBK_ATT_REGULAR}
        if att not in att_types:
            raise NotImplementedError(f"attention_type={att!r}: only RoPEMHA, RelPosMHAXL, hypermixing and regularMHA are built")
        c.attention_type = att_types[att]
        dec_acts = {"gelu": _lib.SBK_ACT_GELU, "relu": _lib.SBK_ACT_RELU, "swish": _lib.SBK_ACT_SILU}
        if cfg.get("decoder_activation", "gelu") not in dec_acts:
            raise NotImplementedError(f"decoder_activation={cfg['decoder_activation']!r}: only gelu, relu and swish are built")
        c.decoder_activation = dec_acts[cfg.get("decoder_activation", "gelu")]
        c.max_len = cfg.get("max_length", 2500)
        enc_module = cfg.get("encoder_module", "conformer")
        if enc_module not in ("conformer", "branchformer", "transformer"):
            raise NotImplementedError(f"encoder_module={enc_module!r}: only conformer, branchformer and transformer are built")
        if enc_module == "transformer":
            c.encoder_module = _lib.SBK_ENC_TRANSFORMER
        c.cnn_blocks = cfg.get("cnn_blocks", 2)
        conformer_acts = {"swish": _lib.SBK_CONFORMER_ACT_SWISH, "gelu": _lib.SBK_CONFORMER_ACT_GELU}
        if cfg.get("conformer_activation", "swish") not in conformer_acts:
            raise NotImplementedError(f"conformer_activation={cfg['conformer_activation']!r}: only swish and gelu are built")
        c.conformer_activation = conformer_acts[cfg.get("conformer_activation", "swish")]
        if enc_module == "branchformer":
            c.encoder_module, c.csgu_linear_units = _lib.SBK_ENC_BRANCHFORMER, cfg["csgu_linear_units"]
            c.branchformer_activation = (_lib.SBK_ACT_GELU if cfg.get("branchformer_activation", "gelu") == "gelu"
                                         else _lib.SBK_ACT_RELU)
        lm = cfg.get("lm")  # dict(d_model, nhead, num_encoder_layers, d_ffn, activation) of a TransformerLM scorer
        if lm is not None:
            c.lm_d_model, c.lm_nhead, c.lm_layers, c.lm_d_ffn = lm["d_model"], lm["nhead"], lm["num_encoder_layers"], lm["d_ffn"]
            c.lm_activation = _lib.SBK_ACT_GELU if lm.get("activation", "gelu") == "gelu" else _lib.SBK_ACT_RELU
        c.parts = sum(_lib.SBK_PARTS[p] for p in self.parts)
        if cfg["num_decoder_layers"] == 0:
            c.parts &= ~_lib.SBK_PARTS["decoder"]
        st = {k: v.detach().float().contiguous().cpu() for k, v in state.items() if torch.is_tensor(v) and v.is_floating_point()}
        c.fbank_amin, c.fbank_top_db = float(cfg.get("fbank_amin", 0.0)), float(cfg.get("fbank_top_db", 0.0))  # 0 = defaults
        c.norm_eps = float(cfg.get("norm_eps", 0.0))
        if "fbank" in self.parts:  # a Fbank module's own tables when the caller passes them, else the recipe defaults
            if "fbank.window" not in st:
                st["fbank.window"] = stft_window(cfg["n_fft"], cfg["win"])
            if "fbank.mel_matrix" not in st:
                st["fbank.mel_matrix"] = mel_filter_matrix(cfg["n_mels"], cfg["n_fft"], cfg.get("sample_rate", 16000),
                                                           cfg.get("f_min", 0), cfg.get("f_max"))
        names = [k.encode() for k in st]
        arr = (_lib.sbk_tensor * len(st))()
        for i, (k, v) in enumerate(st.items()):
            arr[i].name, arr[i].data, arr[i].numel = names[i], v.data_ptr(), v.numel()
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_create(ctypes.byref(c), arr, len(st), ctypes.byref(self._h)), "sbk_asr_create")
        self._keep = (st, names, arr)

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                lib().sbk_asr_destroy(self._h)
                self._h = None
        except Exception:  # interpreter shutdown
            pass

    def clone(self):
        """A lane: shares the repacked weights, owns its workspace / decode graph (one per batch in flight)."""
        other = object.__new__(AsrEngine)
        other.cfg, other.device, other.parts, other._keep = self.cfg, self.device, self.parts, self._keep
        other._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_clone(self._h, ctypes.byref(other._h)), "sbk_asr_clone")
        return other

    def set_dynchunk(self, chunk_size=0, left_context_chunks=None):
        """DynChunkTrainConfig of the following encode calls (0 = full-context; left None = the whole past)."""
        check(lib().sbk_asr_set_dynchunk(self._h, int(chunk_size), -1 if left_context_chunks is None else int(left_context_chunks)),
              "sbk_asr_set_dynchunk")

    def set_poll_interval(self, every_n_steps):
        check(lib().sbk_asr_set_poll_interval(self._h, int(every_n_steps)), "sbk_asr_set_poll_interval")

    def lm_rescore(self, tokens, lens, temperature=1.0, pad_index=0):
        """TransformerLMRescorer.rescore_hyps device part: ``tokens`` [n, L] int32 CUDA (bos ... eos, pad-filled), ``lens`` [n]
        int32 CUDA -> [n] fp32 CUDA scores (sum of log p(token | prefix), pad column excluded from the normalisation)."""
        _lib.require_cuda(tokens, "AsrEngine.lm_rescore")
        tokens = tokens.to(torch.int32).contiguous()
        lens = lens.to(device=tokens.device, dtype=torch.int32).contiguous()
        n, L = tokens.shape
        scores = torch.empty(n, device=tokens.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_lm_rescore(self._h, ptr(tokens), ptr(lens), n, L, ctypes.c_float(temperature), int(pad_index),
                                           ptr(scores), self._sp()), "sbk_asr_lm_rescore")
        return scores

    def lm_forward(self, tokens):
        """TransformerLM.forward(src): ``tokens`` [n, s] integer CUDA (pad id 0) -> [n, s, vocab] fp32 CUDA logits, all
        positions in one whole-sequence pass (causal attention, key-padding mask on id 0)."""
        _lib.require_cuda(tokens, "AsrEngine.lm_forward")
        if tokens.dim() != 2:
            raise ValueError(f"AsrEngine.lm_forward: expected [n, s] token ids, got shape {tuple(tokens.shape)}")
        tokens = tokens.to(torch.int32).contiguous()
        n, s = tokens.shape
        logits = torch.empty(n, s, self.cfg["vocab"], device=tokens.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_lm_forward(self._h, ptr(tokens), n, s, ptr(logits), self._sp()), "sbk_asr_lm_forward")
        return logits

    def lm_step_logits(self, tokens):
        """The logits of ``lm_forward`` computed position by position on the KV-cached LM step (the path the beam search's
        scorer and the rescorer run): ``tokens`` [n, L] integer CUDA -> [n, L, vocab] fp32 CUDA.  For comparing the two."""
        _lib.require_cuda(tokens, "AsrEngine.lm_step_logits")
        tokens = tokens.to(torch.int32).contiguous()
        n, L = tokens.shape
        logits = torch.empty(n, L, self.cfg["vocab"], device=tokens.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_lm_step_logits(self._h, ptr(tokens), n, L, ptr(logits), self._sp()), "sbk_asr_lm_step_logits")
        return logits

    def set_decoder_tc_min_rows(self, rows):
        """Decode steps with >= rows live hypotheses use the wgmma GEMM for the decoder projections (default 64)."""
        check(lib().sbk_asr_set_decoder_tc_min_rows(self._h, int(rows)), "sbk_asr_set_decoder_tc_min_rows")

    def set_decoder_ln_fusion(self, on):
        check(lib().sbk_asr_set_decoder_ln_fusion(self._h, int(bool(on))), "sbk_asr_set_decoder_ln_fusion")

    def _sp(self):
        return stream_ptr(self.device)

    def num_frames(self, n_samples):
        a, b = ctypes.c_int(), ctypes.c_int()
        check(lib().sbk_asr_num_frames(self._h, n_samples, ctypes.byref(a), ctypes.byref(b)), "sbk_asr_num_frames")
        return a.value, b.value

    def cnn(self, feats):
        feats = feats.float().contiguous()
        B, T0, _ = feats.shape
        T1 = (T0 - 1) // 2 + 1
        T2 = (T1 - 1) // 2 + 1
        out = torch.empty(B, T2, self.cfg["input_size"], device=feats.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_cnn_forward(self._h, ptr(feats), B, T0, ptr(out), self._sp()), "sbk_asr_cnn_forward")
        return out

    def encode_from_cnn(self, src, wav_lens=None):
        src = src.float().contiguous()
        B, T, _ = src.shape
        out = torch.empty(B, T, self.cfg["d_model"], device=src.device, dtype=torch.float32)
        wl = wav_lens.float().contiguous().to(src.device) if wav_lens is not None else None
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_encode_from_cnn(self._h, ptr(src), ptr(wl), B, T, ptr(out), self._sp()),
                  "sbk_asr_encode_from_cnn")
        return out

    def stream_create(self, B, chunk_size, left_frames=None):
        """A chunk-by-chunk encoder stream of B streams on this engine's weights (left_frames None = the whole past)."""
        return EncoderStream(self, B, chunk_size, left_frames)

    def encode_feats(self, feats, wav_lens=None, want_cnn=False):
        feats = feats.float().contiguous()
        B, T0, _ = feats.shape
        T1 = (T0 - 1) // 2 + 1
        T2 = (T1 - 1) // 2 + 1
        out = torch.empty(B, T2, self.cfg["d_model"], device=feats.device, dtype=torch.float32)
        cnn = torch.empty(B, T2, self.cfg["input_size"], device=feats.device, dtype=torch.float32) if want_cnn else None
        wl = wav_lens.float().contiguous().to(feats.device) if wav_lens is not None else None
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_encode_feats(self._h, ptr(feats), ptr(wl), B, T0, ptr(cnn), ptr(out), self._sp()),
                  "sbk_asr_encode_feats")
        return (out, cnn) if want_cnn else out

    def greedy_from_enc(self, enc, wav_lens, max_steps, bos, eos, want_log_probs=False):
        enc = enc.float().contiguous()
        B, T, _ = enc.shape
        pred = torch.full((B, max(max_steps, 1)), eos, device=enc.device, dtype=torch.int32)
        score = torch.zeros(B, max(max_steps, 1), device=enc.device, dtype=torch.float32)
        lp = torch.empty(B, max_steps, self.cfg["vocab"], device=enc.device, dtype=torch.float32) if want_log_probs else None
        wl = wav_lens.float().contiguous().to(enc.device) if wav_lens is not None else None
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_greedy_from_enc(self._h, ptr(enc), ptr(wl), B, T, max_steps, bos, eos, ptr(pred), ptr(score),
                                                ptr(lp), ctypes.byref(done), self._sp()), "sbk_asr_greedy_from_enc")
        return pred, score, lp, done.value

    def ctc_head(self, enc=None, shape=None, want_log_probs=False, want_argmax=True):
        """log_softmax(ctc_lin(enc)) [B, T, V] and / or its per-frame arg-max [B, T] (EncoderASR + ctc_greedy_decode).
        ``enc`` None: use the encoder states the previous encode / transcribe call left in the workspace (``shape`` = (B, T))."""
        if enc is not None:
            enc = enc.float().contiguous()
            B, T, _ = enc.shape
        else:
            B, T = shape
        lp = torch.empty(B, T, self.cfg["vocab"], device=self.device, dtype=torch.float32) if want_log_probs else None
        idx = torch.empty(B, T, device=self.device, dtype=torch.int32) if want_argmax else None
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_ctc_head(self._h, ptr(enc), B, T, ptr(lp), ptr(idx), self._sp()), "sbk_asr_ctc_head")
        return lp, idx

    def decode_teacher_forced(self, tgt, enc, enc_len=None):
        """TransformerASR.decode device part: tgt [n, S] token ids, enc [n, T, d], enc_len [n] absolute -> [n, S, d] fp32."""
        enc = enc.float().contiguous()
        n, T, d = enc.shape
        tgt = tgt.to(device=enc.device, dtype=torch.int32).contiguous()
        S = tgt.shape[1]
        el = enc_len.to(device=enc.device, dtype=torch.int32).contiguous() if enc_len is not None else None
        out = torch.empty(n, S, d, device=enc.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_decode_teacher_forced(self._h, ptr(tgt), ptr(enc), ptr(el), n, S, T, ptr(out), self._sp()),
                  "sbk_asr_decode_teacher_forced")
        return out

    def beam_from_enc(self, enc, wav_lens, beam_size, max_steps, min_steps, bos, eos, temperature=1.0,
                      using_eos_threshold=True, eos_threshold=1.5, length_normalization=True, minus_inf=-1e20,
                      lm_weight=0.0, lm_temperature=1.0, ctc_weight=0.0, blank_index=-1, length_weight=0.0,
                      coverage_weight=0.0, coverage_threshold=0.5):
        """Device part of the beam search: returns the per-step history (tok, pred, score, lp) [steps, B*beam] on CPU."""
        enc = enc.float().contiguous()
        B, T, _ = enc.shape
        n_bh = B * beam_size
        S = max(max_steps, 1)
        tok = torch.zeros(S, n_bh, device=enc.device, dtype=torch.int32)
        pred = torch.zeros(S, n_bh, device=enc.device, dtype=torch.int32)
        score = torch.zeros(S, n_bh, device=enc.device, dtype=torch.float32)
        lp = torch.zeros(S, n_bh, device=enc.device, dtype=torch.float32)
        wl = wav_lens.float().contiguous().to(enc.device) if wav_lens is not None else None
        prm = _lib.sbk_beam_params(beam_size, max_steps, min_steps, bos, eos, temperature, int(bool(using_eos_threshold)),
                                   eos_threshold, int(bool(length_normalization)), minus_inf, lm_weight, lm_temperature, ctc_weight,
                                   int(blank_index), length_weight, coverage_weight, coverage_threshold)
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_beam_from_enc(self._h, ptr(enc), ptr(wl), B, T, ctypes.byref(prm), ptr(tok), ptr(pred),
                                              ptr(score), ptr(lp), ctypes.byref(done), self._sp()), "sbk_asr_beam_from_enc")
        n = done.value
        return tok[:n].cpu().long(), pred[:n].cpu().long(), score[:n].cpu(), lp[:n].cpu()

    def transcribe_greedy_dev(self, wav, wav_lens, max_steps, bos, eos, want_enc=False, pred=None, score=None):
        wav = wav.float().contiguous()
        B, L = wav.shape
        _, T = self.num_frames(L)
        if pred is None:
            pred = torch.full((B, max(max_steps, 1)), eos, device=wav.device, dtype=torch.int32)
        if score is None:
            score = torch.zeros(B, max(max_steps, 1), device=wav.device, dtype=torch.float32)
        enc = torch.empty(B, T, self.cfg["d_model"], device=wav.device, dtype=torch.float32) if want_enc else None
        wl = wav_lens.float().contiguous().to(wav.device) if wav_lens is not None else None
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_transcribe_greedy_dev(self._h, ptr(wav), ptr(wl), B, L, max_steps, bos, eos, ptr(enc),
                                                      ptr(pred), ptr(score), None, ctypes.byref(done), self._sp()),
                  "sbk_asr_transcribe_greedy_dev")
        return pred, score, enc, done.value

    def encode_wav(self, wav, wav_lens, out=None):
        """Fbank -> CMVN -> CNN -> encoder on device-resident wav (EncoderDecoderASR.encode_batch): [B, L] -> [B, T, d]."""
        wav = wav.float().contiguous()
        B, L = wav.shape
        _, T = self.num_frames(L)
        if out is None:
            out = torch.empty(B, T, self.cfg["d_model"], device=wav.device, dtype=torch.float32)
        wl = wav_lens.float().contiguous().to(wav.device)
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_transcribe_greedy_dev(self._h, ptr(wav), ptr(wl), B, L, 0, 0, 0, ptr(out), None, None, None,
                                                      ctypes.byref(done), self._sp()), "sbk_asr_transcribe_greedy_dev (encode)")
        return out

    def transcribe_greedy_group_dev(self, wavs, lens, max_steps, bos, eos, preds):
        """Decode coalescing: ``wavs`` / ``lens`` / ``preds`` are lists of G per-batch device tensors ([B, L] fp32,
        [B] fp32, [B, max_steps] int32).  The batches are encoded several at a time (up to 65536 encoder rows per pass, or
        one batch when a batch alone is larger), all G*B
        hypotheses are decoded together."""
        G = len(wavs)
        B, L = wavs[0].shape
        VP = ctypes.c_void_p * G
        w = VP(*[t.data_ptr() for t in wavs])
        r = VP(*[t.data_ptr() for t in lens])
        p = VP(*[t.data_ptr() for t in preds])
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_transcribe_greedy_group_dev(self._h, G, w, r, B, L, max_steps, bos, eos, p, ctypes.byref(done),
                                                            self._sp()), "sbk_asr_transcribe_greedy_group_dev")
        return done.value

    def transcribe_greedy_group_host_async(self, wavs_host, lens_host, max_steps, bos, eos, preds_host, preds_dev=None):
        """The group call from pinned HOST tensors (lists of G per-batch tensors): H2D copies, pipeline and D2H of the ids are
        enqueued on the current stream (copies on the engine's copy stream); the caller synchronises.  ``preds_dev``
        (optional list of device tensors) also keeps the ids on the device."""
        G = len(wavs_host)
        B, L = wavs_host[0].shape
        for t in itertools.chain(wavs_host, lens_host, preds_host):
            if t.is_cuda or not t.is_pinned() or not t.is_contiguous():
                raise RuntimeError("transcribe_greedy_group_host_async: host tensors must be pinned and contiguous")
        VP = ctypes.c_void_p * G
        w = VP(*[t.data_ptr() for t in wavs_host])
        r = VP(*[t.data_ptr() for t in lens_host])
        p = VP(*[t.data_ptr() for t in preds_host])
        pd = VP(*[t.data_ptr() for t in preds_dev]) if preds_dev is not None else None
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_transcribe_greedy_group_host_async(self._h, G, w, r, B, L, max_steps, bos, eos, p, pd,
                                                                   ctypes.byref(done), self._sp()),
                  "sbk_asr_transcribe_greedy_group_host_async")
        return done.value

    def transcribe_greedy_host_async(self, wav_host, lens_host, max_steps, bos, eos, pred_host):
        """Enqueue-only variant on the current stream (all tensors pinned, contiguous); caller synchronises."""
        B, L = wav_host.shape
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_transcribe_greedy_host_async(self._h, ptr(wav_host), ptr(lens_host), B, L, max_steps, bos, eos,
                                                             ptr(pred_host), None, ctypes.byref(done), self._sp()),
                  "sbk_asr_transcribe_greedy_host_async")
        return done.value

    def transcribe_greedy_host(self, wav_host, lens_host, max_steps, bos, eos, pred_host=None):
        """wav_host/lens_host/pred_host: CPU (ideally pinned) tensors; copies happen inside the call."""
        assert not wav_host.is_cuda
        wav_host = wav_host.float().contiguous()
        B, L = wav_host.shape
        if pred_host is None:  # pinned result buffer, cached per shape (pin_memory() costs more than the copy)
            cache = self.__dict__.setdefault("_pinned_pred", {})
            key = (B, max(max_steps, 1))
            if key not in cache:
                cache[key] = torch.empty(*key, dtype=torch.int32).pin_memory()
            pred_host = cache[key]
        pred_host.fill_(eos)
        lh = lens_host.float().contiguous() if lens_host is not None else None
        done = ctypes.c_int()
        with torch.cuda.device(self.device):
            check(lib().sbk_asr_transcribe_greedy_host(self._h, ptr(wav_host), ptr(lh), B, L, max_steps, bos, eos,
                                                       ptr(pred_host), None, ctypes.byref(done), self._sp()),
                  "sbk_asr_transcribe_greedy_host")
        return pred_host, done.value


class EncoderStream:
    """Per-layer left-context caches of B Conformer streams that advance together (sbk_asr_stream_*): ``encode_chunk`` maps
    the CNN output of one chunk [B, n <= chunk_size, input_size] to the encoder output [B, n, d_model] at a cost that does
    not grow with the stream's length."""

    def __init__(self, engine, B, chunk_size, left_frames=None):
        self.engine, self.B, self.chunk_size = engine, int(B), int(chunk_size)
        self.left_frames = None if left_frames is None else int(left_frames)
        self._s = ctypes.c_void_p()
        with torch.cuda.device(engine.device):
            check(lib().sbk_asr_stream_create(engine._h, self.B, self.chunk_size, -1 if left_frames is None else self.left_frames,
                                              ctypes.byref(self._s)), "sbk_asr_stream_create")

    def __del__(self):
        try:
            if getattr(self, "_s", None) and self._s.value:
                lib().sbk_asr_stream_destroy(self._s)
                self._s = None
        except Exception:  # interpreter shutdown
            pass

    def encode_chunk(self, src):
        src = src.float().contiguous()
        B, n, F = src.shape
        if B != self.B or F != self.engine.cfg["input_size"]:
            raise ValueError(f"EncoderStream: expected [{self.B}, n, {self.engine.cfg['input_size']}], got {list(src.shape)}")
        out = torch.empty(B, n, self.engine.cfg["d_model"], device=src.device, dtype=torch.float32)
        with torch.cuda.device(self.engine.device):
            check(lib().sbk_asr_stream_encode_chunk(self.engine._h, self._s, ptr(src), n, ptr(out), self.engine._sp()),
                  "sbk_asr_stream_encode_chunk")
        return out

    def reset(self):
        check(lib().sbk_asr_stream_reset(self._s), "sbk_asr_stream_reset")

    def cached_frames(self):
        n = ctypes.c_int()
        check(lib().sbk_asr_stream_context(self.engine._h, self._s, 0, None, None, ctypes.byref(n), None), "sbk_asr_stream_context")
        return n.value

    def layer_context(self, layer):
        """Copies of layer ``layer``'s caches: (kv [B, cached, 2 * d_model] fp16, per head [key | value]; carry
        [B, (kernel_size - 1) / 2, d_model] fp32, the depthwise-conv inputs of the last frames)."""
        d, K = self.engine.cfg["d_model"], self.engine.cfg.get("kernel_size", 31)
        n = self.cached_frames()
        dev = self.engine.device
        kv = torch.empty(self.B, n, 2 * d, device=dev, dtype=torch.float16)
        carry = torch.empty(self.B, (K - 1) // 2, d, device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib().sbk_asr_stream_context(self.engine._h, self._s, int(layer), ptr(kv), ptr(carry), None, self.engine._sp()),
                  "sbk_asr_stream_context")
        return kv, carry
