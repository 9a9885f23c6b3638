"""ctypes binding of libsbk.so (the C ABI declared in include/sbk.h).

There is NO fallback: if the shared library is missing, or a call fails, a RuntimeError is raised.
PyTorch is used only as plumbing (device memory, streams); the kernels live in csrc/.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsbk.so")

_lib = None


class sbk_tensor(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char_p), ("data", ctypes.c_void_p), ("numel", ctypes.c_int64)]


class sbk_asr_config(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int) for k in (
        "n_fft", "hop", "n_mels", "cnn_c1", "cnn_c2", "input_size", "d_model", "nhead", "num_encoder_layers",
        "num_decoder_layers", "d_ffn", "vocab", "kernel_size", "attention_type", "decoder_activation", "max_len",
        "parts", "lm_d_model", "lm_nhead", "lm_layers", "lm_d_ffn", "lm_activation")] + [
        (k, ctypes.c_float) for k in ("fbank_amin", "fbank_top_db", "norm_eps")] + [
        (k, ctypes.c_int) for k in ("encoder_module", "csgu_linear_units", "branchformer_activation", "cnn_blocks",
                                    "conformer_activation")]


class sbk_beam_params(ctypes.Structure):
    _fields_ = [("beam_size", ctypes.c_int), ("max_steps", ctypes.c_int), ("min_steps", ctypes.c_int),
                ("bos", ctypes.c_int), ("eos", ctypes.c_int), ("temperature", ctypes.c_float),
                ("using_eos_threshold", ctypes.c_int), ("eos_threshold", ctypes.c_float),
                ("length_normalization", ctypes.c_int), ("minus_inf", ctypes.c_float),
                ("lm_weight", ctypes.c_float), ("lm_temperature", ctypes.c_float),
                ("ctc_weight", ctypes.c_float), ("blank_index", ctypes.c_int), ("length_weight", ctypes.c_float),
                ("coverage_weight", ctypes.c_float), ("coverage_threshold", ctypes.c_float)]


class sbk_ctc_beam_params(ctypes.Structure):
    _fields_ = [("blank", ctypes.c_int), ("beam_size", ctypes.c_int), ("prune_history", ctypes.c_int),
                ("token_prune_min_logp", ctypes.c_float), ("beam_prune_logp", ctypes.c_float),
                ("blank_skip_logp", ctypes.c_float)]


class sbk_ctc_prefix_beam_params(ctypes.Structure):
    _fields_ = [("blank", ctypes.c_int), ("beam_size", ctypes.c_int), ("prune_history", ctypes.c_int),
                ("token_prune_min_logp", ctypes.c_float), ("blank_skip_logp", ctypes.c_float),
                ("beam_prune_logp", ctypes.c_double)]


SBK_ATT_ROPE, SBK_ATT_RELPOS, SBK_ATT_HYPERMIX, SBK_ATT_REGULAR = 0, 1, 2, 3
SBK_ACT_RELU, SBK_ACT_GELU, SBK_ACT_SILU = 0, 1, 2
SBK_ENC_CONFORMER, SBK_ENC_BRANCHFORMER, SBK_ENC_TRANSFORMER = 0, 1, 2
SBK_CONFORMER_ACT_SWISH, SBK_CONFORMER_ACT_GELU = 0, 1
SBK_PARTS = {"fbank": 1, "cnn": 2, "encoder": 4, "decoder": 8, "lm": 16}

# every symbol include/sbk.h declares (tests check the library exports all of them)
EXPORTS = [
    "sbk_last_error", "sbk_version", "sbk_launch_count", "sbk_gemm_profile_enable", "sbk_gemm_profile_read", "sbk_fbank_create", "sbk_fbank_destroy", "sbk_fbank_num_frames",
    "sbk_fbank_forward", "sbk_input_norm_global", "sbk_input_norm_sentence", "sbk_gemm_f16_test", "sbk_gemm_f16_resid_test",
    "sbk_gemm_epilogue_test", "sbk_ctc_prefix_test", "sbk_csgu_test", "sbk_hypermix_test",
    "sbk_encoder_attention_test", "sbk_dwconv_test", "sbk_dwconv_act_test",
    "sbk_asr_create", "sbk_asr_destroy", "sbk_asr_num_frames", "sbk_asr_cnn_forward", "sbk_asr_encode_from_cnn",
    "sbk_asr_encode_feats", "sbk_asr_greedy_from_enc", "sbk_asr_transcribe_greedy_dev",
    "sbk_asr_transcribe_greedy_host", "sbk_asr_transcribe_greedy_host_async", "sbk_asr_clone",
    "sbk_asr_set_poll_interval", "sbk_asr_beam_from_enc", "sbk_asr_set_decoder_ln_fusion", "sbk_asr_transcribe_greedy_group_dev",
    "sbk_asr_set_decoder_tc_min_rows", "sbk_asr_lm_rescore", "sbk_asr_transcribe_greedy_group_host_async", "sbk_asr_decode_teacher_forced", "sbk_asr_ctc_head", "sbk_rows_argmax_f32", "sbk_asr_set_dynchunk",
    "sbk_asr_lm_forward", "sbk_asr_lm_step_logits", "sbk_ctc_beam_workspace_bytes", "sbk_ctc_beam_search",
    "sbk_ctc_prefix_beam_workspace_bytes", "sbk_ctc_prefix_beam_search",
    "sbk_transducer_create", "sbk_transducer_destroy", "sbk_transducer_info", "sbk_transducer_greedy",
    "sbk_transducer_beam",
    "sbk_asr_stream_create", "sbk_asr_stream_encode_chunk", "sbk_asr_stream_reset", "sbk_asr_stream_destroy",
    "sbk_asr_stream_context", "sbk_asr_stream_encode_chunk_strided", "sbk_asr_stream_frontend_chunk", "sbk_stream_qkv_test", "sbk_step_proj_test", "sbk_dec_attention_test",
    "sbk_beam_step_test", "sbk_coverage_score_test", "sbk_xatt_fold_test", "sbk_lm_causal_attention_test",
]


def lib():
    """Load libsbk.so once. Raises if it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: the sm_90a CUDA library is required (no CPU fallback). "
                "Build it with `make -C speechbrain_b200/csrc` or `__graft_entry__.build()`.")
        L = ctypes.CDLL(LIB_PATH)
        L.sbk_last_error.restype = ctypes.c_char_p
        for name in EXPORTS:
            getattr(L, name)  # AttributeError if the ABI is incomplete
        for name in EXPORTS:
            if name not in ("sbk_last_error", "sbk_fbank_destroy", "sbk_asr_destroy", "sbk_launch_count",
                            "sbk_gemm_profile_enable", "sbk_transducer_destroy", "sbk_asr_stream_destroy"):
                getattr(L, name).restype = ctypes.c_int
        L.sbk_launch_count.restype = ctypes.c_longlong
        L.sbk_gemm_profile_enable.restype = None
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError(f"libsbk: {what} failed ({rc}): {lib().sbk_last_error().decode()}")


def ptr(t):
    """Raw address of a (contiguous) torch tensor, or NULL."""
    if t is None:
        return ctypes.c_void_p(0)
    assert t.is_contiguous(), "libsbk needs contiguous tensors"
    return ctypes.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"{what}: expected a CUDA tensor (speechbrain_b200 has no CPU path)")
