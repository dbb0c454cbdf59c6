"""ctypes binding of libmvb200.so (include/mvb200.h).  There is no fallback: if the CUDA library is
missing or does not export the declared ABI, importing the engine fails loudly."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("MVB200_LIB") or os.path.join(_HERE, "libmvb200.so")   # override: A/B two builds on one box

MVB_KV_BF16, MVB_KV_FP32, MVB_KV_FP8 = 0, 1, 2
MVB_S1_MAX_VOICES = 16                             # voices of one stage-1 engine, the base included
MVB_OK, MVB_ERR_CUDA, MVB_ERR_ARG, MVB_ERR_PROMPT_TOO_LONG, MVB_ERR_UNSUPPORTED = 0, 1, 2, 3, 4
GLOBAL_TENSORS, LAYER_TENSORS = 5, 7
# `options` bits of the engine configs (include/mvb200.h): reference and identity paths, fixed at create time
MVB_S1_NO_ROWS_PATH, MVB_S1_NO_RESIDENT, MVB_S1_UNFUSED_SAMPLER, MVB_S1_TRACE = 0x1, 0x2, 0x4, 0x8
MVB_S2_EAGER = 0x1
MVB_S2_NORM_RMS, MVB_S2_NORM_LAYER = 0, 1          # mvb_s2_arch.norm
MVB_S2_MLP_SWIGLU, MVB_S2_MLP_GELU = 0, 1          # mvb_s2_arch.mlp
MVB_S1_NORM_RMS, MVB_S1_NORM_LAYER = 0, 1          # mvb_s1_arch.norm
MVB_S1_MLP_SWIGLU, MVB_S1_MLP_GELU = 0, 1          # mvb_s1_arch.mlp
MVB_MBD_CUDA_CORES, MVB_MBD_ONE_STREAM = 0x1, 0x2
SPK_MAX_BATCH, RESAMPLE_MAX_TAPS = 32, 16384      # MVB_SPK_MAX_BATCH, MVB_RESAMPLE_MAX_TAPS


class S1Config(C.Structure):
    _fields_ = [("n_layer", C.c_int32), ("n_head", C.c_int32), ("head_dim", C.c_int32), ("dim", C.c_int32),
                ("intermediate", C.c_int32), ("vocab", C.c_int32), ("block_size", C.c_int32),
                ("spk_dim", C.c_int32), ("norm_eps", C.c_float), ("max_utts", C.c_int32),
                ("kv_dtype", C.c_int32), ("max_new", C.c_int32), ("options", C.c_int32)]


class Sampling(C.Structure):
    _fields_ = [("guidance_scale", C.c_float), ("temperature", C.c_float), ("top_p", C.c_float),
                ("top_k", C.c_int32), ("end_of_audio", C.c_int32), ("seed", C.c_uint64)]


class S2Config(C.Structure):
    _fields_ = [("n_layer", C.c_int32), ("n_head", C.c_int32), ("n_embd", C.c_int32), ("hidden", C.c_int32),
                ("block_size", C.c_int32), ("n_in", C.c_int32), ("vocab_in", C.c_int32 * 8), ("n_out", C.c_int32),
                ("vocab_out", C.c_int32 * 8), ("spk_dim", C.c_int32), ("norm_eps", C.c_float), ("max_batch", C.c_int32),
                ("options", C.c_int32)]


class S1Arch(C.Structure):
    _fields_ = [("norm", C.c_int32), ("mlp", C.c_int32), ("bias", C.c_int32)]


class S2Arch(C.Structure):
    _fields_ = [("norm", C.c_int32), ("mlp", C.c_int32), ("bias", C.c_int32)]


class VocConfig(C.Structure):
    _fields_ = [("n_q", C.c_int32), ("hidden", C.c_int32), ("n_filters", C.c_int32), ("n_ratios", C.c_int32),
                ("ratios", C.c_int32 * 8), ("kernel", C.c_int32), ("res_kernel", C.c_int32), ("last_kernel", C.c_int32),
                ("compress", C.c_int32), ("max_frames", C.c_int32)]


class EncConfig(C.Structure):
    _fields_ = VocConfig._fields_


class MbdConfig(C.Structure):
    _fields_ = [("n_models", C.c_int32), ("chin", C.c_int32), ("hidden", C.c_int32), ("depth", C.c_int32), ("res_blocks", C.c_int32),
                ("norm_groups", C.c_int32), ("kernel", C.c_int32), ("stride", C.c_int32), ("growth", C.c_float),
                ("emb_all_layers", C.c_int32), ("codec_dim", C.c_int32), ("num_steps", C.c_int32), ("n_calls", C.c_int32),
                ("noise_scale", C.c_float), ("clip", C.c_float), ("proc_bands", C.c_int32), ("proc_taps", C.c_int32),
                ("eq_bands", C.c_int32), ("eq_taps", C.c_int32), ("max_samples", C.c_int32), ("options", C.c_int32)]


class SpkConfig(C.Structure):
    _fields_ = [("n_mels", C.c_int32), ("hidden", C.c_int32), ("n_layers", C.c_int32), ("emb", C.c_int32), ("n_fft", C.c_int32),
                ("hop", C.c_int32), ("partial_frames", C.c_int32), ("max_samples", C.c_int32)]


# name -> (restype, argtypes); also the list the symbol-export test checks against include/mvb200.h
SIGNATURES = {
    "mvb_abi_version": (C.c_int, []),
    "mvb_last_error": (C.c_char_p, []),
    "mvb_s1_kv_bytes": (C.c_size_t, [C.POINTER(S1Config)]),
    "mvb_s1_workspace_bytes": (C.c_size_t, [C.POINTER(S1Config)]),
    "mvb_s1_create_ex": (C.c_int, [C.POINTER(S1Config), C.POINTER(S1Arch), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64),
                                   C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "mvb_s1_create": (C.c_int, [C.POINTER(S1Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                C.c_void_p, C.POINTER(C.c_void_p)]),
    "mvb_s1_destroy": (C.c_int, [C.c_void_p]),
    "mvb_s1_set_speaker": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_s1_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                 C.c_void_p]),
    "mvb_s1_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(Sampling), C.c_void_p, C.c_uint64, C.c_void_p,
                                C.c_void_p, C.c_void_p]),
    "mvb_s1_generate": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(Sampling),
                                  C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_s1_decode": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "mvb_s1_begin": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(Sampling), C.c_void_p,
                               C.c_void_p, C.c_void_p]),
    "mvb_s1_fetch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32),
                               C.POINTER(C.c_int32), C.c_void_p]),
    "mvb_s1_admit": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(Sampling), C.c_int32,
                               C.c_void_p, C.c_void_p]),
    "mvb_s1_release": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "mvb_s1_poll": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_s1_admit_guided": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(Sampling),
                                      C.c_float, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_s1_sample_guided": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(Sampling), C.c_float, C.c_void_p, C.c_uint64, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "mvb_s1_step_logits": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_s1_launch_count": (C.c_uint64, [C.c_void_p]),
    "mvb_s1_add_voice": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int32, C.POINTER(C.c_uint64), C.c_int32,
                                   C.POINTER(C.c_int32)]),
    "mvb_s1_set_voice": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32]),
    "mvb_s1_int4_workspace_bytes": (C.c_size_t, [C.POINTER(S1Config)]),
    "mvb_s1_create_int4": (C.c_int, [C.POINTER(S1Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                     C.c_void_p, C.POINTER(C.c_void_p)]),
    "mvb_s1_int8_workspace_bytes": (C.c_size_t, [C.POINTER(S1Config)]),
    "mvb_s1_create_int8": (C.c_int, [C.POINTER(S1Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                     C.c_void_p, C.POINTER(C.c_void_p)]),
    "mvb_s1_fp8_workspace_bytes": (C.c_size_t, [C.POINTER(S1Config)]),
    "mvb_s1_create_fp8": (C.c_int, [C.POINTER(S1Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                    C.c_void_p, C.POINTER(C.c_void_p)]),
    "mvb_s2_workspace_bytes": (C.c_size_t, [C.POINTER(S2Config)]),
    "mvb_s2_create": (C.c_int, [C.POINTER(S2Config), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                C.POINTER(C.c_void_p)]),
    "mvb_s2_create_ex": (C.c_int, [C.POINTER(S2Config), C.POINTER(S2Arch), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64),
                                   C.c_void_p, C.POINTER(C.c_void_p)]),
    "mvb_s2_destroy": (C.c_int, [C.c_void_p]),
    "mvb_s2_forward": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_void_p,
                                 C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_voc_workspace_bytes": (C.c_size_t, [C.POINTER(VocConfig)]),
    "mvb_voc_create": (C.c_int, [C.POINTER(VocConfig), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                 C.POINTER(C.c_void_p)]),
    "mvb_voc_destroy": (C.c_int, [C.c_void_p]),
    "mvb_voc_decode_latent": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_voc_decode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_voc_batch_workspace_bytes": (C.c_size_t, [C.POINTER(VocConfig), C.c_int32, C.c_int32]),
    "mvb_voc_decode_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p]),
    "mvb_voc_decode_latent_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_int32,
                                              C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_enc_workspace_bytes": (C.c_size_t, [C.POINTER(EncConfig)]),
    "mvb_enc_create": (C.c_int, [C.POINTER(EncConfig), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                 C.POINTER(C.c_void_p)]),
    "mvb_enc_destroy": (C.c_int, [C.c_void_p]),
    "mvb_enc_encode": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_enc_batch_workspace_bytes": (C.c_size_t, [C.POINTER(EncConfig), C.c_int32, C.c_int32]),
    "mvb_enc_encode_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_mbd_workspace_bytes": (C.c_size_t, [C.POINTER(MbdConfig)]),
    "mvb_mbd_create": (C.c_int, [C.POINTER(MbdConfig), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                 C.POINTER(C.c_void_p)]),
    "mvb_mbd_destroy": (C.c_int, [C.c_void_p]),
    "mvb_mbd_tokens_to_wav": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_uint64,
                                        C.c_void_p, C.c_void_p]),
    "mvb_spk_workspace_bytes": (C.c_size_t, [C.POINTER(SpkConfig)]),
    "mvb_spk_create": (C.c_int, [C.POINTER(SpkConfig), C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64), C.c_void_p,
                                 C.POINTER(C.c_void_p)]),
    "mvb_spk_destroy": (C.c_int, [C.c_void_p]),
    "mvb_spk_mel": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_spk_embed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_resample_batch": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                     C.c_void_p]),
    "mvb_spk_batch_workspace_bytes": (C.c_size_t, [C.POINTER(SpkConfig), C.c_int32, C.c_int64]),
    "mvb_spk_trim_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_int64,
                                     C.c_void_p, C.c_void_p]),
    "mvb_spk_embed_batch": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_int32, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_audio_post_workspace_bytes": (C.c_size_t, [C.c_int32]),
    "mvb_audio_post": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p]),
    "mvb_audio_post_batch_workspace_bytes": (C.c_size_t, [C.c_int32, C.c_int32]),
    "mvb_audio_post_batch": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_float, C.c_int32, C.c_void_p,
                                       C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_linear": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_float,
                             C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    # test / debug hooks (declared in the header as such)
    "mvb_s1_fetch_sampled": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]),
    "mvb_s1_trace_fetch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "mvb_gemm_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                C.c_void_p, C.c_float, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "mvb_mbd_conv_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "mvb_mbd_op_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_uint64,
                                  C.c_void_p]),
    "mvb_mbd_unet_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                    C.c_void_p]),
    "mvb_s2_attn_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_w4_gemv_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "mvb_w4_dequant_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_w8_gemv_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "mvb_w8_gemm_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                   C.c_int32, C.c_int32, C.c_void_p, C.c_float, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                   C.c_void_p]),
    "mvb_w8_widen_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_f8_gemv_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_float, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "mvb_f8_widen_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "mvb_s1_kv_f8_store_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_s1_arch_gemv_test": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                        C.c_float, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "mvb_s2_sample_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p]),
    "mvb_s2_embed_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_s2_linear_test": (C.c_int, [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.c_int32,
                                     C.c_void_p, C.c_int32, C.c_void_p]),
    "mvb_voc_op_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_enc_op_test": (C.c_int, [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                  C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "mvb_audio_post_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_int32, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.c_void_p]),
    "mvb_spk_op_test": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p,
                                  C.c_void_p]),
    "mvb_test_set_sm_limit": (C.c_int, [C.c_int32]),
}
ABI_VERSION = 3

_lib = None


class MvbError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the library once; raise (never fall back) when it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise MvbError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(libmvb200 has no CPU or PyTorch fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
        fn.restype = res
        fn.argtypes = args
    if lib.mvb_abi_version() != ABI_VERSION:
        raise MvbError("libmvb200 ABI version mismatch")
    _lib = lib
    return lib


def check(rc: int) -> None:
    """Map C status codes to the exceptions the reference raises (SURVEY.md 8b error convention)."""
    if rc == MVB_OK:
        return
    msg = load().mvb_last_error().decode("utf-8", "replace")
    if rc == MVB_ERR_PROMPT_TOO_LONG:
        raise ValueError("Prompt is too long to generate more tokens")  # fast_inference_utils.py:203-204
    if rc == MVB_ERR_ARG:
        raise ValueError(msg)
    raise MvbError(msg)
