"""ctypes binding of libfs2b200.so (include/fs2_b200.h).

The library is the product path.  There is no CPU or PyTorch fallback: if the shared
object is missing or a call fails, the error is raised to the caller.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfs2b200.so")

FS2_DUR_I64, FS2_DUR_F32, FS2_DUR_I32 = 0, 1, 2
FS2_PER_UTTERANCE = 1      # flag of fs2_encode_ex / fs2_decode_ex
MATH_FP32, MATH_TF32, MATH_3XTF32, MATH_F16 = 0, 1, 2, 3
# "3xtf32" is the historical name of the error-compensated mode (now three f16 products per term); "3xf16" is an alias
MATH_MODES = {"fp32": MATH_FP32, "tf32": MATH_TF32, "3xtf32": MATH_3XTF32, "3xf16": MATH_3XTF32, "f16": MATH_F16}


class Fs2Error(RuntimeError):
    pass


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "idim", "odim", "adim", "aheads", "elayers", "eunits", "ddim", "dlayers", "dunits", "ffn_kernel",
        "pred_layers", "pred_chans", "pred_kernel", "postnet_layers", "postnet_chans", "postnet_filts",
        "n_bins", "pe_len", "math_mode")]


class WeightDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("ndim", C.c_int32), ("shape", C.c_int64 * 4),
                ("dtype", C.c_int32)]


class VocoderConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_fft", "hop", "win_length", "n_mels", "math_mode")]


class FeaturesConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("sample_rate", "n_fft", "hop", "win_length", "n_mels", "math_mode")] + \
               [(n, C.c_double) for n in ("f0_floor", "f0_ceil", "channels_in_octave", "allowed_range")]


FS2_FEAT_BAD_LENGTH, FS2_FEAT_RANGE = 1, 2   # bits of fs2_mel_energy's / fs2_dio's device status word
FS2_VOC_BAD_LENGTH, FS2_VOC_RANGE = 1, 2     # bits of fs2_griffin_lim's / fs2_mel_magnitude's device status word
FS2_MELGAN_BAD_LENGTH, FS2_MELGAN_RANGE = 1, 2   # bits of fs2_melgan's device status word
FS2_MELGAN_BAD_START = 4                          # and of fs2_melgan_window's
FS2_WAVEGLOW_BAD_LENGTH, FS2_WAVEGLOW_RANGE = 1, 2   # bits of fs2_waveglow's device status word
FS2_WAVEGLOW_BAD_START = 4                           # and of fs2_waveglow_window's
FS2_HIFIGAN_BAD_LENGTH, FS2_HIFIGAN_RANGE = 1, 2     # bits of fs2_hifigan's device status word
FS2_HIFIGAN_BAD_START = 4                            # and of fs2_hifigan_window's
FS2_HIFIGAN_MAX_UPSAMPLES, FS2_HIFIGAN_MAX_KERNELS = 8, 8
FS2_BIGVGAN_BAD_LENGTH, FS2_BIGVGAN_RANGE, FS2_BIGVGAN_BAD_START = 1, 2, 4   # bits of fs2_bigvgan's / fs2_bigvgan_window's status word
FS2_BIGVGAN_SNAKE, FS2_BIGVGAN_SNAKEBETA = 0, 1
FS2_ISTFTNET_BAD_LENGTH, FS2_ISTFTNET_RANGE, FS2_ISTFTNET_BAD_START = 1, 2, 4   # bits of fs2_istftnet's / fs2_istftnet_window's status word
FS2_EVAL_BAD_LENGTH, FS2_EVAL_NONFINITE = 1, 2   # bits of fs2_mcd_dtw's / fs2_path_prosody's status word
FS2_RS_BAD_LENGTH, FS2_RS_NONFINITE = 1, 2       # bits of fs2_resample's status word
FS2_WORLD_BAD_LENGTH, FS2_WORLD_NONFINITE, FS2_WORLD_F0_RANGE = 1, 2, 4   # bits of fs2_stonemask's / fs2_cheaptrick's / fs2_mcep's
FS2_ALIGN_BAD_LENGTH, FS2_ALIGN_INFEASIBLE, FS2_ALIGN_NONFINITE = 1, 2, 4   # bits of the fs2_align_* status word
FS2_ALIGN_DIM, FS2_ALIGN_MAX_T = 80, 1024
FS2_RESAMPLE_TABLE = 32769                        # entries of the resampling filter's right wing
FS2_PLAN_BAD_ILENS,FS2_PLAN_BAD_CONTROL, FS2_PLAN_OVERFLOW = 1, 2, 4   # bits of fs2_length_plan_cap's status word
FS2_PLAN_BAD_SPEAKER = 8                          # and of fs2_length_plan_cap_spk's
FS2_SPEMB_NONFINITE = 16                          # fs2_spemb_project's / fs2_encode_spemb's status bit, and fs2_length_plan_cap_spemb's
FS2_SPEMB_MAX_DIM = 4096                          # the largest speaker-embedding width D
FS2_ECAPA_BAD_LENGTH, FS2_ECAPA_RANGE = 1, 2       # bits of fs2_ecapa's / fs2_op_ecapa_stage's status word
FS2_ECAPA_MAX_BLOCKS, FS2_ECAPA_MAX_SCALE = 8, 16
FS2_SYNTH_VOC_SHIFT = 8                          # fs2_synth_status: the vocoder's bits sit this far up in the word


class HiFiGANConfig(C.Structure):
    _fields_ = [("resblock", C.c_int32), ("num_upsamples", C.c_int32),
                ("upsample_rates", C.c_int32 * FS2_HIFIGAN_MAX_UPSAMPLES),
                ("upsample_kernel_sizes", C.c_int32 * FS2_HIFIGAN_MAX_UPSAMPLES),
                ("upsample_initial_channel", C.c_int32), ("num_kernels", C.c_int32),
                ("resblock_kernel_sizes", C.c_int32 * FS2_HIFIGAN_MAX_KERNELS), ("num_dilations", C.c_int32),
                ("resblock_dilation_sizes", (C.c_int32 * 4) * FS2_HIFIGAN_MAX_KERNELS)]


class BigVGANConfig(C.Structure):
    _fields_ = [("gen", HiFiGANConfig), ("activation", C.c_int32), ("snake_logscale", C.c_int32), ("use_tanh_at_final", C.c_int32),
                ("use_bias_at_final", C.c_int32)]


class ISTFTNetConfig(C.Structure):
    _fields_ = [("gen", HiFiGANConfig), ("istft_n_fft", C.c_int32), ("istft_hop", C.c_int32)]


class WorldConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("sample_rate", "fft_size", "order")] + \
               [(n, C.c_double) for n in ("frame_period", "q1", "alpha")]


class ECAPAConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("n_mels", "channels", "n_blocks", "scale", "se_channels", "attention_channels",
                                         "mfa_channels", "lin_neurons", "global_context")] + \
               [("kernel_sizes", C.c_int32 * (FS2_ECAPA_MAX_BLOCKS + 2)), ("dilations", C.c_int32 * (FS2_ECAPA_MAX_BLOCKS + 2))]


class NoamAdamHp(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("rate_scale", "warmup_pow", "beta1", "beta2", "eps")]


class RowNormDesc(C.Structure):
    """fs2_row_norm_desc: the row LayerNorm and its fusions (fs2_op_row_norm); unset pointers are NULL, unset ints 0."""
    _fields_ = [("x", C.c_void_p), ("ldx", C.c_int32), ("resid", C.c_void_p), ("ldr", C.c_int32),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("eps", C.c_float), ("rows", C.c_int64), ("C", C.c_int32),
                ("out", C.c_void_p), ("ldo", C.c_int32), ("relu_after", C.c_int32),
                ("pe", C.c_void_p), ("alpha", C.c_void_p), ("L", C.c_int32),
                ("head_w", C.c_void_p), ("head_b", C.c_void_p), ("head_out", C.c_void_p), ("dur_out", C.c_void_p),
                ("head_scale", C.c_void_p), ("lens", C.c_void_p), ("split_out", C.c_void_p), ("split_lo", C.c_int32),
                ("spk_table", C.c_void_p), ("spk", C.c_void_p), ("n_spk", C.c_int32), ("spk_L", C.c_int32)]


FS2_OPTIM_CHUNK = 65536                           # elements per chunk of the optimizer's parameter table
_P, _I, _F, _L, _SZ = C.c_void_p, C.c_int, C.c_float, C.c_int64, C.c_size_t

# name -> argtypes; every function returns int except the three noted below
SIGNATURES = {
    "fs2_create": [C.POINTER(_P), C.POINTER(Config), _I],
    "fs2_set_math_mode": [_P, _I],
    "fs2_profile_enable": [_P, _I],
    "fs2_profile_classes": [],
    "fs2_profile_read": [_P, C.POINTER(C.c_double), C.POINTER(_L), C.POINTER(C.c_double), C.POINTER(C.c_double)],
    "fs2_load_weights": [_P, C.POINTER(WeightDesc), _I, _P],
    "fs2_workspace_bytes": [_P, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_encode": [_P, _P, _P, _I, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_encode_ex": [_P, _P, _P, _I, _I, _P, _P, _P, _P, _SZ, _I, _P],
    "fs2_encode_spk": [_P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _SZ, _I, _P],
    "fs2_encode_spemb": [_P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _SZ, _I, _P, _P, _P],
    "fs2_length_plan": [_P, _I, _P, _F, _I, _I, _I, _P, _P, _P, _P],
    "fs2_length_gather": [_P, _P, _P, _I, _I, _I, _P, _I, _P],
    "fs2_length_plan_ex": [_P, _I, _P, _F, _P, _I, _I, _I, _P, _P, _P, _P, _P],
    "fs2_length_gather_ex": [_P, _P, _P, _I, _I, _I, _P, _I, _P, _P, _P],
    "fs2_length_plan_cap": [_P, _I, _P, _P, _P, _I, _I, _L, _P, _P, _P, _P, _P, _P],
    "fs2_length_plan_cap_spk": [_P, _I, _P, _P, _P, _P, _I, _I, _I, _L, _P, _P, _P, _P, _P, _P],
    "fs2_length_plan_cap_spemb": [_P, _I, _P, _P, _P, _P, _I, _P, _I, _I, _L, _P, _P, _P, _P, _P, _P],
    "fs2_synth_status": [_P, _P, _P, _I, _I, _P, _P, _P],
    "fs2_decode": [_P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_decode_ex": [_P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _SZ, _I, _P],
    "fs2_decode_ctl": [_P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _SZ, _I, _P],
    "fs2_masked_losses": [_P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P],
    "fs2_bucketize": [_P, _P, _I, _L, _P, _P],
    "fs2_one_hot": [_P, _L, _I, _P, _P],
    "fs2_op_tap_gemm": [_I, _P, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P],
    "fs2_op_tap_gemm_ex": [_I, _P, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P, _I, _I, _P, _I, _P],
    "fs2_op_tap_gemm_dil": [_I, _P, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P, _I, _I, _P, _I, _I, _P],
    "fs2_op_attention": [_I, _P, _P, _I, _I, _I, _I, _P, _P],
    "fs2_op_attention_planes": [_I, _P, _P, _I, _P, _I, _I, _I, _I, _P, _P, _P],
    "fs2_op_gemm_layernorm": [_I, _P, _L, _I, _I, _P, _P, _P, _P, _P, _F, _P, _P, _P],
    "fs2_op_layernorm": [_P, _P, _P, _P, _F, _L, _I, _P, _P],
    "fs2_op_row_norm": [C.POINTER(RowNormDesc), _P],
    "fs2_op_row_norm_spemb": [C.POINTER(RowNormDesc), _P, _P],
    "fs2_op_variance_embed_add": [_P, _P, _P, _P, _P, _I, _P, _P, _P, _P, _L, _I, _P, _P, _I, _P, _P, _P, _I, _P],
    "fs2_dropout_mask": [_P, _L, _F, C.c_uint64, C.c_uint64, _P],
    "fs2_dropout_apply": [_P, _P, _F, _P, _L, _P],
    "fs2_act_backward": [_P, _P, _I, _P, _L, _P],
    "fs2_relu": [_P, _P, _L, _P],
    "fs2_add": [_P, _P, _P, _L, _P],
    "fs2_colsum": [_P, _L, _I, _P, _P],
    "fs2_conv_forward": [_P, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P],
    "fs2_conv_dgrad": [_P, _I, _I, _I, _P, _I, _I, _P, _P, _P],
    "fs2_conv_wgrad": [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P],
    "fs2_conv_forward_ex": [_P, _I, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P, _I, _P],
    "fs2_conv_dgrad_ex": [_P, _I, _I, _I, _P, _I, _I, _P, _P, _I, _P],
    "fs2_conv_wgrad_tc_ws_bytes": [_I, _I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_conv_wgrad_tc": [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_layernorm_backward": [_P, _P, _P, _F, _L, _I, _P, _P, _P, _P],
    "fs2_batchnorm_train": [_P, _L, _I, _P, _P, _F, _F, _I, _P, _P, _P, _P, _P, _P],
    "fs2_batchnorm_backward": [_P, _P, _P, _P, _F, _L, _I, _P, _P, _P, _P, _P],
    "fs2_bgemm": [_P, _L, _L, _L, _L, _P, _L, _L, _L, _L, _P, _L, _L, _L, _L, _I, _I, _I, _I, _I, _F, _P],
    "fs2_attn_softmax": [_P, _P, _P, _F, _I, _I, _I, _P, _P, _P],
    "fs2_attn_softmax_backward": [_P, _P, _P, _F, _I, _I, _I, _P, _P],
    "fs2_attn_train_ws_bytes": [_I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_attn_train_forward": [_P, _P, _P, _P, _I, _I, _I, _I, _F, _P, C.c_uint64, C.c_uint64, _P, _P, _P, _SZ, _P],
    "fs2_attn_train_backward": [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P, C.c_uint64, C.c_uint64, _P, _P, _P, _P, _SZ, _P],
    "fs2_embed_posenc": [_P, _P, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P],
    "fs2_embed_backward": [_P, _P, _P, _I, _I, _I, _I, _P, _P, _P],
    "fs2_posenc_add": [_P, _P, _P, _I, _I, _I, _P, _P],
    "fs2_speaker_add": [_P, _P, _P, _I, _I, _I, _I, _P, _P],
    "fs2_speaker_add_backward_ws_bytes": [_I, _I, C.POINTER(_SZ)],
    "fs2_speaker_add_backward": [_P, _P, _I, _I, _I, _I, _P, _P, _SZ, _P],
    "fs2_spemb_project": [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P],
    "fs2_spemb_project_backward": [_P, _P, _I, _I, _I, _P, _P, _P],
    "fs2_onehot_linear_forward": [_P, _P, _P, _P, _L, _I, _I, _P, _P],
    "fs2_onehot_linear_backward": [_P, _P, _L, _I, _I, _P, _P, _P],
    "fs2_length_regulator_backward": [_P, _P, _P, _I, _I, _I, _I, _P, _P],
    "fs2_rowdot": [_P, _P, _P, _P, _L, _I, _I, _P, _P],
    "fs2_rowdot_backward": [_P, _P, _P, _P, _L, _I, _I, _P, _P, _P, _P],
    "fs2_loss_backward": [_P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P],
    "fs2_colsum_det_ws_bytes": [_L, _I, C.POINTER(_SZ)],
    "fs2_colsum_det": [_P, _L, _I, _P, _P, _SZ, _P],
    "fs2_conv_wgrad_det_ws_bytes": [_I, _I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_conv_wgrad_det": [_P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_layernorm_backward_det_ws_bytes": [_L, _I, C.POINTER(_SZ)],
    "fs2_layernorm_backward_det": [_P, _P, _P, _F, _L, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_batchnorm_train_det_ws_bytes": [_L, _I, C.POINTER(_SZ)],
    "fs2_batchnorm_train_det": [_P, _L, _I, _P, _P, _F, _F, _I, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_batchnorm_backward_det_ws_bytes": [_L, _I, C.POINTER(_SZ)],
    "fs2_batchnorm_backward_det": [_P, _P, _P, _P, _F, _L, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_embed_backward_det_ws_bytes": [_I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_embed_backward_det": [_P, _P, _P, _I, _I, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_onehot_linear_backward_det_ws_bytes": [_L, _I, _I, C.POINTER(_SZ)],
    "fs2_onehot_linear_backward_det": [_P, _P, _L, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_rowdot_backward_det_ws_bytes": [_L, _I, C.POINTER(_SZ)],
    "fs2_rowdot_backward_det": [_P, _P, _P, _P, _L, _I, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_masked_losses_det_ws_bytes": [_I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_masked_losses_det": [_P, _P, _P, _I, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _P, _P, _SZ, _P],
    "fs2_stft_frames": [_P, _I, _I, _I, _I, _I, _P, _P],
    "fs2_stft_magphase": [_P, _I, _I, _I, _I, _P, _P, _P],
    "fs2_istft_recombine": [_P, _P, _I, _I, _I, _I, _P, _P],
    "fs2_istft_overlap_add": [_P, _I, _I, _I, _I, _P, _F, _P, _P],
    "fs2_vocoder_create": [C.POINTER(_P), C.POINTER(VocoderConfig)],
    "fs2_vocoder_load": [_P, _P, _P, _P, _P, _P],
    "fs2_vocoder_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_mel_magnitude": [_P, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_griffin_lim": [_P, _P, _P, _I, _I, _I, _F, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_features_create": [C.POINTER(_P), C.POINTER(FeaturesConfig)],
    "fs2_features_load": [_P, _P, _P, _P],
    "fs2_features_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_mel_energy": [_P, _P, _P, _I, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_dio": [_P, _P, _P, _I, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_dtw_workspace_bytes": [_I, _I, _I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_mcd_dtw": [_P, _P, _I, _P, _P, _I, _I, _I, _P, _I, C.c_double, _P, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_path_prosody": [_P, _P, _I, _I, _P, _P, _I, _P, _P, _I, _P, _I, _P, _I, _P, _P, _P, _P],
    "fs2_mcd_dtw_cep": [_P, _P, _I, _P, _P, _I, _I, _I, C.c_double, _P, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_world_workspace_bytes": [C.POINTER(WorldConfig), _I, _I, _I, C.POINTER(_SZ)],
    "fs2_stonemask": [C.POINTER(WorldConfig), _P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _SZ, _P],
    "fs2_cheaptrick": [C.POINTER(WorldConfig), _P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _SZ, _P],
    "fs2_mcep": [C.POINTER(WorldConfig), _P, _P, _I, _I, _P, _P, _I, _P, _P, _P, _SZ, _P],
    "fs2_resample_workspace_bytes": [_I, _I, _I, _I, _I, C.POINTER(_SZ)],
    "fs2_resample": [_P, _P, _I, _I, _P, _I, _I, _P, _P, _I, _P, _P, _SZ, _P],
    "fs2_align_workspace_bytes": [_I, _I, _I, C.POINTER(_SZ)],
    "fs2_align_logprob": [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_align_logprob_backward": [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_align_forward_sum": [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_align_mas": [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _SZ, _P],
    "fs2_align_bin_loss": [_P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_align_mask_rows": [_P, _P, _I, _I, _I, _P, _P],
    "fs2_melgan_create": [C.POINTER(_P), _I],
    "fs2_melgan_load": [_P, C.POINTER(_P), C.POINTER(_P), _P],
    "fs2_melgan_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_melgan": [_P, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_melgan_window_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_melgan_window": [_P, _P, _P, _P, _I, _I, _I, _P, _L, _P, _P, _SZ, _P],
    "fs2_op_melgan_block": [_I, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "fs2_op_melgan_upsample": [_I, _I, _I, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P],
    "fs2_hifigan_create": [C.POINTER(_P), _I, C.POINTER(HiFiGANConfig)],
    "fs2_hifigan_load": [_P, C.POINTER(_P), C.POINTER(_P), _P],
    "fs2_hifigan_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_hifigan": [_P, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_hifigan_window_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_hifigan_window": [_P, _P, _P, _P, _I, _I, _I, _P, _L, _P, _P, _SZ, _P],
    "fs2_op_hifigan_resblock": [_I, _I, _I, _I, _I, C.POINTER(_I), _P, _P, _I, _I, C.POINTER(_P), C.POINTER(_P), _P, _P, _P],
    "fs2_op_hifigan_upsample": [_I, _I, _I, _I, _P, _P, _I, _I, _P, _P, _P, _P, _P],
    "fs2_bigvgan_create": [C.POINTER(_P), _I, C.POINTER(BigVGANConfig)],
    "fs2_bigvgan_load": [_P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), _P],
    "fs2_bigvgan_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_bigvgan": [_P, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_bigvgan_window_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_bigvgan_window": [_P, _P, _P, _P, _I, _I, _I, _P, _L, _P, _P, _SZ, _P],
    "fs2_op_bigvgan_act": [_I, _I, _P, _P, _I, _I, C.POINTER(_P), _I, _I, _P, _P, _P],
    "fs2_op_bigvgan_resblock": [_I, _I, _I, _I, _I, C.POINTER(_I), _P, _P, _I, _I, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P), _I, _I, _P,
                                _P, _P],
    "fs2_istftnet_create": [C.POINTER(_P), _I, C.POINTER(ISTFTNetConfig)],
    "fs2_istftnet_load": [_P, C.POINTER(_P), C.POINTER(_P), _P],
    "fs2_istftnet_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_istftnet": [_P, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_istftnet_window_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_istftnet_window": [_P, _P, _P, _P, _I, _I, _I, _P, _L, _P, _P, _SZ, _P],
    "fs2_op_istftnet_head": [_I, _I, _I, _P, _P, _I, _I, _P, _P, _P, _P],
    "fs2_waveglow_create": [C.POINTER(_P), _I, _I],
    "fs2_waveglow_load": [_P, C.POINTER(_P), _I, _P],
    "fs2_waveglow_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_waveglow": [_P, _P, _P, _I, _I, C.c_double, _P, _P, _P, _P, _P, _SZ, _P],
    "fs2_waveglow_noise": [_P, _P, _I, _I, _P, _P],
    "fs2_op_waveglow_upsample": [_P, _P, _P, _I, _I, _P, _P, _P, _P],
    "fs2_op_waveglow_flow": [_P, _I, _P, _P, _P, _P, _P, _I, _I, _P, _P, _P],
    "fs2_waveglow_window_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_waveglow_window": [_P, _P, _P, _P, _I, _I, _I, C.c_double, _P, _P, _P, _L, _P, _P, _SZ, _P],
    "fs2_ecapa_create": [C.POINTER(_P), _I, C.POINTER(ECAPAConfig)],
    "fs2_ecapa_n_tensors": [C.POINTER(ECAPAConfig)],
    "fs2_ecapa_load": [_P, C.POINTER(_P), _I, _P],
    "fs2_ecapa_workspace_bytes": [_P, _I, _I, C.POINTER(_SZ)],
    "fs2_ecapa": [_P, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_op_ecapa_stage": [_P, _I, _P, _P, _I, _I, _P, _P, _P, _SZ, _P],
    "fs2_peer_alloc": [_SZ, C.POINTER(_P), _P],
    "fs2_peer_free": [_P],
    "fs2_peer_open": [_P, C.POINTER(_P)],
    "fs2_peer_close": [_P],
    "fs2_peer_copy": [_P, _P, _SZ, _P],
    "fs2_flag_signal": [_P, _L, _P],
    "fs2_flag_wait": [_P, _I, _I, _L, _P],
    "fs2_optim_ws_bytes": [_P, _I, C.POINTER(_SZ)],
    "fs2_optim_noam_adam": [_P, _P, _I, C.POINTER(NoamAdamHp), _P, _P, _P, _SZ, _P],
    "fs2_optim_clip_noam_adam": [_P, _P, _I, C.POINTER(NoamAdamHp), _F, _P, _P, _P, _P, _SZ, _P],
    "fs2_optim_noam_scalars": [_L, _I, C.POINTER(NoamAdamHp), _P, _P, _P, _P],
}
OTHER_SYMBOLS = ("fs2_last_error", "fs2_version", "fs2_destroy", "fs2_kernel_launches", "fs2_profile_label", "fs2_vocoder_destroy",
                 "fs2_melgan_destroy", "fs2_waveglow_destroy", "fs2_features_destroy", "fs2_hifigan_destroy",
                 "fs2_bigvgan_destroy", "fs2_istftnet_destroy", "fs2_ecapa_destroy")
ALL_SYMBOLS = tuple(SIGNATURES) + OTHER_SYMBOLS

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """dlopen the in-tree library and set prototypes.  Raises if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Fs2Error(
            f"{LIB_PATH} not found: build it with `python -m fastspeech2_b200.build` "
            "(there is no CPU / PyTorch fallback for this path)")
    lib = C.CDLL(LIB_PATH)
    for name, args in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = C.c_int
    lib.fs2_last_error.restype = C.c_char_p
    lib.fs2_last_error.argtypes = []
    lib.fs2_version.restype = C.c_char_p
    lib.fs2_version.argtypes = []
    lib.fs2_kernel_launches.restype = C.c_ulonglong
    lib.fs2_kernel_launches.argtypes = []
    lib.fs2_profile_label.restype = C.c_char_p
    lib.fs2_profile_label.argtypes = [_I]
    lib.fs2_destroy.restype = None
    lib.fs2_destroy.argtypes = [_P]
    lib.fs2_vocoder_destroy.restype = None
    lib.fs2_vocoder_destroy.argtypes = [_P]
    lib.fs2_melgan_destroy.restype = None
    lib.fs2_melgan_destroy.argtypes = [_P]
    lib.fs2_waveglow_destroy.restype = None
    lib.fs2_waveglow_destroy.argtypes = [_P]
    lib.fs2_features_destroy.restype = None
    lib.fs2_features_destroy.argtypes = [_P]
    lib.fs2_hifigan_destroy.restype = None
    lib.fs2_hifigan_destroy.argtypes = [_P]
    lib.fs2_bigvgan_destroy.restype = None
    lib.fs2_bigvgan_destroy.argtypes = [_P]
    lib.fs2_istftnet_destroy.restype = None
    lib.fs2_istftnet_destroy.argtypes = [_P]
    lib.fs2_ecapa_destroy.restype = None
    lib.fs2_ecapa_destroy.argtypes = [_P]
    lib.fs2_embed_posenc = _embed_posenc_with_optional_planes(lib.fs2_embed_posenc)
    _lib = lib
    return lib


def _embed_posenc_with_optional_planes(fn):
    """fs2_embed_posenc took no planes and lens before they were added to it: the binding still accepts that form,
    (xs, table, n_sym, pe, alpha, B, T, C, out, stream), and passes both as NULL."""
    def call(*args):
        if len(args) == len(fn.argtypes) - 2:
            args = args[:-1] + (None, None) + args[-1:]
        return fn(*args)
    call.argtypes = fn.argtypes
    return call


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().fs2_last_error().decode("utf-8", "replace")
        raise Fs2Error(f"{what} failed (code {rc}): {msg}")


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    """Device pointer of a contiguous CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise Fs2Error("expected a CUDA tensor: the H100 path has no CPU fallback")
    if not t.is_contiguous():
        raise Fs2Error("expected a contiguous tensor")
    return t.data_ptr()


def stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def dur_dtype(t: torch.Tensor) -> int:
    if t.dtype == torch.int64:
        return FS2_DUR_I64
    if t.dtype == torch.float32:
        return FS2_DUR_F32
    if t.dtype == torch.int32:
        return FS2_DUR_I32
    raise Fs2Error(f"durations must be int64, int32 or float32, got {t.dtype}")
