"""ctypes binding of libtts_b200.so (the C ABI in include/tts_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or a call fails, the product
path raises.  (The CPU oracle under oracle/ is test infrastructure and is never imported here.)
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtts_b200.so")
_lib = None


class HifiganConfigC(ctypes.Structure):
    _fields_ = [
        ("in_channels", ctypes.c_int),
        ("out_channels", ctypes.c_int),
        ("upsample_initial_channel", ctypes.c_int),
        ("cond_channels", ctypes.c_int),
        ("resblock_type", ctypes.c_int),
        ("num_upsamples", ctypes.c_int),
        ("upsample_factors", ctypes.c_int * 8),
        ("upsample_kernel_sizes", ctypes.c_int * 8),
        ("num_kernels", ctypes.c_int),
        ("resblock_kernel_sizes", ctypes.c_int * 8),
        ("num_dilations", ctypes.c_int),
        ("resblock_dilations", (ctypes.c_int * 8) * 8),
    ]


class FlowConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("channels", "hidden_channels", "kernel_size", "dilation_rate",
                                            "num_layers", "num_flows", "cond_channels")]


class TextEncoderConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "out_channels", "hidden_channels", "hidden_channels_ffn",
                                            "num_heads", "num_layers", "kernel_size", "rel_attn_window_size",
                                            "language_emb_dim")]


class SdpConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "hidden_channels", "kernel_size", "num_flows",
                                            "cond_channels", "language_emb_dim", "num_bins")] + \
               [("tail_bound", ctypes.c_float)]


class PosteriorConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "out_channels", "hidden_channels", "kernel_size",
                                            "dilation_rate", "num_layers", "cond_channels")]


class DurationPredictorConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "hidden_channels", "kernel_size", "cond_channels",
                                            "language_emb_dim")]


class Conv1dConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "out_channels", "kernel_size", "dilation", "padding",
                                            "transposed", "stride")]


class SpeakerEncoderConfigC(ctypes.Structure):
    _fields_ = [("input_dim", ctypes.c_int), ("proj_dim", ctypes.c_int), ("layers", ctypes.c_int * 4),
                ("num_filters", ctypes.c_int * 4)] + \
               [(n, ctypes.c_int) for n in ("encoder_type", "log_input", "use_torch_spec", "fft_size", "win_length",
                                            "hop_length")]


class GlowTTSConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "out_channels", "hidden_channels_enc", "hidden_channels_ffn",
                                            "num_heads", "num_layers_enc", "kernel_size_enc", "use_prenet", "mean_only",
                                            "hidden_channels_dp", "c_in_channels", "hidden_channels_dec",
                                            "kernel_size_dec", "dilation_rate", "num_flow_blocks", "num_block_layers",
                                            "num_splits", "num_squeeze", "sigmoid_scale")]


class ForwardTTSConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "hidden_channels", "out_channels", "enc_heads", "enc_layers",
                                            "enc_ffn", "dec_heads", "dec_layers", "dec_ffn", "proj_g_in", "dp_hidden",
                                            "dp_kernel", "use_pitch", "pitch_hidden", "pitch_kernel",
                                            "pitch_emb_kernel", "use_energy", "energy_hidden", "energy_kernel",
                                            "energy_emb_kernel", "pe_len")]


class MelganConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "out_channels", "base_channels", "proj_kernel", "res_kernel",
                                            "num_res_blocks", "num_upsamples")] + \
               [("upsample_factors", ctypes.c_int * 8), ("pqmf_bands", ctypes.c_int), ("pqmf_taps", ctypes.c_int)]


class WavegradConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "out_channels", "y_conv_channels", "x_conv_channels",
                                            "num_upsamples")] + \
               [("upsample_factors", ctypes.c_int * 8), ("dblock_out_channels", ctypes.c_int * 8),
                ("ublock_out_channels", ctypes.c_int * 8), ("upsample_dilations", (ctypes.c_int * 4) * 8)]


class PwganConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("num_res_blocks", "stacks", "num_upsamples")] + \
               [("upsample_factors", ctypes.c_int * 8)]


class UnivnetConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("in_channels", "out_channels", "hidden_channels", "cond_channels",
                                            "num_upsamples")] + \
               [("upsample_factors", ctypes.c_int * 8)] + \
               [(n, ctypes.c_int) for n in ("lvc_layers", "lvc_kernel_size", "kpnet_hidden_channels", "kpnet_conv_size")]


class OverflowConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "encoder_dim", "n_convs", "state_per_phone", "out_channels",
                                            "ar_order", "prenet_dim", "prenet_n_layers", "prenet_dropout",
                                            "memory_rnn_dim", "outputnet_n_layers")] + \
               [("outputnet_size", ctypes.c_int * 8), ("std_floor", ctypes.c_float)] + \
               [(n, ctypes.c_int) for n in ("has_decoder", "hidden_channels_dec", "kernel_size_dec", "dilation_rate",
                                            "num_flow_blocks", "num_block_layers", "num_splits", "num_squeeze",
                                            "sigmoid_scale")]


class Tacotron2ConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "out_channels", "r_init", "attention_type", "location_attn",
                                            "attention_norm", "prenet_bn", "prenet_dropout")]


class TacotronConfigC(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in ("n_vocab", "frame_channels", "out_channels", "r_init", "memory_size",
                                            "attention_type", "location_attn", "attention_norm", "prenet_bn",
                                            "prenet_dropout")]


# padding modes of b200tts_conv1d_create_padded (B200TTS_PAD_* in include/tts_b200.h)
PADDING_MODES = {"zeros": 0, "reflect": 1}


# b200tts_debug_conv1d_launch's arguments and its flag / activation values (B200TTS_DEBUG_* in include/tts_b200.h)
EPI_GATE, EPI_MASK_PRE, EPI_MASK_POST, EPI_ACCUM, EPI_SPLIT, EPI_ACCUM2 = 1, 2, 4, 8, 16, 32
ACT_NONE, ACT_RELU, ACT_TANH, ACT_LOGCLAMP = 0, 1, 2, 3


class DebugConvIOC(ctypes.Structure):
    _fields_ = [("x", ctypes.c_void_p), ("x_batch_stride", ctypes.c_longlong), ("x_channel_stride", ctypes.c_int),
                ("T", ctypes.c_int),
                ("xmask", ctypes.c_void_p), ("xmask_batch_stride", ctypes.c_longlong),
                ("in_slope", ctypes.c_float),
                ("cond", ctypes.c_void_p), ("cond_batch_stride", ctypes.c_longlong),
                ("y", ctypes.c_void_p), ("y_batch_stride", ctypes.c_longlong), ("y_channel_stride", ctypes.c_int),
                ("res", ctypes.c_void_p), ("res_batch_stride", ctypes.c_longlong), ("res_channel_stride", ctypes.c_int),
                ("ymask", ctypes.c_void_p), ("ymask_batch_stride", ctypes.c_longlong),
                ("y2", ctypes.c_void_p), ("y2_batch_stride", ctypes.c_longlong), ("y2_channel_stride", ctypes.c_int),
                ("split", ctypes.c_int),
                ("scale", ctypes.c_float), ("post_div", ctypes.c_float),
                ("act", ctypes.c_int), ("act_param", ctypes.c_float),
                ("flags", ctypes.c_int),
                ("B", ctypes.c_int),
                ("lens", ctypes.c_void_p), ("rate_out", ctypes.c_int), ("need_out", ctypes.c_int), ("rate_in", ctypes.c_int),
                ("need_in", ctypes.c_int),
                ("q_lo", ctypes.c_int), ("q_hi", ctypes.c_int), ("in_lo", ctypes.c_int), ("in_hi", ctypes.c_int)]


class AudioNormC(ctypes.Structure):
    _fields_ = [("signal_norm", ctypes.c_int), ("symmetric_norm", ctypes.c_int), ("clip_norm", ctypes.c_int),
                ("max_norm", ctypes.c_float), ("min_level_db", ctypes.c_float), ("ref_level_db", ctypes.c_float),
                ("scaler_mean", ctypes.c_void_p), ("scaler_scale", ctypes.c_void_p)]


DISPATCH_NAMES = {0: "fma", 3: "tc3", 5: "tc3_grouped", 6: "row1", 8: "tc16", 9: "tc16_grouped", 10: "attn_tc3",
                  11: "attn_fma", 12: "tc3w_tf32", 13: "tc3w_tf32_near", 14: "tc3w_f16x3", 15: "tc3w_f16x3_near",
                  16: "fma_wg", 17: "fma_wg_near", 18: "lstm_bi", 19: "lstm_cell", 20: "hmm_linear", 21: "hmm_step",
                  22: "pwgan_tc", 23: "pwgan_aux", 24: "taco_attn", 25: "taco_step", 26: "lstm_cell32",
                  27: "univnet_predict", 28: "univnet_lvc", 29: "gru_cell", 30: "gru_cell32", 31: "bigru",
                  32: "highway", 33: "taco1_step", 34: "gl_prepare", 35: "gl_iter", 36: "gl_deemphasis"}

# tensor-core operand precision (B200TTS_PRECISION_* in include/tts_b200.h)
PRECISIONS = {"fp32": 0, "bf16": 1, "fp16": 2, "tf32x3": 3, "f16x3": 4}


def precision_id(name):
    """B200TTS_PRECISION_* of ``"fp32"`` / ``"bf16"`` / ``"fp16"`` / ``"tf32x3"`` / ``"f16x3"``; ValueError for anything
    else."""
    if not isinstance(name, str) or name not in PRECISIONS:
        raise ValueError(f"tts_b200: precision must be one of {sorted(PRECISIONS)}, got {name!r}")
    return PRECISIONS[name]


def _declare(lib):
    vp, sz, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
    lib.b200tts_last_error.restype = ctypes.c_char_p
    lib.b200tts_launch_count.restype = ctypes.c_ulonglong
    lib.b200tts_version.restype = ci
    lib.b200tts_debug_tc_error.restype = ci
    lib.b200tts_debug_device_buffers.restype = ctypes.c_longlong
    lib.b200tts_debug_dispatch_begin.restype = None
    lib.b200tts_debug_dispatch_end.restype = ci
    lib.b200tts_debug_dispatch_end.argtypes = [vp, ci]
    lib.b200tts_conv1d_create.restype = ci
    lib.b200tts_conv1d_create.argtypes = [ctypes.POINTER(Conv1dConfigC), vp, vp, ci, ctypes.POINTER(vp)]
    lib.b200tts_conv1d_create_ex.restype = ci
    lib.b200tts_conv1d_create_ex.argtypes = [ctypes.POINTER(Conv1dConfigC), vp, vp, ci, ctypes.POINTER(vp)]
    lib.b200tts_conv1d_create_padded.restype = ci
    lib.b200tts_conv1d_create_padded.argtypes = [ctypes.POINTER(Conv1dConfigC), vp, vp, ci, ci, ci, ctypes.POINTER(vp)]
    lib.b200tts_conv1d_forward_strided.restype = ci
    lib.b200tts_conv1d_forward_strided.argtypes = [vp, vp, ctypes.c_longlong, ci, ci, ci, ctypes.c_float, vp,
                                                   ctypes.c_float, ci, ctypes.c_float, ci, vp, vp, vp]
    lib.b200tts_debug_conv1d_create.restype = ci
    lib.b200tts_debug_conv1d_create.argtypes = [ctypes.POINTER(Conv1dConfigC), vp, vp, ci, ci, ci, ci, vp, vp,
                                                ctypes.POINTER(vp)]
    lib.b200tts_debug_conv1d_launch.restype = ci
    lib.b200tts_debug_conv1d_launch.argtypes = [vp, ctypes.POINTER(DebugConvIOC), vp]
    lib.b200tts_debug_attention.restype = ci
    lib.b200tts_debug_attention.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp]
    lib.b200tts_debug_add_layernorm.restype = ci
    lib.b200tts_debug_add_layernorm.argtypes = [ci, vp, vp, ci, vp, vp, vp, vp, ci, ci, ci, ctypes.c_float, vp]
    lib.b200tts_melgan_create.restype = ci
    lib.b200tts_melgan_create.argtypes = [ctypes.POINTER(MelganConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    lib.b200tts_melgan_destroy.restype = None
    lib.b200tts_melgan_destroy.argtypes = [vp]
    lib.b200tts_melgan_workspace_bytes.restype = sz
    lib.b200tts_melgan_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_melgan_out_len.restype = ci
    lib.b200tts_melgan_out_len.argtypes = [vp, ci]
    lib.b200tts_melgan_forward.restype = ci
    lib.b200tts_melgan_forward.argtypes = [vp, vp, ci, ci, ci, vp, vp, vp, sz, vp]
    lib.b200tts_wavegrad_create.restype = ci
    lib.b200tts_wavegrad_create.argtypes = [ctypes.POINTER(WavegradConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    lib.b200tts_wavegrad_destroy.restype = None
    lib.b200tts_wavegrad_destroy.argtypes = [vp]
    lib.b200tts_wavegrad_workspace_bytes.restype = sz
    lib.b200tts_wavegrad_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_wavegrad_forward.restype = ci
    lib.b200tts_wavegrad_forward.argtypes = [vp, vp, vp, vp, ctypes.POINTER(vp), ci, ci, ci, vp, vp, sz, vp]
    lib.b200tts_wavegrad_condition.restype = ci
    lib.b200tts_wavegrad_condition.argtypes = [vp, vp, ci, ci, vp, sz, vp]
    lib.b200tts_wavegrad_step.restype = ci
    lib.b200tts_wavegrad_step.argtypes = [vp, vp, vp, ctypes.POINTER(vp), ci, ctypes.c_float, ctypes.c_float,
                                          ctypes.c_float, vp, ci, ci, vp, sz, vp]
    ll = ctypes.c_longlong
    lib.b200tts_conv1d_forward_wavegrad.restype = ci
    lib.b200tts_conv1d_forward_wavegrad.argtypes = [vp, vp, ll, ci, ci, ci, ci, ctypes.c_float, ci, vp, vp, ll, ci, vp, ll,
                                                    ci, ci, vp, ll, ci, vp, vp]
    lib.b200tts_pwgan_create.restype = ci
    lib.b200tts_pwgan_create.argtypes = [ctypes.POINTER(PwganConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    lib.b200tts_pwgan_destroy.restype = None
    lib.b200tts_pwgan_destroy.argtypes = [vp]
    lib.b200tts_pwgan_workspace_bytes.restype = sz
    lib.b200tts_pwgan_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_pwgan_min_frames.restype = ci
    lib.b200tts_pwgan_min_frames.argtypes = [vp]
    lib.b200tts_pwgan_forward.restype = ci
    lib.b200tts_pwgan_forward.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, sz, vp]
    lib.b200tts_pwgan_layer.restype = ci
    lib.b200tts_pwgan_layer.argtypes = [vp, ci, vp, ci, ci, ci, vp, vp, vp, ci, vp, sz, vp]
    lib.b200tts_pwgan_upsample.restype = ci
    lib.b200tts_pwgan_upsample.argtypes = [vp, vp, ci, ci, vp, vp]
    lib.b200tts_univnet_create.restype = ci
    lib.b200tts_univnet_create.argtypes = [ctypes.POINTER(UnivnetConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    lib.b200tts_univnet_destroy.restype = None
    lib.b200tts_univnet_destroy.argtypes = [vp]
    lib.b200tts_univnet_workspace_bytes.restype = sz
    lib.b200tts_univnet_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_univnet_forward.restype = ci
    lib.b200tts_univnet_forward.argtypes = [vp, vp, vp, ci, ci, vp, vp, sz, vp]
    lib.b200tts_univnet_predict.restype = ci
    lib.b200tts_univnet_predict.argtypes = [vp, ci, vp, ci, ci, vp, vp, sz, vp]
    lib.b200tts_univnet_lvc_layer.restype = ci
    lib.b200tts_univnet_lvc_layer.argtypes = [vp, ci, ci, vp, vp, ci, ci, vp, ci, vp]
    lib.b200tts_pqmf_synthesis.restype = ci
    lib.b200tts_pqmf_synthesis.argtypes = [vp, ci, ci, ci, vp, ci, vp, vp, vp]
    lib.b200tts_conv1d_destroy.restype = None
    lib.b200tts_conv1d_destroy.argtypes = [vp]
    lib.b200tts_conv1d_out_len.restype = ci
    lib.b200tts_conv1d_out_len.argtypes = [vp, ci]
    lib.b200tts_conv1d_forward.restype = ci
    lib.b200tts_conv1d_forward.argtypes = [vp, vp, ci, ci, ctypes.c_float, vp, ctypes.c_float, ci, ctypes.c_float, vp, vp]
    lib.b200tts_hifigan_forward_ex.restype = ci
    lib.b200tts_hifigan_forward_ex.argtypes = [vp, vp, vp, ci, ci, vp, vp, vp, vp, sz, vp]
    lib.b200tts_hifigan_forward_window.restype = ci
    lib.b200tts_hifigan_forward_window.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp, vp, vp, vp, sz, vp]
    lib.b200tts_hifigan_margin_frames.restype = ci
    lib.b200tts_hifigan_margin_frames.argtypes = [vp]
    lib.b200tts_flow_reverse_ragged.restype = ci
    lib.b200tts_flow_reverse_ragged.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, sz, vp]
    lib.b200tts_vocoder_input_len.restype = ci
    lib.b200tts_vocoder_input_len.argtypes = [ci, ctypes.c_float, ci]
    lib.b200tts_vocoder_input.restype = ci
    lib.b200tts_vocoder_input.argtypes = [vp, ctypes.c_longlong, ci, ci, ci, ci, ci, ctypes.POINTER(AudioNormC),
                                          ctypes.POINTER(AudioNormC), ctypes.c_float, ci, vp, ci, vp]
    lib.b200tts_absmax.restype = ci
    lib.b200tts_absmax.argtypes = [vp, ctypes.c_longlong, vp, vp]
    lib.b200tts_to_int16.restype = ci
    lib.b200tts_to_int16.argtypes = [vp, ctypes.c_longlong, vp, vp, vp]
    lib.b200tts_mas_workspace_bytes.restype = sz
    lib.b200tts_mas_workspace_bytes.argtypes = [ci, ci, ci]
    lib.b200tts_mas.restype = ci
    lib.b200tts_mas.argtypes = [vp, vp, vp, vp, ci, ci, ci, vp, ci, vp, sz, vp]
    lib.b200tts_mas_from_stats_workspace_bytes.restype = sz
    lib.b200tts_mas_from_stats_workspace_bytes.argtypes = [ci, ci, ci]
    lib.b200tts_mas_from_stats.restype = ci
    lib.b200tts_mas_from_stats.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, ci, vp, ci, vp, vp, sz, vp]
    lib.b200tts_hifigan_create.restype = ci
    lib.b200tts_hifigan_create.argtypes = [ctypes.POINTER(HifiganConfigC), ctypes.POINTER(vp), ci,
                                           ctypes.POINTER(vp)]
    lib.b200tts_hifigan_create_ex.restype = ci
    lib.b200tts_hifigan_create_ex.argtypes = [ctypes.POINTER(HifiganConfigC), ctypes.POINTER(vp), ci, ci,
                                              ctypes.POINTER(vp)]
    lib.b200tts_hifigan_precision.restype = ci
    lib.b200tts_hifigan_precision.argtypes = [vp]
    lib.b200tts_hifigan_destroy.restype = None
    lib.b200tts_hifigan_destroy.argtypes = [vp]
    lib.b200tts_hifigan_workspace_bytes.restype = sz
    lib.b200tts_hifigan_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_hifigan_out_len.restype = ci
    lib.b200tts_hifigan_out_len.argtypes = [vp, ci]
    lib.b200tts_hifigan_forward.restype = ci
    lib.b200tts_hifigan_forward.argtypes = [vp, vp, vp, ci, ci, vp, vp, sz, vp]
    cf = ctypes.c_float
    for name, cfgt in (("flow", FlowConfigC), ("text_encoder", TextEncoderConfigC), ("sdp", SdpConfigC),
                       ("posterior", PosteriorConfigC), ("duration_predictor", DurationPredictorConfigC)):
        f = getattr(lib, f"b200tts_{name}_create")
        f.restype = ci
        f.argtypes = [ctypes.POINTER(cfgt), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
        f = getattr(lib, f"b200tts_{name}_destroy")
        f.restype = None
        f.argtypes = [vp]
        f = getattr(lib, f"b200tts_{name}_workspace_bytes")
        f.restype = sz
        f.argtypes = [vp, ci, ci]
    lib.b200tts_speaker_encoder_create.restype = ci
    lib.b200tts_speaker_encoder_create.argtypes = [ctypes.POINTER(SpeakerEncoderConfigC), ctypes.POINTER(vp), ci,
                                                   ctypes.POINTER(vp)]
    lib.b200tts_speaker_encoder_destroy.restype = None
    lib.b200tts_speaker_encoder_destroy.argtypes = [vp]
    lib.b200tts_speaker_encoder_workspace_bytes.restype = sz
    lib.b200tts_speaker_encoder_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_speaker_encoder_forward.restype = ci
    lib.b200tts_speaker_encoder_forward.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp, vp, sz, vp]
    lib.b200tts_speaker_encoder_features.restype = ci
    lib.b200tts_speaker_encoder_features.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, sz, vp]
    lib.b200tts_glow_tts_create.restype = ci
    lib.b200tts_glow_tts_create.argtypes = [ctypes.POINTER(GlowTTSConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    lib.b200tts_glow_tts_destroy.restype = None
    lib.b200tts_glow_tts_destroy.argtypes = [vp]
    lib.b200tts_glow_tts_workspace_bytes.restype = sz
    lib.b200tts_glow_tts_workspace_bytes.argtypes = [vp, ci, ci, ci]
    lib.b200tts_glow_tts_encode.restype = ci
    lib.b200tts_glow_tts_encode.argtypes = [vp, vp, vp, vp, ctypes.c_float, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                                            sz, vp]
    lib.b200tts_glow_tts_decode.restype = ci
    lib.b200tts_glow_tts_decode.argtypes = [vp, vp, vp, vp, vp, vp, vp, ctypes.c_float, ci, ci, ci, vp, vp, vp, vp, vp,
                                            sz, vp]
    lib.b200tts_forward_tts_create.restype = ci
    lib.b200tts_forward_tts_create.argtypes = [ctypes.POINTER(ForwardTTSConfigC), ctypes.POINTER(vp), ci,
                                               ctypes.POINTER(vp)]
    lib.b200tts_forward_tts_destroy.restype = None
    lib.b200tts_forward_tts_destroy.argtypes = [vp]
    lib.b200tts_forward_tts_encode_workspace_bytes.restype = sz
    lib.b200tts_forward_tts_encode_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_forward_tts_decode_workspace_bytes.restype = sz
    lib.b200tts_forward_tts_decode_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_forward_tts_encode.restype = ci
    lib.b200tts_forward_tts_encode.argtypes = [vp, vp, vp, vp, ctypes.c_float, ci, ci, vp, vp, vp, vp, vp, vp, vp, vp,
                                               vp, vp, sz, vp]
    lib.b200tts_forward_tts_decode.restype = ci
    lib.b200tts_forward_tts_decode.argtypes = [vp, vp, vp, vp, vp, ci, ci, ci, vp, vp, vp, sz, vp]
    lib.b200tts_attention_tc3.restype = ci
    lib.b200tts_attention_tc3.argtypes = [vp, vp, ci, ci, ci, ci, ci, vp, vp]
    lib.b200tts_stft_create.restype = ci
    lib.b200tts_stft_create.argtypes = [ci, ci, vp, vp, ci, ctypes.POINTER(vp)]
    lib.b200tts_stft_destroy.restype = None
    lib.b200tts_stft_destroy.argtypes = [vp]
    lib.b200tts_stft_magnitude.restype = ci
    lib.b200tts_stft_magnitude.argtypes = [vp, vp, ci, ci, ci, ci, ci, cf, vp, ci, vp]
    lib.b200tts_stft_mel_project.restype = ci
    lib.b200tts_stft_mel_project.argtypes = [vp, vp, ci, ci, cf, vp, vp]
    lib.b200tts_griffin_lim_create.restype = ci
    lib.b200tts_griffin_lim_create.argtypes = [ci, ci, vp, vp, ci, ctypes.POINTER(vp)]
    lib.b200tts_griffin_lim_destroy.restype = None
    lib.b200tts_griffin_lim_destroy.argtypes = [vp]
    lib.b200tts_griffin_lim_workspace_bytes.restype = sz
    lib.b200tts_griffin_lim_workspace_bytes.argtypes = [vp, ci, ci]
    lib.b200tts_griffin_lim_forward.restype = ci
    lib.b200tts_griffin_lim_forward.argtypes = [vp, vp, ctypes.c_longlong, ci, ci, ci, ci, ci, vp,
                                                ctypes.POINTER(AudioNormC), cf, cf, cf, ci, cf, vp, vp,
                                                ctypes.c_longlong, vp, vp, sz, vp]
    lib.b200tts_flow_create_forward.restype = ci
    lib.b200tts_flow_create_forward.argtypes = [ctypes.POINTER(FlowConfigC), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
    lib.b200tts_posterior_forward.restype = ci
    lib.b200tts_posterior_forward.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, vp, vp, sz, vp]
    lib.b200tts_duration_predictor_forward.restype = ci
    lib.b200tts_duration_predictor_forward.argtypes = [vp, vp, vp, vp, vp, ci, ci, vp, vp, sz, vp]
    lib.b200tts_upsample_linear.restype = ci
    lib.b200tts_upsample_linear.argtypes = [vp, ci, ci, cf, vp, ci, vp]
    lib.b200tts_flow_reverse.restype = ci
    lib.b200tts_flow_reverse.argtypes = [vp, vp, vp, vp, ci, ci, vp, sz, vp]
    lib.b200tts_text_encoder_forward.restype = ci
    lib.b200tts_text_encoder_forward.argtypes = [vp, vp, vp, vp, ci, ci, vp, vp, vp, vp, sz, vp]
    lib.b200tts_sdp_reverse.restype = ci
    lib.b200tts_sdp_reverse.argtypes = [vp, vp, vp, vp, vp, vp, cf, ci, ci, vp, vp, vp, sz, vp]
    lib.b200tts_durations.restype = ci
    lib.b200tts_durations.argtypes = [vp, vp, cf, ci, ci, vp, vp, vp, vp, vp, vp]
    lib.b200tts_expand_prior.restype = ci
    lib.b200tts_expand_prior.argtypes = [vp, vp, vp, vp, vp, cf, ci, ci, ci, ci, vp, vp, vp, vp, vp, vp]
    for name, cfgt in (("overflow", OverflowConfigC), ("tacotron2", Tacotron2ConfigC), ("tacotron", TacotronConfigC)):
        f = getattr(lib, f"b200tts_{name}_create")
        f.restype = ci
        f.argtypes = [ctypes.POINTER(cfgt), ctypes.POINTER(vp), ci, ctypes.POINTER(vp)]
        f = getattr(lib, f"b200tts_{name}_destroy")
        f.restype = None
        f.argtypes = [vp]
        f = getattr(lib, f"b200tts_{name}_workspace_bytes")
        f.restype = sz
        f.argtypes = [vp, ci, ci, ci]
        f = getattr(lib, f"b200tts_{name}_encode")
        f.restype = ci
        f.argtypes = [vp, vp, vp, ci, ci, vp, vp, sz, vp]
    lib.b200tts_overflow_sample.restype = ci
    lib.b200tts_overflow_sample.argtypes = [vp, vp, ci, ci, cf, ci, cf, vp, vp, ci, vp, vp, vp, vp, sz, vp]
    lib.b200tts_overflow_decode.restype = ci
    lib.b200tts_overflow_decode.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, sz, vp]
    for name in ("tacotron2", "tacotron"):
        f = getattr(lib, f"b200tts_{name}_decode_loop")
        f.restype = ci
        f.argtypes = [vp, vp, vp, ci, ci, ci, ci, vp, ci, vp, vp, vp, vp, vp, sz, vp]
        f = getattr(lib, f"b200tts_{name}_postnet")
        f.restype = ci
        f.argtypes = [vp, vp, vp, ci, ci, ci, vp, vp, sz, vp]


def lib():
    """The loaded CUDA library.  Raises (never falls back) when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"tts_b200: {LIB_PATH} is missing -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(tts_b200/csrc/build.sh).  There is no CPU fallback.")
        _lib = ctypes.CDLL(LIB_PATH)
        _declare(_lib)
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().b200tts_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"tts_b200.{what} failed (status {rc}): {msg}")


def ptr(t):
    """Raw device (or host) pointer of a tensor; None -> NULL."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr(device=None):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def require_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"tts_b200: `{name}` must be a CUDA tensor -- this package has no CPU path")
    return t


class dispatch_log:
    """``with dispatch_log() as log: ...`` -> ``log.names``: the kernel family of every conv launch inside the block."""

    def __enter__(self):
        lib().b200tts_debug_dispatch_begin()
        self.names = []
        return self

    def __exit__(self, *exc):
        buf = (ctypes.c_int32 * 4096)()
        n = lib().b200tts_debug_dispatch_end(buf, 4096)
        self.names = [DISPATCH_NAMES.get(int(buf[i]), str(int(buf[i]))) for i in range(min(n, 4096))]
        return False


def launch_count():
    return int(lib().b200tts_launch_count())


_workspaces = {}


def workspace(device, nbytes, tag="default"):
    """A cached per-(device, stream, tag) scratch buffer that only ever grows."""
    key = (device, torch.cuda.current_stream(device).cuda_stream, tag)
    buf = _workspaces.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
        _workspaces[key] = buf
    return buf
