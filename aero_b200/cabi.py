"""ctypes binding of libaero_b200.so (include/aero_b200.h).  Nothing but pointers, PODs and a stream
crosses this boundary.  Import fails loudly when the library is missing or cannot be loaded: there is
no CPU or eager-PyTorch fallback for the product path."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libaero_b200.so")

i32, i64, f32 = C.c_int32, C.c_int64, C.c_float
vp = C.c_void_p


class StftParams(C.Structure):
    _fields_ = [("n_fft", i32), ("hop", i32), ("win", i32), ("n_signals", i32), ("channels", i32),
                ("length", i32), ("frames", i32), ("bins_out", i32),
                ("z_stride_b", i64), ("z_stride_c", i64), ("z_stride_k", i64), ("z_stride_t", i64),
                ("flags", i32), ("reserved", i32)]


class IstftParams(C.Structure):
    _fields_ = [("n_fft", i32), ("hop", i32), ("win", i32), ("n_signals", i32), ("channels", i32),
                ("frames", i32), ("bins_in", i32), ("out_len", i32),
                ("z_stride_b", i64), ("z_stride_c", i64), ("z_stride_k", i64), ("z_stride_t", i64),
                ("flags", i32), ("reserved", i32)]


class TapGemmParams(C.Structure):
    _fields_ = [("B", i32), ("F_out", i32), ("T", i32), ("N", i32), ("F_in", i32), ("T_in", i32),
                ("C1", i32), ("C2", i32),
                ("mode", i32), ("kf", i32), ("kt", i32), ("stride_f", i32), ("pad_f", i32), ("dil_t", i32),
                ("pad_t", i32), ("f_out_offset", i32),
                ("act", i32), ("glu", i32), ("stats_mode", i32), ("groups", i32),
                ("a1_sb", i64), ("a1_sf", i64), ("a1_st", i64),
                ("a2_sb", i64), ("a2_sf", i64), ("a2_st", i64),
                ("w_sb", i64),
                ("o_sb", i64), ("o_sf", i64), ("o_st", i64),
                ("r_sb", i64), ("r_sf", i64), ("r_st", i64),
                ("cs_sb", i64), ("cs_st", i64),
                ("precision", i32), ("flags", i32)]


class NormActParams(C.Structure):
    _fields_ = [("B", i32), ("F_in", i32), ("F_out", i32), ("f_off", i32), ("T", i32), ("C", i32),
                ("groups", i32), ("scope", i32), ("op", i32), ("eps", f32), ("flags", i32)]


class LstmParams(C.Structure):
    _fields_ = [("rows", i32), ("T", i32), ("H", i32), ("n_win", i32), ("steps", i32), ("win_stride", i32),
                ("in_windowed", i32), ("out_windowed", i32), ("flags", i32), ("precision", i32)]


class FtbLinParams(C.Structure):
    _fields_ = [("B", i32), ("F", i32), ("T", i32), ("N", i32), ("J", i32), ("flags", i32),
                ("z_sb", i64), ("z_sf", i64), ("zm_sb", i64), ("zm_sf", i64)]


class AttnParams(C.Structure):
    _fields_ = [("rows", i32), ("T", i32), ("H", i32), ("heads", i32), ("ndecay", i32), ("ld", i32), ("flags", i32)]


class ResampleParams(C.Structure):
    _fields_ = [("B", i32), ("C", i32), ("L_in", i32), ("orig", i32), ("up", i32), ("width", i32), ("taps", i32),
                ("L_hr", i32), ("L_valid", i32), ("halo", i32), ("fill", i32), ("normalize", i32), ("floor_", f32)]


class GanTerm(C.Structure):
    _fields_ = [("x", vp), ("ref", vp), ("dx", vp), ("adv_scale", C.c_double), ("l1_scale", C.c_double),
                ("n_seg", i32), ("seg", i32), ("halo", i32), ("H", i32), ("C", i32), ("adv", i32)]


ABI_VERSION = 3
TAPS_CONV, TAPS_CONVT, TAPS_MIX = 0, 1, 2
ACT_NONE, ACT_GELU, ACT_RELU, ACT_LEAKY, ACT_TANH = 0, 1, 2, 3, 4
TG_ROUND_TF32, TG_A_F16, TG_OUT_F16, TG_REVERSE = 1, 2, 4, 8      # storage-type flags (AERO_TG_*)
NA_NONE, NA_GELU, NA_GLU, NA_SNAKE, NA_GLU_SCALE_RES, NA_RELU, NA_LEAKY, NA_TANH = 0, 1, 2, 3, 4, 5, 6, 7
NA_NO_NORM = 16
STFT_ZERO_PAD, STFT_ADJ_SCALE, ISTFT_RAW = 1, 2, 1
GAN_NONE, GAN_LSGAN_REAL, GAN_LSGAN_FAKE, GAN_LSGAN_GEN, GAN_HINGE_REAL, GAN_HINGE_FAKE, GAN_HINGE_GEN = 0, 1, 2, 3, 4, 5, 6
GAN_FWD_BLOCKS = 128                                              # AERO_GAN_FWD_BLOCKS

# every symbol include/aero_b200.h declares (tests/test_cabi.py checks the library exports them all)
SYMBOLS = {
    "aero_abi_version": (C.c_int, []),
    "aero_last_error": (C.c_char_p, []),
    "aero_device_arch": (C.c_int, []),
    "aero_launch_count": (C.c_uint64, []),
    "aero_stft_fwd": (C.c_int, [vp, vp, vp, vp, C.POINTER(StftParams), vp]),
    "aero_istft_fwd": (C.c_int, [vp, vp, vp, C.POINTER(IstftParams), vp]),
    "aero_tapgemm_fwd": (C.c_int, [vp] * 10 + [C.POINTER(TapGemmParams), vp]),
    "aero_tapgemm_tc_eligible": (C.c_int, [C.POINTER(TapGemmParams)]),
    "aero_sample_norm_fwd": (C.c_int, [vp, vp, vp, vp, i32, i64, i64, i32, vp]),
    "aero_norm_act_fwd": (C.c_int, [vp] * 8 + [C.POINTER(NormActParams), vp]),
    "aero_ftb_lin_out_fwd": (C.c_int, [vp] * 7 + [C.POINTER(FtbLinParams), vp]),
    "aero_ftb_lin_squeeze_fwd": (C.c_int, [vp, vp, vp, vp, i32, C.POINTER(FtbLinParams), vp]),
    "aero_freq_mix_small_fwd": (C.c_int, [vp, vp, vp, vp, i32, i32, i64, i32, vp]),
    "aero_lstm_rec_fwd": (C.c_int, [vp, vp, vp, vp, C.POINTER(LstmParams), vp]),
    "aero_lstm_tc_shape": (C.c_int, [i32, i32, i32, C.POINTER(i32)]),
    "aero_local_attn_fwd": (C.c_int, [vp, vp, C.POINTER(AttnParams), vp]),
    "aero_lsd_fwd": (C.c_int, [vp, vp, vp, i32, i32, i32, i32, vp]),
    "aero_lsd_varlen_fwd": (C.c_int, [vp, vp, i32, i32, vp, vp, vp, i32, i32, vp, vp, vp]),
    "aero_stft_loss_fwd": (C.c_int, [vp, vp, vp, i32, i32, i32, i32, vp]),
    "aero_stft_loss_bwd": (C.c_int, [vp, vp, vp, vp, i32, i32, i32, i32, f32, f32, vp]),
    # training (SURVEY.md section 8f rank 1)
    "aero_tapgemm_wgrad": (C.c_int, [vp, vp, vp, vp, C.POINTER(TapGemmParams), i64, i64, i64, vp]),
    "aero_colsum": (C.c_int, [vp, vp, vp, vp, i32, i32, i64, i64, i64, i64, i32, i64, i64, vp]),
    "aero_add": (C.c_int, [vp, vp, i64, f32, vp]),
    "aero_add_f64": (C.c_int, [vp, vp, i64, vp]),
    "aero_gram": (C.c_int, [vp, vp, vp, vp, i32, i32, i64, i64, i64, i64, vp]),
    "aero_bcast_add": (C.c_int, [vp, vp, i32, i32, i32, i32, vp]),
    "aero_scale_rows": (C.c_int, [vp, vp, vp, i32, i64, i32, vp]),
    "aero_norm_act_train_fwd": (C.c_int, [vp] * 8 + [C.POINTER(NormActParams), vp]),
    "aero_norm_act_train_bwd": (C.c_int, [vp] * 13 + [i32, C.POINTER(NormActParams), vp]),
    "aero_adam_step": (C.c_int, [vp, i32, f32, f32, f32, f32, i32, f32, vp]),
    "aero_pack_kmajor_tf32": (C.c_int, [vp, vp, vp, i32, i32, i32, vp]),
    "aero_split_tf32": (C.c_int, [vp, vp, vp, i64, vp]),
    "aero_tapgemm_wgrad_tc_eligible": (C.c_int, [C.POINTER(TapGemmParams), vp, vp, vp]),
    "aero_gconv1d_fwd": (C.c_int, [vp, vp, vp, vp] + [i32] * 9 + [vp]),
    "aero_gconv1d_dgrad": (C.c_int, [vp, vp, vp] + [i32] * 9 + [vp]),
    "aero_gconv1d_wgrad": (C.c_int, [vp, vp, vp] + [i32] * 9 + [vp]),
    "aero_weight_norm_fwd": (C.c_int, [vp, vp, vp, i32, i32, vp]),
    "aero_weight_norm_bwd": (C.c_int, [vp, vp, vp, vp, vp, i32, i32, vp]),
    "aero_lstm_train_fwd": (C.c_int, [vp] * 7 + [C.POINTER(LstmParams), vp]),
    "aero_lstm_bwd": (C.c_int, [vp] * 5 + [C.POINTER(LstmParams), vp]),
    "aero_lstm_fold": (C.c_int, [vp, vp, i32, i32, i32, i32, i32, i32, vp]),
    "aero_local_attn_train_fwd": (C.c_int, [vp, vp, vp, C.POINTER(AttnParams), vp]),
    "aero_local_attn_bwd": (C.c_int, [vp] * 5 + [C.POINTER(AttnParams), vp]),
    # SEANet generator
    "aero_seanet_input_fwd": (C.c_int, [vp, vp, vp, vp, C.POINTER(ResampleParams), vp]),
    "aero_resample_fwd": (C.c_int, [vp, vp, vp, i64, i32, i32, i32, i32, i32, i32, vp]),
    "aero_reflect_act_fwd": (C.c_int, [vp, vp, i32, i32, i32, i64, i64, i32, i32, i32, vp]),
    "aero_reflect_act_bwd": (C.c_int, [vp, vp, vp, i32, i32, i32, i64, i64, i32, i32, vp]),
    "aero_seanet_output_fwd": (C.c_int, [vp, vp, vp, vp, i32, i64, vp]),
    "aero_seanet_output_bwd": (C.c_int, [vp, vp, vp, vp, i32, i64, vp]),
    # HiFi-GAN multi-period discriminator
    "aero_mpd_fold_fwd": (C.c_int, [vp, vp] + [i32] * 6 + [vp]),
    "aero_mpd_fold_bwd": (C.c_int, [vp, vp] + [i32] * 6 + [vp]),
    "aero_mpd_repack_fwd": (C.c_int, [vp, vp] + [i32] * 6 + [f32, vp]),
    "aero_mpd_repack_bwd": (C.c_int, [vp, vp, vp] + [i32] * 6 + [f32, vp]),
    # GAN loss terms
    "aero_gan_loss_fwd": (C.c_int, [vp, i32, vp, vp, vp]),
    "aero_gan_loss_bwd": (C.c_int, [vp, i32, vp]),
    # ragged batches (clips of different lengths in one forward)
    "aero_stft_varlen_fwd": (C.c_int, [vp, vp, vp, vp, vp, C.POINTER(StftParams), vp]),
    "aero_istft_varlen_fwd": (C.c_int, [vp, vp, vp, vp, vp, C.POINTER(IstftParams), vp]),
    "aero_sample_norm_varlen_fwd": (C.c_int, [vp, vp, vp, vp, vp, i32, i64, i64, i32, vp]),
    "aero_masked_stats_fwd": (C.c_int, [vp, vp, vp] + [i32] * 7 + [vp]),
    "aero_frame_mask_fwd": (C.c_int, [vp, vp] + [i32] * 5 + [vp]),
    "aero_gather_rows_fwd": (C.c_int, [vp, vp, vp, vp, i64, i32, i32, i32, vp]),
    "aero_local_attn_varlen_fwd": (C.c_int, [vp, vp, vp, i32, C.POINTER(AttnParams), vp]),
    "aero_seanet_input_varlen_fwd": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.POINTER(ResampleParams), vp]),
    "aero_reflect_act_varlen_fwd": (C.c_int, [vp, vp, vp, i32, i32, i32, i64, i64, i32, i32, i32, vp]),
}


class AeroLibraryError(RuntimeError):
    pass


_lib = None


def load(path=None):
    """dlopen the kernel library and attach prototypes.  Raises AeroLibraryError if it is absent."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise AeroLibraryError(
            f"{path} not found: build it with `python -m aero_b200.build` (nvcc, sm_90a). "
            "aero_b200 has no CPU / eager fallback.")
    try:
        lib = C.CDLL(path)
    except OSError as e:  # pragma: no cover
        raise AeroLibraryError(f"cannot load {path}: {e}") from e
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    if lib.aero_abi_version() != ABI_VERSION:
        raise AeroLibraryError(f"{path} has ABI version {lib.aero_abi_version()}, this package needs {ABI_VERSION}: "
                               "rebuild with `python -m aero_b200.build`")
    _lib = lib
    return lib


def check(rc, lib=None):
    if rc != 0:
        lib = lib or load()
        raise AeroLibraryError(f"libaero_b200 error {rc}: {lib.aero_last_error().decode()}")
