"""ctypes loader for libpsb200.so (the C-ABI declared in include/psb200.h).

There is no CPU fallback: if the library is missing, or a call fails, this raises.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libpsb200.so")

MAX_FEAT = 8


class PsbError(RuntimeError):
    pass


class ModelDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_sen", C.c_int32), ("n_mgau", C.c_int32), ("n_feat", C.c_int32),
                ("n_density", C.c_int32), ("topn", C.c_int32), ("featlen", C.c_int32 * MAX_FEAT),
                ("ds_ratio", C.c_int32), ("aw", C.c_int32), ("logadd_ms_size", C.c_int32),
                ("logadd_ms_zero", C.c_int32), ("on_device", C.c_int32),
                ("mean", C.c_void_p), ("var", C.c_void_p), ("det", C.c_void_p), ("mixw", C.c_void_p),
                ("mixw_cb", C.c_void_p), ("sen2cb", C.c_void_p), ("logadd8", C.c_void_p),
                ("logadd_ms", C.c_void_p), ("topn_beam", C.c_void_p), ("fixed_point", C.c_int32)]


# every symbol include/psb200.h declares: (name, restype, argtypes)
_VP, _I32, _I64 = C.c_void_p, C.c_int32, C.c_int64
class FeDesc(C.Structure):
    _fields_ = [("frame_size", C.c_int32), ("frame_shift", C.c_int32), ("fft_size", C.c_int32), ("fft_order", C.c_int32),
                ("n_filt", C.c_int32), ("n_cep", C.c_int32), ("remove_dc", C.c_int32), ("remove_noise", C.c_int32),
                ("transform", C.c_int32), ("lifter_val", C.c_int32), ("window", C.c_int32), ("cmn", C.c_int32),
                ("n_coeffs", C.c_int32), ("pre_emphasis_alpha", C.c_float), ("sqrt_inv_n", C.c_float),
                ("sqrt_inv_2n", C.c_float), ("hamming", C.c_void_p), ("ccc", C.c_void_p), ("sss", C.c_void_p),
                ("spec_start", C.c_void_p), ("filt_start", C.c_void_p), ("filt_width", C.c_void_p),
                ("filt_coeffs", C.c_void_p), ("mel_cosine", C.c_void_p), ("lifter", C.c_void_p)]


class FeOpts(C.Structure):
    _fields_ = [("feat", C.c_int32), ("cmn", C.c_int32), ("varnorm", C.c_int32), ("dither", C.c_int32), ("seed", C.c_int32),
                ("cmn_init", C.c_float * 32), ("agc", C.c_int32), ("agc_thresh", C.c_float), ("lda", C.c_void_p),
                ("lda_rows", C.c_int32), ("lda_cols", C.c_int32), ("ldadim", C.c_int32)]


class FeState(C.Structure):
    _fields_ = [("cmn_mean", C.c_float * 32), ("cmn_sum", C.c_float * 32), ("cmn_nframe", C.c_int32), ("mt_index", C.c_int32),
                ("mt", C.c_uint32 * 624), ("agc_max", C.c_float), ("agc_obs_max", C.c_float), ("agc_obs_max_sum", C.c_float),
                ("agc_obs_frame", C.c_int32), ("agc_obs_utt", C.c_int32)]


class FeNoise(C.Structure):
    _fields_ = [("undefined", C.c_int32), ("reserved", C.c_int32), ("power", C.c_double * 64), ("noise", C.c_double * 64),
                ("floor", C.c_double * 64), ("peak", C.c_double * 64)]


class FsgDesc(C.Structure):
    _fields_ = [("n_pnode", C.c_int32), ("pnodes", C.c_void_p), ("n_state", C.c_int32), ("roots", C.c_void_p),
                ("n_link", C.c_int32), ("links", C.c_void_p), ("nulloff", C.c_void_p), ("nullarc", C.c_void_p),
                ("n_ciphone", C.c_int32), ("silcipid", C.c_int32), ("start_state", C.c_int32), ("beam", C.c_int32),
                ("pbeam", C.c_int32), ("wbeam", C.c_int32), ("maxhmmpf", C.c_int32)]


class VadOpts(C.Structure):
    _fields_ = [("mode", C.c_int32), ("sample_rate", C.c_int32), ("frame_length", C.c_double), ("window", C.c_double),
                ("ratio", C.c_double), ("warmup", C.c_int32)]


class PitchOpts(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("smooth_window", C.c_int32), ("flen", C.c_double), ("fshift", C.c_double),
                ("voice_thresh", C.c_double), ("search_range", C.c_double)]


class NgramDesc(C.Structure):
    _fields_ = [("info", C.c_void_p), ("model", C.c_void_p), ("model_len", C.c_int64), ("ci_tmat", C.c_void_p),
                ("ci_ssid", C.c_void_p), ("lm_arrays", C.c_void_p), ("lm_arrays_len", C.c_int64)]


SYMBOLS = [
    ("psb_last_error", C.c_char_p, []),
    ("psb_abi_version", C.c_int, []),
    ("psb_device_count", C.c_int, []),
    ("psb_model_create", C.c_int, [C.POINTER(ModelDesc), C.c_int, C.POINTER(_VP)]),
    ("psb_model_free", None, [_VP]),
    ("psb_model_update_gaussians", C.c_int, [_VP, _VP, _VP, _VP]),
    ("psb_model_n_sen", C.c_int, [_VP]),
    ("psb_model_device", C.c_int, [_VP]),
    ("psb_scorer_create", C.c_int, [_VP, _I32, C.POINTER(_VP)]),
    ("psb_scorer_free", None, [_VP]),
    ("psb_scorer_reset", C.c_int, [_VP]),
    ("psb_scorer_set_frame_idx", C.c_int, [_VP, _I32]),
    ("psb_scorer_get_frame_idx", _I32, [_VP]),
    ("psb_scorer_frame_eval", C.c_int, [_VP, _VP, _VP, _I32, _VP, _I32, _I32]),
    ("psb_batch_create", C.c_int, [_VP, _I32, _I64, C.POINTER(_VP)]),
    ("psb_batch_free", None, [_VP]),
    ("psb_batch_score_host", C.c_int, [_VP, _VP, _VP, _I32, _VP]),
    ("psb_batch_score_device", C.c_int, [_VP, _VP, _VP, _I32, _VP]),
    ("psb_batch_sync", C.c_int, [_VP]),
    ("psb_batch_senscr_device", _VP, [_VP]),
    ("psb_batch_last_kernel_ms", C.c_int, [_VP, _VP]),
    ("psb_batch_get_topn", C.c_int, [_VP, _VP, _I64]),
    ("psb_batch_event_record", C.c_int, [_VP, C.c_int]),
    ("psb_batch_event_elapsed_ms", C.c_int, [_VP, _VP]),
    ("psb_hmmctx_create", C.c_int, [_I32, _VP, _I32, _VP, _I32, _I32, C.c_int, C.POINTER(_VP)]),
    ("psb_hmmctx_free", None, [_VP]),
    ("psb_hmm_vit_eval_batch", C.c_int, [_VP, _VP, _I32, _VP, _VP]),
    ("psb_hmm_vit_eval_ptrs", C.c_int, [_VP, _VP, _I32, _VP, _VP]),
    ("psb_hmmset_create", C.c_int, [_VP, C.c_int64, _I32, C.POINTER(_VP)]),
    ("psb_hmmset_free", None, [_VP]),
    ("psb_hmmset_upload", C.c_int, [_VP, _VP, C.c_int64, _VP, _I32]),
    ("psb_hmmset_download", C.c_int, [_VP, _VP]),
    ("psb_hmmset_eval_frames_device", C.c_int, [_VP, _VP, _VP, _VP, _I32, _VP, C.POINTER(C.c_float)]),
    ("psb_batch_tc_check", C.c_int, [_VP, C.POINTER(C.c_float), C.POINTER(C.c_int32), _VP]),
    ("psb_batch_tc_counters", C.c_int, [_VP, _VP, _I32]),
    ("psb_batch_ms_plan", C.c_int, [_VP, _I64, _VP, _I32]),
    ("psb_batch_tm_plan", C.c_int, [_VP, _I64, _VP, _I32]),
    ("psb_hmmset_use_batch_stream", C.c_int, [_VP, _VP]),
    ("psb_hmmset_snapshot", C.c_int, [_VP]),
    ("psb_hmmset_restore", C.c_int, [_VP]),
    ("psb_hmmset_sweep_device", C.c_int, [_VP, _VP, _I64, _VP, _VP, _I32, _VP, C.POINTER(C.c_float)]),
    ("psb_hmmset_sweep_beam_device", C.c_int, [_VP, _VP, _I64, _VP, _VP, _I32, _I32, _I32, _I32, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_hmmset_eval_host", C.c_int, [_VP, _VP, _VP]),
    ("psb_allphone_batch_device", C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _VP, _I32, _VP]),
    ("psb_allphone_lm_batch_device", C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _VP, _VP, _VP, _VP, _I32, _VP]),
    ("psb_allphone_net_batch_device", C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP, _VP, _VP, _VP, _VP, _I32, _I32, _I32, _I32, _I32, _VP, _VP, _I32, _VP, _VP, _I32, _VP]),
    ("psb_allphone_lm_tables", C.c_int, [_VP, _I32, _VP, _VP]),
    ("psb_kws_batch_device", C.c_int, [_VP, _VP, _VP, _I32, _I32, _VP, _VP, _I32, _VP, _VP, _VP, _VP, _I32, _I32, _VP, _I32, _VP]),
    ("psb_fsg_batch_device", C.c_int, [_VP, C.POINTER(FsgDesc), _VP, _VP, _I32, _VP, _I32, _VP]),
    ("psb_ngram_fwdtree_batch_device", C.c_int, [_VP, C.POINTER(NgramDesc), _VP, _VP, _I32, _VP, _I32, _VP, _I32, _VP, _I32, _VP, _VP]),
    ("psb_ngram_fwdflat_batch_device", C.c_int, [_VP, C.POINTER(NgramDesc), _VP, _VP, _I32, _VP, _I32, _VP, _VP, _I32, _VP, _I32, _VP, _VP]),
    ("psb_selftest_block_scan", C.c_int, [C.c_int, _VP, _I32, _VP]),
    ("psb_fsg_find_exit", C.c_int, [_VP, _I32, _VP, _I32, _I32, _I32, _I32, _VP, _VP]),
    ("psb_fsg_backtrace", _I32, [_VP, _I32, _VP, _I32, _I32, _VP, _I32]),
    ("psb_ngram_find_exit", C.c_int, [_VP, _I32, _VP, _I32, _I32, _VP, _VP]),
    ("psb_ngram_backtrace", _I32, [_VP, _I32, _I32, _VP, _I32]),
    ("psb_ngram_segments", _I32, [C.POINTER(NgramDesc), _VP, _I32, _VP, _I32, _I32, C.c_float, _VP, _I32]),
    ("psb_ngram_two_pass_batch_device", C.c_int, [_VP, C.POINTER(NgramDesc), _VP, _VP, _I32, _VP, _I32, _I32, _I32, _VP, _I32, _VP, _I32,
                                                   _VP, _VP, _VP]),
    ("psb_align_batch_device", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    ("psb_align_last_kernel_ms", C.c_float, [_VP]),
    ("psb_align_last_token_bytes", C.c_int64, [_VP]),
    ("psb_align_batch_host", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    ("psb_fe_create", C.c_int, [C.POINTER(FeDesc), C.c_int, C.POINTER(_VP)]),
    ("psb_fe_free", None, [_VP]),
    ("psb_fe_n_frames", C.c_int32, [_VP, C.c_int64]),
    ("psb_fe_process_host", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP]),
    ("psb_fe_device_feats", _VP, [_VP]),
    ("psb_fe_feat_dim", C.c_int32, [_VP]),
    ("psb_decode_batch_pcm_host", C.c_int, [_VP, _VP, _VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP]),
    ("psb_fe_process_device", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_fe_create_ex", C.c_int, [C.POINTER(FeDesc), C.POINTER(FeOpts), C.c_int, C.POINTER(_VP)]),
    ("psb_fe_state_init", C.c_int, [_VP, C.POINTER(FeState)]),
    ("psb_fe_set_sessions", C.c_int, [_VP, _VP, _I32, _VP]),
    ("psb_fe_get_states", C.c_int, [_VP, _VP, _I32]),
    ("psb_fe_set_stream_starts", C.c_int, [_VP, _VP, _I32, _VP, _I32]),
    ("psb_fe_get_noise_states", C.c_int, [_VP, _VP, _I32]),
    ("psb_fe_set_filterbanks", C.c_int, [_VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _I32]),
    ("psb_fe_cancel_settings", C.c_int, [_VP]),
    ("psb_phoneloop_create", C.c_int, [_VP, _I32, _VP, _VP, _I32, _I32, _I32, _I32, C.c_double, C.POINTER(_VP)]),
    ("psb_phoneloop_free", None, [_VP]),
    ("psb_phoneloop_run_device", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP]),
    ("psb_phoneloop_run_host", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP]),
    ("psb_decode_batch_host", C.c_int, [_VP, _VP, _VP, _VP, _I32, _VP, _VP, _VP]),
    ("psb_decode_batch_device", C.c_int, [_VP, _VP, _VP, _VP, _I32, _VP, _VP]),
    ("psb_sendump_write", C.c_int, [C.c_char_p, C.c_char_p, _I32, C.c_double, _VP, _I64]),
    ("psb_sendump_read", _I64, [C.c_char_p, _VP, _VP, _I64]),
    ("psb_batch_set_pipeline", C.c_int, [_VP, C.c_int]),
    ("psb_vad_create", C.c_int, [C.POINTER(VadOpts), C.c_int, C.POINTER(_VP)]),
    ("psb_vad_free", None, [_VP]),
    ("psb_vad_frame_size", _I32, [_VP]),
    ("psb_vad_frame_length", C.c_double, [_VP]),
    ("psb_vad_sample_rate", _I32, [_VP]),
    ("psb_vad_start_frames", _I32, [_VP]),
    ("psb_vad_end_frames", _I32, [_VP]),
    ("psb_vad_maxlen", _I32, [_VP]),
    ("psb_vad_warmup", _I32, [_VP]),
    ("psb_vad_last_repairs", _I64, [_VP]),
    ("psb_vad_last_passes", _I32, [_VP]),
    ("psb_vad_process_host", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP]),
    ("psb_vad_process_device", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_vad_live_open", C.c_int, [_VP, _I32]),
    ("psb_vad_live_reset", C.c_int, [_VP, _VP, _I32]),
    ("psb_vad_feed_host", C.c_int, [_VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP]),
    ("psb_vad_feed_device", C.c_int, [_VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_pitch_create", C.c_int, [C.POINTER(PitchOpts), C.c_int, C.POINTER(_VP)]),
    ("psb_pitch_free", None, [_VP]),
    ("psb_pitch_frame_size", _I32, [_VP]),
    ("psb_pitch_frame_shift", _I32, [_VP]),
    ("psb_pitch_ndiff", _I32, [_VP]),
    ("psb_pitch_process_host", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_pitch_process_device", C.c_int, [_VP, _VP, _VP, _I32, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_pitch_live_open", C.c_int, [_VP, _I32]),
    ("psb_pitch_live_reset", C.c_int, [_VP, _VP, _I32]),
    ("psb_pitch_feed_host", C.c_int, [_VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_pitch_feed_device", C.c_int, [_VP, _VP, _I32, _VP, _VP, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)]),
    ("psb_kernel_launch_count", _I64, []),
    ("psb_device_bytes_live", _I64, []),
]

_lib = None


def lib():
    """Load libpsb200.so and bind every ABI symbol; raises if the library or a symbol is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PsbError("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback)" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, res, args in SYMBOLS:
            fn = getattr(L, name)           # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        raise PsbError("%s failed (%d): %s" % (what or "psb call", rc, lib().psb_last_error().decode()))
